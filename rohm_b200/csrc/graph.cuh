// Cached CUDA graphs of a denoiser engine's forward (posenet.cu, trajnet.cu).  A forward, optionally followed by the sampler
// update, is captured once per shape and then issued as one cudaGraphLaunch.  The few kernels that touch caller memory (the
// boundary kernels) get those arguments replaced before every replay.
#pragma once
#include <cstring>
#include <functional>
#include <memory>
#include <tuple>
#include <type_traits>
#include <vector>

#include "common.h"

namespace rohm {

// Argument I of a boundary kernel, set to `value` on every replay.
template <size_t I, typename V>
struct Arg {
  V value;
};
template <size_t I, typename V>
Arg<I, V> arg(V value) {
  return {value};
}

// A boundary kernel and those of its arguments that change from call to call.  The kernel's function type gives the
// argument count and the type of every patched parameter: an index past the end, or a value whose type is not the
// parameter's (a pointer may gain const), does not compile.
class KernelPatch {
 public:
  template <typename... P, size_t... I, typename... V>
  KernelPatch(void (*kernel)(P...), Arg<I, V>... args)
      : func_(reinterpret_cast<const void*>(kernel)), nargs_(sizeof...(P)) {
    static_assert(sizeof...(P) <= kMaxArgs && sizeof...(I) <= kMaxPatched, "KernelPatch: raise kMaxArgs / kMaxPatched");
    (put<std::tuple_element_t<I, std::tuple<P...>>>(I, args.value), ...);
  }
  const void* func() const { return func_; }
  // Sets the arguments of `node` in `exec` to `captured` (the node's parameters as captured) with the patched ones replaced.
  cudaError_t apply(cudaGraphExec_t exec, cudaGraphNode_t node, const cudaKernelNodeParams& captured) const;

 private:
  static constexpr int kMaxArgs = 32, kMaxPatched = 8;
  struct Slot {
    size_t index;
    alignas(8) unsigned char bytes[8];
  };
  template <typename T, typename V>
  void put(size_t index, const V& value) {
    static_assert(std::is_same<V, T>::value || (std::is_pointer<V>::value && std::is_convertible<V, T>::value),
                  "KernelPatch: the value's type is not the kernel parameter's");
    static_assert(sizeof(T) <= sizeof(Slot::bytes), "KernelPatch: parameter wider than a slot");
    const T v = value;
    slots_[n_].index = index;
    std::memcpy(slots_[n_].bytes, &v, sizeof v);
    ++n_;
  }
  const void* func_;
  int nargs_;
  Slot slots_[kMaxPatched];
  int n_ = 0;
};

// Fork / join between the streams of a forward's parallel branches.  order_after(from, to): everything issued on `from` so
// far happens-before what is issued on `to` afterwards (event record + wait; during stream capture this adds a graph
// edge).  The events are reused from forward to forward: rewind() before each one.
class BranchEvents {
 public:
  BranchEvents() = default;
  BranchEvents(const BranchEvents&) = delete;
  BranchEvents& operator=(const BranchEvents&) = delete;
  ~BranchEvents();
  void rewind() { next_ = 0; }
  int order_after(rohm_ctx* ctx, cudaStream_t from, cudaStream_t to);

 private:
  std::vector<cudaEvent_t> events_;
  size_t next_ = 0;
};

// What a forward graph appends to the forward: nothing, the single-stream update (DdpmStep) or the per-clip one
// (DdpmClipStep).  Part of the graph key, since the two updates are different kernels.
enum StepKind : int { kNoStep = 0, kStepSingleStream = 1, kStepPerClip = 2 };

// An engine's captured forwards, keyed by (B, T, step kind, per-clip lengths); at most kMaxGraphs, the oldest evicted first.
class ForwardGraphs {
 public:
  static constexpr size_t kMaxGraphs = 8;
  bool enabled = true;  // false: every forward is launched eagerly

  ForwardGraphs() = default;
  ForwardGraphs(const ForwardGraphs&) = delete;
  ForwardGraphs& operator=(const ForwardGraphs&) = delete;
  ~ForwardGraphs();

  // Issues one forward on `st`.  launches(stream) issues its kernels on `stream`.  That runs directly on `st` when `eager`,
  // when graphs are off, or when the caller is capturing `st`.  Otherwise the graph of (B, T, step) is replayed with
  // the arguments of `patches` set; launches() is captured into it on first use.  Every call passes the same kernels in
  // `patches` for the same key.  `lengths` (empty: uniform clips) is part of the key: the packed layout it implies sets
  // grids and row counts that a replay cannot change.
  int run(rohm_ctx* ctx, int B, int T, StepKind step, bool eager, cudaStream_t st,
          const std::function<int(cudaStream_t)>& launches, const std::vector<KernelPatch>& patches,
          const std::vector<int>& lengths = {});
  void clear() { graphs_.clear(); }  // the next run() of every key captures again

 private:
  struct DestroyGraph {
    void operator()(cudaGraph_t g) const { cudaGraphDestroy(g); }
  };
  struct DestroyExec {
    void operator()(cudaGraphExec_t e) const { cudaGraphExecDestroy(e); }
  };
  struct Entry {
    int B = 0, T = 0;
    StepKind step = kNoStep;
    std::vector<int> lengths;
    std::unique_ptr<std::remove_pointer_t<cudaGraph_t>, DestroyGraph> graph;  // owns the captured arguments in `params`
    std::unique_ptr<std::remove_pointer_t<cudaGraphExec_t>, DestroyExec> exec;
    std::vector<cudaGraphNode_t> nodes;  // the boundary nodes, in the order of the patches
    std::vector<cudaKernelNodeParams> params;
  };
  int capture(rohm_ctx* ctx, const std::function<int(cudaStream_t)>& launches, const std::vector<KernelPatch>& patches,
              Entry* e);

  cudaStream_t capture_stream_ = nullptr;
  std::vector<Entry> graphs_;
};

// sampler.cu: the Philox-fused ancestral update that the engines append to their forward (rohm_posenet_sample_step,
// rohm_trajnet_sample_step).  x_next = coef_row-weighted x0, x_t and noise; the noise is what torch.randn_like would draw
// from the generator state (seed, offset).
struct DdpmStep {
  const float* x0;  // the forward's output
  const float* x_t;
  float* x_next;
  int64_t numel, clip_elems;
  const float* coef_row;  // one row for every clip
  unsigned long long seed, offset;
  int64_t G = 0;  // launch geometry of torch's normal_ for numel, set by ddpm_step_plan
  int iters = 0;
};
// Sets s->G and s->iters; *offset_increment (if not null) = what the generator's offset advances by.
int ddpm_step_plan(rohm_ctx* ctx, DdpmStep* s, uint64_t* offset_increment);
int launch_ddpm_step(rohm_ctx* ctx, const DdpmStep& s, cudaStream_t st, bool pdl);
// The update node's per-call arguments in a replayed graph.
KernelPatch ddpm_step_patch(const DdpmStep& s);

// Per-clip noise streams.  Clip b of a padded batch draws its noise from its own Philox stream, exactly as
// torch.randn(S_b, generator=g_b) draws it for the shape S_b the clip has alone: [1, C, 1, n_b] channel-major (PoseNet,
// padded layout [B][C][T]) or [1, n_b, C] channels-last (TrajNet, padded layout [B][T][C]).  Clip b uses the launch
// geometry torch's normal_ kernel picks for C * n_b elements; the launch concatenates the clips' grids, and blk[] (a prefix
// sum of the per-clip block counts) tells each block its clip.  Padded frames get zero.
constexpr int kMaxStreamClips = 256;  // keeps ClipPlan, a kernel parameter, within the 4 KB parameter space
struct ClipPlan {
  int B, C, T;
  int channels_last;                 // 0: [B][C][T], 1: [B][T][C]
  int blk[kMaxStreamClips + 1];      // clip b owns blocks [blk[b], blk[b + 1]); blk[B] = the grid
  int n[kMaxStreamClips];            // real frames of clip b
};
// Fills *p for B clips of C channels padded to T frames; lengths (host, NULL: all T).  incs (host [B], optional): what
// clip b's generator offset advances by per draw, as torch would advance it for the clip alone.
int clip_plan(rohm_ctx* ctx, int B, int C, int T, bool channels_last, const int* lengths, ClipPlan* p, uint64_t* incs);

// The per-clip form of DdpmStep (rohm_posenet_sample_step_clips, rohm_trajnet_sample_step_clips).  streams: device
// uint64 [B][2] of (seed, offset at draw 0); draw k of clip b starts at offset + k * incs[b].
struct DdpmClipStep {
  const float* x0;
  const float* x_t;
  float* x_next;
  const float* coef_row;  // one row for every clip
  const unsigned long long* streams;
  unsigned long long draw;
  ClipPlan plan;
};
int launch_ddpm_clip_step(rohm_ctx* ctx, const DdpmClipStep& s, cudaStream_t st, bool pdl);
KernelPatch ddpm_clip_step_patch(const DdpmClipStep& s);

}  // namespace rohm
