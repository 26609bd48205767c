// Cached forward graphs of the denoiser engines (graph.cuh).
#include <algorithm>

#include "graph.cuh"

namespace rohm {

cudaError_t KernelPatch::apply(cudaGraphExec_t exec, cudaGraphNode_t node, const cudaKernelNodeParams& captured) const {
  void* args[kMaxArgs];
  std::copy(captured.kernelParams, captured.kernelParams + nargs_, args);
  for (int i = 0; i < n_; ++i) args[slots_[i].index] = const_cast<unsigned char*>(slots_[i].bytes);  // only read
  cudaKernelNodeParams kp = captured;
  kp.kernelParams = args;
  return cudaGraphExecKernelNodeSetParams(exec, node, &kp);
}

BranchEvents::~BranchEvents() {
  for (cudaEvent_t e : events_) cudaEventDestroy(e);
}

int BranchEvents::order_after(rohm_ctx* ctx, cudaStream_t from, cudaStream_t to) {
  if (from == to) return ROHM_OK;
  if (next_ == events_.size()) {
    cudaEvent_t e = nullptr;
    ROHM_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    events_.push_back(e);
  }
  cudaEvent_t e = events_[next_++];
  ROHM_CUDA(ctx, cudaEventRecord(e, from));
  ROHM_CUDA(ctx, cudaStreamWaitEvent(to, e, 0));
  return ROHM_OK;
}

ForwardGraphs::~ForwardGraphs() {
  if (capture_stream_) cudaStreamDestroy(capture_stream_);
}

int ForwardGraphs::run(rohm_ctx* ctx, int B, int T, StepKind step, bool eager, cudaStream_t st,
                       const std::function<int(cudaStream_t)>& launches, const std::vector<KernelPatch>& patches,
                       const std::vector<int>& lengths) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  ROHM_CUDA(ctx, cudaStreamIsCapturing(st, &cap));
  if (eager || !enabled || cap != cudaStreamCaptureStatusNone) return launches(st);

  Entry* g = nullptr;
  for (Entry& e : graphs_)
    if (e.B == B && e.T == T && e.step == step && e.lengths == lengths) g = &e;
  if (g == nullptr) {
    Entry e;
    e.B = B, e.T = T, e.step = step;
    e.lengths = lengths;
    const int rc = capture(ctx, launches, patches, &e);
    if (rc != ROHM_OK) return rc;
    if (graphs_.size() >= kMaxGraphs) graphs_.erase(graphs_.begin());
    graphs_.push_back(std::move(e));
    g = &graphs_.back();
  }
  for (size_t i = 0; i < patches.size(); ++i) ROHM_CUDA(ctx, patches[i].apply(g->exec.get(), g->nodes[i], g->params[i]));
  ROHM_CUDA(ctx, cudaGraphLaunch(g->exec.get(), st));
  return ROHM_OK;
}

int ForwardGraphs::capture(rohm_ctx* ctx, const std::function<int(cudaStream_t)>& launches,
                           const std::vector<KernelPatch>& patches, Entry* e) {
  // Capture on a private stream: the caller's stream may be the legacy default stream, which cannot be captured.
  // Nothing executes during capture; the instantiated graph is then launched on the caller's stream.
  if (capture_stream_ == nullptr) ROHM_CUDA(ctx, cudaStreamCreateWithFlags(&capture_stream_, cudaStreamNonBlocking));
  ROHM_CUDA(ctx, cudaStreamBeginCapture(capture_stream_, cudaStreamCaptureModeThreadLocal));
  const int rc = launches(capture_stream_);
  cudaGraph_t graph = nullptr;
  const cudaError_t ended = cudaStreamEndCapture(capture_stream_, &graph);
  e->graph.reset(graph);
  if (rc != ROHM_OK) return rc;
  ROHM_CUDA(ctx, ended);

  size_t n = 0;
  ROHM_CUDA(ctx, cudaGraphGetNodes(graph, nullptr, &n));
  std::vector<cudaGraphNode_t> nodes(n);
  ROHM_CUDA(ctx, cudaGraphGetNodes(graph, nodes.data(), &n));
  e->nodes.assign(patches.size(), nullptr);
  e->params.resize(patches.size());
  for (cudaGraphNode_t node : nodes) {
    cudaGraphNodeType type;
    ROHM_CUDA(ctx, cudaGraphNodeGetType(node, &type));
    if (type != cudaGraphNodeTypeKernel) continue;
    cudaKernelNodeParams kp{};
    ROHM_CUDA(ctx, cudaGraphKernelNodeGetParams(node, &kp));
    for (size_t i = 0; i < patches.size(); ++i) {
      if (kp.func != patches[i].func()) continue;
      if (e->nodes[i] != nullptr) return fail(ctx, ROHM_ERR_CUDA, "forward graph: boundary kernel %zu launched twice", i);
      e->nodes[i] = node, e->params[i] = kp;
    }
  }
  for (cudaGraphNode_t node : e->nodes)
    if (node == nullptr) return fail(ctx, ROHM_ERR_CUDA, "forward graph: could not locate the boundary kernel nodes");
  cudaGraphExec_t exec = nullptr;
  ROHM_CUDA(ctx, cudaGraphInstantiate(&exec, graph, 0));
  e->exec.reset(exec);
  return ROHM_OK;
}

}  // namespace rohm
