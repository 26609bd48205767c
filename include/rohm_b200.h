/* rohm_b200 -- C ABI of the H100-native RoHM hot path.
 *
 * The reference (sanweiliti/RoHM) is pure Python/PyTorch and has no FFI; its boundary is a set of Python symbols
 * (SURVEY.md 8b, layer A).  This header is layer B: the plain-C entry points the Python drop-in
 * (rohm_b200/dropin/{model,diffusion,utils}) binds with ctypes.  Each entry point names the reference code it
 * replaces (file:line @ 57ba22c).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to fp32 (or int64 where stated) unless marked "host";
 *   - `stream` is a cudaStream_t passed as void*; all calls are asynchronous on it;
 *   - no entry point allocates device memory except the *_create functions;
 *   - return value: 0 on success, negative rohm_status otherwise; rohm_last_error(ctx) gives the message;
 *   - one ctx per device/stream user; handles are not thread-safe.
 */
#ifndef ROHM_B200_H_
#define ROHM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define ROHM_API __attribute__((visibility("default")))
#else
#define ROHM_API
#endif

typedef enum {
  ROHM_OK = 0,
  ROHM_ERR_INVALID = -1,   /* bad argument / unsupported shape */
  ROHM_ERR_CUDA = -2,      /* CUDA runtime or driver error */
  ROHM_ERR_NO_DEVICE = -3, /* no sm_90 (H100) device */
  ROHM_ERR_STATE = -4      /* call order violated (e.g. forward before set_cond) */
} rohm_status;

/* Arithmetic mode of the tensor-core GEMMs. */
typedef enum {
  ROHM_PRECISION_TF32X3 = 3, /* error-compensated TF32 hi/lo pairs: fp32-grade results (parity mode) */
  ROHM_PRECISION_F16X2 = 2,  /* error-compensated fp16 hi/lo pairs: the same 2 x 11 significant bits per value in half
                                the bytes (fp32-grade results, the default of every engine; activations must stay below 1.3e5) */
  ROHM_PRECISION_TF32 = 1    /* single-pass TF32: ~1e-3 relative (fast mode) */
} rohm_precision;

typedef struct rohm_ctx rohm_ctx;
typedef struct rohm_posenet rohm_posenet;
typedef struct rohm_trajnet rohm_trajnet;
typedef struct rohm_body rohm_body;

ROHM_API int rohm_version(void);
ROHM_API int rohm_ctx_create(int device, rohm_ctx** out);
ROHM_API void rohm_ctx_destroy(rohm_ctx* ctx);
ROHM_API const char* rohm_last_error(const rohm_ctx* ctx);

/* ------------------------------------------------------------------------------------------------------------
 * Sampler arithmetic (diffusion/gaussian_diffusion_posenet.py and _trajnet.py)
 * ---------------------------------------------------------------------------------------------------------- */

/* One ancestral update over n_clips clips of clip_elems contiguous elements each (all operands share the layout):
 *   mean = c1*x0 + c2*x_t                           q_posterior_mean_variance  :212-234, p_mean_variance :236-280
 *   mean += gs_k*grad_k        for k < n_grads      p_sample_with_grad         :461-477 (gs = weight*variance[t])
 *   out  = mean + sigma*noise                       p_sample :426-434          (sigma = (t!=0)*exp(0.5*logvar[t]))
 * coef points to device rows of ROHM_DDPM_COEFS floats {c1, c2, sigma, gs0, gs1, unused, unused, unused}; clip b reads
 * row coef + b*coef_clip_stride (stride 0 = one row for the whole batch, e.g. a row of a per-step table uploaded once).
 * Products and sums are rounded individually (no FMA contraction) so the result matches the reference's chain of
 * separate elementwise kernels bit for bit.  grads may be NULL when n_grads == 0.  `out` may alias x_t. */
#define ROHM_DDPM_COEFS 8
ROHM_API int rohm_ddpm_step(rohm_ctx* ctx, const float* x0, const float* x_t, const float* noise, const float* grad0,
                            const float* grad1, int n_grads, float* out, int64_t n_clips, int64_t clip_elems,
                            const float* coef, int64_t coef_clip_stride, void* stream);

/* rohm_ddpm_step with the noise = th.randn_like(x) (:426, :458) drawn INSIDE the kernel: Philox4_32_10(seed, offset) consumed
 * exactly as torch's CUDA normal_ kernel consumes it for a tensor of n_clips*clip_elems fp32 elements on this device, so
 * with (seed, offset) = the state of torch's CUDA generator the result is bit-identical to
 * rohm_ddpm_step(..., noise = torch.randn_like(x), ...).  *offset_increment (host, optional) receives the amount the caller
 * must advance the generator's offset by afterwards (what torch itself would have added). */
ROHM_API int rohm_ddpm_step_philox(rohm_ctx* ctx, const float* x0, const float* x_t, const float* grad0, const float* grad1,
                                   int n_grads, float* out, int64_t n_clips, int64_t clip_elems, const float* coef,
                                   int64_t coef_clip_stride, uint64_t seed, uint64_t offset, uint64_t* offset_increment,
                                   void* stream);

/* Per-clip noise streams.  out: a padded batch of B clips of C channels and T frames, [B][C][T] (channels_last = 0, PoseNet
 * [B, C, 1, T]) or [B][T][C] (channels_last = 1, TrajNet [B, T, C]); clip b has lengths_host[b] real frames (1..T; NULL:
 * T).  streams: device uint64 [B][2], clip b's (seed, offset) at draw 0.  Clip b's real frames receive exactly what
 * torch.randn(S_b, generator=g_b) returns for a CUDA generator in state (seed_b, offset_b + draw * inc_b), S_b being
 * [1, C, 1, n_b] or [1, n_b, C]; its padded frames receive 0.  offset_increments (host uint64 [B], optional) receives inc_b,
 * what torch advances that generator's offset by for this draw.  At most 256 clips. */
ROHM_API int rohm_randn_clips(rohm_ctx* ctx, float* out, int B, int C, int T, int channels_last, const int* lengths_host,
                              const uint64_t* streams, uint64_t draw, uint64_t* offset_increments, void* stream);

/* rohm_ddpm_step with noise = rohm_randn_clips(same arguments) drawn inside the kernel: bit-identical to rohm_ddpm_step on
 * that noise tensor, and 0 in every clip's padded frames.  coef: device float[8] (coef_clip_stride = 0) or [B][8]
 * (coef_clip_stride = 8). */
ROHM_API int rohm_ddpm_step_philox_clips(rohm_ctx* ctx, const float* x0, const float* x_t, const float* grad0,
                                         const float* grad1, int n_grads, float* out, int B, int C, int T, int channels_last,
                                         const int* lengths_host, const float* coef, int64_t coef_clip_stride,
                                         const uint64_t* streams, uint64_t draw, uint64_t* offset_increments, void* stream);

/* q_sample :192-210:  out = sqrt_ac*x_start + sqrt_1m_ac*noise. */
ROHM_API int rohm_q_sample(rohm_ctx* ctx, const float* x_start, const float* noise, float* out, int64_t n, float sqrt_ac,
                  float sqrt_one_minus_ac, void* stream);

/* DDIM update as INTENDED by ddim_sample :665-715 (unreachable in the reference, see DESIGN.md):
 *   eps  = (sqrt_recip_ac*x_t - x0) / sqrt_recipm1_ac
 *   out  = x0*sqrt(ac_prev) + sqrt(1 - ac_prev - sigma^2)*eps + nonzero*sigma*noise
 * The four scalars are precomputed on the host from the float64 tables. */
ROHM_API int rohm_ddim_step(rohm_ctx* ctx, const float* x0, const float* x_t, const float* noise, float* out, int64_t n,
                   float sqrt_recip_ac, float sqrt_recipm1_ac, float sqrt_ac_prev, float dir_coef, float sigma,
                   void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * PoseNet denoiser (model/posenet.py:75-96, model/heads.py:112-176, nn.TransformerEncoder post-norm/gelu)
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct {
  const float* in_proj_w;  /* self_attn.in_proj_weight [3D, D] */
  const float* in_proj_b;  /* [3D] */
  const float* out_proj_w; /* self_attn.out_proj.weight [D, D] */
  const float* out_proj_b;
  const float* lin1_w; /* linear1.weight [F, D] */
  const float* lin1_b;
  const float* lin2_w; /* linear2.weight [D, F] */
  const float* lin2_b;
  const float* norm1_w;
  const float* norm1_b;
  const float* norm2_w;
  const float* norm2_b;
} rohm_posenet_layer;

typedef struct {
  int d_model;     /* latent_dim (512) */
  int ff_size;     /* 1024 */
  int num_layers;  /* 8 */
  int num_heads;   /* 4 */
  int in_feats;    /* body_feat_dim (294) */
  int out_feats;   /* pose_feat_dim (272) */
  int traj_feats;  /* channels copied from cond to the output (22) */
  int pe_len;      /* rows of the positional table (5000) */
  const float* in_w;   /* input_process.poseEmbedding.weight [D, in_feats] */
  const float* in_b;
  const float* cond_w; /* input_process_cond.poseEmbedding.weight [D, in_feats] */
  const float* cond_b;
  const float* pe;     /* sequence_pos_encoder.pe as [pe_len, D] */
  const float* t0_w;   /* embed_timestep.time_embed.0 [D, D] */
  const float* t0_b;
  const float* t2_w;   /* embed_timestep.time_embed.2 [D, D] */
  const float* t2_b;
  const float* out_w;  /* output_process.poseFinal.weight [out_feats, D] */
  const float* out_b;
  const rohm_posenet_layer* layers; /* host array of num_layers entries */
} rohm_posenet_weights;

/* Copies and repacks the weights (TF32 hi/lo split, K-padded) into library-owned device memory and allocates the
 * activation workspace for up to max_batch clips of max_frames frames.
 * Clip length (S = max_frames + 1 tokens): S <= pe_len always.  ROHM_PRECISION_F16X2 with head dim 128 (RoHM's
 * configuration) reaches S = pe_len (4999 frames with the 5000-row table) on the streaming wgmma attention kernel.
 * ROHM_PRECISION_TF32X3 / ROHM_PRECISION_TF32, and head dim 64, run clips above 160 tokens on the SIMT attention kernel,
 * which keeps the clip's K and V in shared memory: at most 211 frames at head dim 128 and 255 at head dim 64.  A longer
 * clip returns ROHM_ERR_INVALID with the rule in the message. */
ROHM_API int rohm_posenet_create(rohm_ctx* ctx, const rohm_posenet_weights* w, int max_batch, int max_frames, int precision,
                        rohm_posenet** out);
ROHM_API void rohm_posenet_destroy(rohm_posenet* pn);

/* Step-invariant part of PoseNet.forward (posenet.py:86, 90-91): input_process_cond(cond) + positional rows.
 * cond: [B, in_feats, 1, T] contiguous.  Must be called whenever batch['cond'], B or T change. */
ROHM_API int rohm_posenet_set_cond(rohm_posenet* pn, const float* cond, int B, int T, void* stream);

/* Per-clip lengths for the following set_cond, forward, sample_step and profile calls: clip b of the padded
 * [B, in_feats, 1, T] tensors has lengths_host[b] real frames, 1 <= lengths_host[b] <= T.  Frames [0, lengths[b]) of the
 * output equal a forward of that clip alone as a [1, in_feats, 1, lengths[b]] batch, bit for bit; frames past it are zero,
 * and the input values there are never read.  Inside, the clips' tokens are packed with no padding rows, so a batch of
 * mixed lengths does no wasted tensor work.  NULL returns to uniform clips of T frames.  Precision f16x2 with head dim 128
 * only (else ROHM_ERR_INVALID).  Changing the lengths waits for the device to go idle; call set_cond again afterwards. */
ROHM_API int rohm_posenet_set_lengths(rohm_posenet* pn, const int* lengths_host, int B);

/* PoseNet.forward (posenet.py:75-96).  x_t: [B, in_feats, 1, T]; timesteps: int64 [B] (original, un-respaced);
 * out: [B, in_feats, 1, T] with channels [0, traj_feats) copied from the cond given to set_cond. */
ROHM_API int rohm_posenet_forward(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B, int T,
                         void* stream);

/* One whole ancestral step of the PoseNet sampler (p_mean_variance :236-280 + p_sample :388-434) as ONE graph launch:
 * x0_out = PoseNet(x_t, timesteps) followed by x_next = c1 x0 + c2 x_t + sigma N(0, I) with the noise drawn in the update
 * kernel exactly as torch.randn_like(x_t) would draw it from (seed, offset) (see rohm_ddpm_step_philox).  coef_row: device
 * row {c1, c2, sigma, ...} of this step (shared by all clips).  *offset_increment: what to advance the generator by. */
ROHM_API int rohm_posenet_sample_step(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* x0_out,
                                      float* x_next, const float* coef_row, uint64_t seed, uint64_t offset,
                                      uint64_t* offset_increment, int B, int T, void* stream);

/* rohm_posenet_sample_step with per-clip noise streams: the update is rohm_ddpm_step_philox_clips over the engine's current
 * lengths (rohm_posenet_set_lengths), so clip b's frames past its length come out 0 in x_next.  streams: device
 * uint64 [B][2]; draw: this step's draw index; offset_increments: host uint64 [B] (optional), see rohm_randn_clips. */
ROHM_API int rohm_posenet_sample_step_clips(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* x0_out,
                                            float* x_next, const float* coef_row, const uint64_t* streams, uint64_t draw,
                                            uint64_t* offset_increments, int B, int T, void* stream);

/* Same as rohm_posenet_forward but with CUDA events recorded on `stream` around every kernel launch, always as the serial
 * layer chain on that one stream; synchronises the stream and returns, per category {0: tensor-core GEMM, 1: attention, 2: LayerNorm, 3: pack/unpack/time-token}, the
 * summed device milliseconds (host float[4]) and the number of launches (host int[4]).  For bench.py's roofline. */
ROHM_API int rohm_posenet_profile(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B, int T,
                         void* stream, float* ms_by_category, int* launches_by_category);

/* Options: 0 = replay the forward as a CUDA graph (default 1; the graph is captured on first use per (B, T) and its
 * three caller-memory pointers are patched per call); 1 = programmatic dependent launch on the GEMMs (default 1);
 * 2 = clip groups of uniform clips: 0 = chosen from B and T (default: two concurrent groups when the batch's QKV GEMM
 * has more tiles than the GPU has SMs), 1 = the serial layer chain, 2 = two groups whenever B >= 2 (for timing the two
 * against each other; the results are the same bits). */
ROHM_API int rohm_posenet_set_option(rohm_posenet* pn, int option, int value);

/* Kernel launches issued by the last forward outside rohm_posenet_profile (for bench.py's gpu_launches accounting). */
ROHM_API int rohm_posenet_launches_per_forward(const rohm_posenet* pn);

/* ------------------------------------------------------------------------------------------------------------
 * TrajNet denoiser + TrajControl branch (model/trajnet.py:10-75, 177-275; blocks model/heads.py:20-106)
 * ---------------------------------------------------------------------------------------------------------- */

/* Parameters are handed over by their reference state-dict key ("diff_enc1.blocks.0.block.0.weight",
 * "controlnet.control_zero_conv_0.bias", "time_mlp.1.weight", ...): `names[i]` (host strings), `ptrs[i]` (device fp32),
 * `numels[i]`.  Every key the architecture needs must be present with the reference's shape; extra keys (e.g. the
 * never-evaluated cond_downsample4.*) are ignored.  `frames` must be a multiple of 16, and a GroupNorm group of the widest
 * levels (frames x mid_dim / 64 values) must fit the shared memory of a cluster of 8 CTAs:
 * frames <= 8 x floor(M / (mid_dim / 16)), M = the device's opt-in shared memory per block less the GroupNorm kernel's
 * static shared memory -- about 58 000 frames at mid_dim 512 on an H100.  A longer clip is refused with ROHM_ERR_INVALID
 * before anything is allocated.  The library repacks all convolution weights into GEMM layout (TF32 hi/lo, tap-major K) and
 * owns its copies. */
ROHM_API int rohm_trajnet_create(rohm_ctx* ctx, int n_params, const char* const* names, const float* const* ptrs,
                                 const int64_t* numels, int time_dim, int cond_dim, int traj_feat_dim, int mid_dim,
                                 int trajcontrol, int control_cond_dim, int max_batch, int frames, int precision,
                                 rohm_trajnet** out);
/* rohm_trajnet_create for a batch-invariant engine (same arguments).  Every real frame of clip b is then a function of that
 * clip's inputs, its length, the weights and the precision only: not of B, `frames`, `max_batch`, the clip's position, the
 * engine serving it, the graph / PDL options or the GPU.  Each convolution's GEMM tile width and split-K ranges are chosen
 * for a fixed row count per level (64 x (144 + 32) / 2^L, so a 64-clip, 144-frame batch runs the default engine's plan and
 * bits), and each packed clip's GroupNorm statistics are reduced over the slices the clip has alone.  A clip as a one-clip
 * batch of its own length, without lengths, gives the same bits as inside any ragged batch. */
ROHM_API int rohm_trajnet_create_batch_invariant(rohm_ctx* ctx, int n_params, const char* const* names,
                                                 const float* const* ptrs, const int64_t* numels, int time_dim, int cond_dim,
                                                 int traj_feat_dim, int mid_dim, int trajcontrol, int control_cond_dim,
                                                 int max_batch, int frames, int precision, rohm_trajnet** out);
ROHM_API void rohm_trajnet_destroy(rohm_trajnet* tn);

/* Step-invariant part of TrajNet.forward: the condition pyramid cond_enc1..4 (trajnet.py:192-208) and, with
 * TrajControl, control_zero_conv_0(control_cond) (:51-52).  cond: [B, frames, cond_dim]; control_cond:
 * [B, frames, control_cond_dim] or NULL for the vanilla network.  Call whenever batch['cond'] / ['control_cond'] change. */
ROHM_API int rohm_trajnet_set_cond(rohm_trajnet* tn, const float* cond, const float* control_cond, int B, void* stream);

/* Per-clip lengths for the following set_cond, forward and sample_step calls: clip b of the padded [B, frames, *] tensors
 * has lengths_host[b] real frames, a multiple of 16 with 16 <= lengths_host[b] <= frames.  Inside, the clips are packed
 * with no padding rows past each clip's own 32 (so a batch of mixed lengths does no wasted tensor work).  Frames
 * [0, lengths[b]) of the output depend on that clip alone: bit-identical to the clip as a one-clip padded batch through
 * the same engine, and equal to the clip at its own length up to summation order (another engine may choose other
 * split-K ranges; in a batch-invariant engine, bit-identical to it).  Frames past it are zero, and the input values there are never read.  NULL returns to uniform clips.
 * Changing the lengths waits for the device to go idle; call set_cond again afterwards.  ROHM_ERR_INVALID for B outside
 * the created capacity or a bad length. */
ROHM_API int rohm_trajnet_set_lengths(rohm_trajnet* tn, const int* lengths_host, int B);

/* TrajNet.forward (trajnet.py:177-275).  x_t: [B, frames, traj_feat_dim]; time: int64 [B]; out: same shape as x_t. */
ROHM_API int rohm_trajnet_forward(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* out, int B,
                                  void* stream);
/* One whole ancestral step of the TrajNet sampler (gaussian_diffusion_trajnet.py:388-434, p_sample without cond_fn):
 * x0_out = TrajNet.forward(x_t, time), x_next = coef1 x0 + coef2 x_t + sigma z with z drawn inside the update kernel exactly as
 * torch.randn_like(x_t) would draw it from (seed, offset) -- forward and update are ONE graph launch.  Arguments as
 * rohm_posenet_sample_step (coef_row: device float[8] of the step). */
ROHM_API int rohm_trajnet_sample_step(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* x0_out, float* x_next,
                                      const float* coef_row, uint64_t seed, uint64_t offset, uint64_t* offset_increment, int B,
                                      void* stream);
/* rohm_trajnet_sample_step with per-clip noise streams over the engine's current lengths; arguments as
 * rohm_posenet_sample_step_clips. */
ROHM_API int rohm_trajnet_sample_step_clips(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* x0_out,
                                            float* x_next, const float* coef_row, const uint64_t* streams, uint64_t draw,
                                            uint64_t* offset_increments, int B, void* stream);
ROHM_API int rohm_trajnet_set_option(rohm_trajnet* tn, int option, int value); /* 0: CUDA-graph replay, 1: programmatic dependent launch (both default 1) */
ROHM_API int rohm_trajnet_launches_per_forward(const rohm_trajnet* tn);

/* ------------------------------------------------------------------------------------------------------------
 * SMPL-X body model: joints FK, skating guidance, full LBS
 * (third-party smplx==0.1.28 lbs.py / body_models.py as called from data_loaders/motion_representation.py:373-398,
 *  model/posenet.py:196-257; see DESIGN.md for provenance -- the body model is not part of the reference tree)
 * ---------------------------------------------------------------------------------------------------------- */

/* v_template [V,3], shapedirs [V,3,shape_comps] (first 10 components = betas), posedirs [486, V*3],
 * J_regressor [55,V], lbs_weights [V,55] (device fp32); parents_host: host int[55] (-1 for the root).
 * max_frames: capacity in frames (B*T) of the per-call workspace.  with_vertices = 0 skips the LBS data (joints and
 * guidance only; posedirs / lbs_weights may then be NULL). */
ROHM_API int rohm_body_create(rohm_ctx* ctx, const float* v_template, const float* shapedirs, int shape_comps,
                              const float* posedirs, const float* J_regressor, const float* lbs_weights,
                              const int* parents_host, int num_verts, int64_t max_frames, int with_vertices,
                              int precision, rohm_body** out);
ROHM_API void rohm_body_destroy(rohm_body* bd);
/* The skinning path rohm_body_forward takes for the vertices, chosen at rohm_body_create from the model's weights:
 *   0  fused: blend GEMM with the skinning in its epilogue, one launch (fp16 pairs, every 32-vertex tile touches <= 16 bones);
 *   1  sparse two-kernel: blend GEMM -> v_posed chunks -> skinning kernel (otherwise, every vertex has <= 8 bones);
 *   2  dense two-kernel: blend GEMM -> v_posed chunks -> dense skinning kernel (some vertex has > 8 bones);
 *  -1  the handle has no vertex support (or is NULL).
 * ROHM_B200_FUSED_LBS=0 and ROHM_B200_DENSE_SKIN=1 move a handle to a later path.  Introspection only. */
ROHM_API int rohm_body_skin_path(const rohm_body* bd);

/* Row pitch, in floats, of the `vertices` buffers handed to rohm_body_forward / rohm_body_from_repr from now on:
 * frame n's vertices start at vertices + n * pitch.  0 (the default) = dense [N, V, 3] as smplx returns them
 * (reference: body_model output `.vertices`, test_amass_full.py:392-428).  A pitch that is a multiple of 4 floats (>= 3 V;
 * 16-byte-aligned buffer) lets the fused launch write the vertices with TMA bulk stores instead of 4-byte stores (3 V =
 * 31425 floats is not 16-byte divisible); only valid when rohm_body_skin_path() is 0. */
ROHM_API int rohm_body_set_vertex_pitch(rohm_body* bd, int64_t pitch_floats);

/* SMPLX.forward with jaw / eyes / hands / expression = 0 (exactly how RoHM calls it): global_orient [N,3], body_pose
 * [N,63] axis-angle, betas [N,10], transl [N,3] -> joints [N, num_joints, 3] (first num_joints <= 55 posed joints +
 * transl; NULL to skip) and vertices [N, V, 3] (NULL to skip). */
ROHM_API int rohm_body_forward(rohm_body* bd, const float* global_orient, const float* body_pose, const float* betas,
                               const float* transl, int64_t N, float* joints, int num_joints, float* vertices,
                               void* stream);

/* Clips of different lengths inside padded tensors.  The entry points below that take `lengths` read the clips' frame
 * counts from device arrays: lengths (int[B], in the frame count of the tensor that call works on) and, where frames are
 * packed, clip_off (int[B+1], the exclusive prefix sum of lengths) with total_frames = clip_off[B] known to the host.  Packed
 * means frame t of clip b is row clip_off[b] + t.  Frames past a clip are never read, whatever they hold; where an output
 * keeps its padded shape its frames past a clip are written as zeros.  lengths = NULL means uniform clips of T frames; then
 * clip_off must be NULL and total_frames 0, anything else returns ROHM_ERR_INVALID. */

/* recover_from_repr_smpl(recover_mode='smplx_params') on a normalised representation x with the dataset's mean/std [294]:
 * denormalise, rot6d -> rotmat -> axis-angle (kornia route), then rohm_body_forward.  channels_last = 0 -> x is
 * [B,294,1,T] (PoseNet tensors); 1 -> x is [B,T,294] (the drivers' tensors, test_amass_full.py:279-293, 386-428).
 * Uniform clips: joints [B*T, num_joints, 3] and optionally vertices [B*T, V, 3].  With lengths (1 <= lengths[b] <= T):
 * the clips' own frames only, packed: joints [total_frames, num_joints, 3] and optionally vertices [total_frames, V, 3]; FK
 * and the blend GEMM + skinning run over total_frames rows, and total_frames (not B*T) is what has to fit the handle's
 * capacity.  Each frame equals the same frame of the uniform call bit for bit.  Vertices are pitched as rohm_body_forward's. */
ROHM_API int rohm_body_from_repr(rohm_body* bd, const float* x, int channels_last, const float* mean, const float* stdv,
                                 int B, int T, const int* lengths, const int* clip_off, int64_t total_frames, float* joints,
                                 int num_joints, float* vertices, void* stream);

/* PoseNet.guide_skating_with_smpl(compute_grad='x_0'): grad [B,294,1,T] = d(-(loss_smpl + loss_abs))/d x0 with the
 * channels [0,22) and the 4 contact channels zero.  Analytic VJP (no autograd); all-zero if nothing skates.
 * loss_out: optional device float[4] = {sum_abs, count_abs, sum_smpl, count_smpl}.  With lengths (1 <= lengths[b] <= T):
 * frames at or past lengths[b] add nothing to the sums or counts and get a zero gradient, a velocity pair (t, t + 1) counts
 * only when t + 1 < lengths[b], and their values are never used.  per_clip = 0: the normalisers are batch-wide over the
 * real frames (the reference on the whole batch).  per_clip = 1: clip b is normalised by its own counts, so its gradient
 * equals this call on clip b alone ([1,294,1,n_b], n_b = lengths[b] or T, per_clip = 0) bit for bit, and loss_out is
 * device float[B][4], the four sums per clip.  The counts are exact; the speed sums in loss_out depend on the order of
 * the device's additions and may differ in the last bits between calls. */
ROHM_API int rohm_skating_guidance(rohm_body* bd, const float* x0, const float* mean, const float* stdv, const int* lengths,
                                   int B, int T, int per_clip, float* grad, float* loss_out, void* stream);

/* rohm_skating_guidance in two halves, for clip-sharded runs that reproduce the reference's BATCH-GLOBAL normalisers
 * (posenet.py:230-233, 242-248): _sums computes this shard's {sum_abs, count_abs, sum_smpl, count_smpl} into sums_out (device
 * float[4]; per-frame state stays in the handle), the caller all-reduces the four floats over the ranks, _backward produces
 * this shard's gradient with the global sums.  _sums followed by _backward with the same sums == rohm_skating_guidance. */
ROHM_API int rohm_skating_guidance_sums(rohm_body* bd, const float* x0, const float* mean, const float* stdv, int B, int T,
                                        float* sums_out, void* stream);
ROHM_API int rohm_skating_guidance_backward(rohm_body* bd, const float* x0, const float* mean, const float* stdv, int B, int T,
                                            const float* sums, float* grad, void* stream);

/* PoseNet.guide_2d_projection_with_smpl(compute_grad='x_0') (model/posenet.py:260-317, utils/other_utils.py:150-185):
 * grad [B,294,1,T] = d(-loss_2d)/d x0, loss_2d = mean over (clip, frame, 10 selected joints, 2) of
 * |perspective_projection(camera <- scene <- canonical joints) - keypoints| * confidence; channels [0,22) and the 4 contact
 * channels zero.  cam_affine [B,12]: rows of the 3x4 map canonical -> camera coordinates per clip
 * (inv(cam_R) (inv(transf_matrix) p - cam_t)); focal, center [B,2]; keypoints_2d [B, kp_frames >= T, 22, 3] = (u, v, conf).
 * Analytic VJP through the 22-joint kinematic tree (no autograd).  per_clip = 0: the mean runs over the whole batch and
 * loss_out (optional) is device float[1], the un-normalised sum.  per_clip = 1: the mean of clip b runs over its own
 * n_b frames (n_b = lengths[b] or T), so its gradient equals this call on clip b alone ([1,294,1,n_b], per_clip = 0) bit for
 * bit, and loss_out is device float[B], the un-normalised sum per clip.  lengths (1 <= lengths[b] <= T) is accepted only
 * with per_clip = 1, else ROHM_ERR_INVALID: x0 and keypoints_2d are not read at or past lengths[b] and the gradient there
 * is zero. */
ROHM_API int rohm_projection_guidance(rohm_body* bd, const float* x0, const float* mean, const float* stdv,
                                      const int* lengths, int B, int T, int per_clip, const float* cam_affine,
                                      const float* focal, const float* center, const float* keypoints_2d, int kp_frames,
                                      float* grad, float* loss_out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Either side of the sampling loops: the drivers' inter-round glue and representation recovery, on the device
 * ---------------------------------------------------------------------------------------------------------- */

/* test_amass_full.py:268-311 (per-clip host loop in the reference): TrajNet output traj_out [B,T,traj_dim] (z-scored,
 * traj_dim = 13 for repr_abs_only else <= 22) is scattered into repr_clean [B,T,294] -> composite_out [B,T,294]
 * (z-scored with the trajectory dataset's mean/std) -> SMPL-X joints (rot6d -> axis-angle -> FK) -> get_repr_smplx
 * (data_loaders/motion_representation.py:187-282: forward direction, root quaternion incl. the first-NaN repair, velocities,
 * global-orient 6-D / angular velocity, translation) -> traj_full_out [B,T-1,22], z-scored with the pose dataset's stats.
 * 2 <= T <= 8192 (one cluster of at most 8 CTAs of 1024 frames per clip).  With lengths (2 <= lengths[b] <= T trajectory
 * frames): composite_out and traj_full_out keep their padded shapes, rows lengths[b] .. T-1 (composite) and
 * lengths[b]-1 .. T-2 (traj_full) are zeros.  FK runs over the total_frames packed frames; the first-NaN search and repair of
 * the root quaternion and the velocity pairs stay inside the clip (the repair of frame 0 takes frame lengths[b]-1).  A
 * clip's rows equal the uniform call on the clip alone with T = lengths[b], bit for bit. */
ROHM_API int rohm_traj_glue(rohm_body* bd, const float* traj_out, int traj_dim, const float* repr_clean,
                            const float* traj_mean, const float* traj_std, const float* pose_mean, const float* pose_std,
                            int B, int T, const int* lengths, const int* clip_off, int64_t total_frames,
                            float* composite_out, float* traj_full_out, void* stream);

/* The last stage of rohm_traj_glue on its own: get_repr_smplx's trajectory block (motion_representation.py:187-282) from
 * joints [B,T,22,3], global-orient axis-angles [B*T,3] and translations [B*T,3] -> traj_full_out [B,T-1,22], z-scored with
 * mean/stdv (the first 22 entries are read).  2 <= T <= 8192, as rohm_traj_glue.  With lengths (2 <= lengths[b] <= T):
 * joints [total_frames,22,3] and global_orient_aa / transl [total_frames,3] hold the clips packed, and traj_full_out keeps
 * its padded shape with zeros from row lengths[b]-1. */
ROHM_API int rohm_traj_repr_from_joints(rohm_ctx* ctx, const float* joints, const float* global_orient_aa,
                                        const float* transl, const float* mean, const float* stdv, int B, int T,
                                        const int* lengths, const int* clip_off, float* traj_full_out, void* stream);

/* test_amass_full.py:256-258: control_cond [B,T,cond_feats] from the PoseNet output pose_out [B,traj_feats+cond_feats,1,Tp]
 * (frames [0,Tp) copied, frames [Tp,T) repeat frame Tp-1).  With lengths (1 <= lengths[b] <= Tp pose frames, and then
 * T > Tp): control frames [0, lengths[b]) are the clip's pose frames, frame lengths[b] repeats the clip's own last pose
 * frame, later frames are zeros. */
ROHM_API int rohm_pose_to_control_cond(rohm_ctx* ctx, const float* pose_out, int B, int Tp, int T, int traj_feats,
                                       int cond_feats, const int* lengths, float* control_cond, void* stream);

/* test_amass_full.py:320-370: PoseNet condition cond_out [B,294,1,Tp] = src (channel-major [B,294,1,src_T] or channels-last
 * [B,src_T,294]) with channels [0,22) replaced by traj_full [B,Tp,22] (NULL keeps src) and channels >= 22 zeroed where
 * chan_keep[c] == 0 (294 bytes, NULL = keep all: the 'lower' / 'upper' joint masks), where frame_lo[b] <= t < frame_hi[b]
 * (int [B], NULL = none: the 'full' scheme) and, with zero_contact, in the 4 contact channels.  With lengths
 * (1 <= lengths[b] <= Tp): frames past a clip are zeros in every channel.  With vis_mask (test_prox_egobody.py:302-309,
 * channels-last [B,vis_T,294] with vis_T >= Tp, frames [0,Tp) read; NULL = none; not with lengths): after the occlusion
 * zeroing every channel of frame t is multiplied by vis_mask[b,t,c] (IEEE products: -x*0 = -0, NaN*1 = NaN, Inf*0 = NaN),
 * and the contact zeroing comes after the multiply. */
ROHM_API int rohm_build_pose_cond(rohm_ctx* ctx, const float* src, int src_channel_major, int src_T, const float* traj_full,
                                  const unsigned char* chan_keep, const int* frame_lo, const int* frame_hi,
                                  int zero_contact, int B, int Tp, const int* lengths, const float* vis_mask, int vis_T,
                                  float* cond_out, void* stream);

/* rot6d_to_rotmat (quaternion.py:482-501) and rotation_matrix_to_angle_axis (konia_transform.py:317-340 -> :350-444 ->
 * :561-631) on n 6-D rotations: aa [n,3] and/or rotmat [n,9] (row-major), either may be NULL. */
ROHM_API int rohm_rot6d_to_aa(rohm_ctx* ctx, const float* rot6d, int64_t n, float* aa, float* rotmat, void* stream);

/* recover_from_repr_smpl(recover_mode='joint_abs_traj' | 'joint_rel_traj') (motion_representation.py:285-371) on a z-scored
 * representation in either layout -> joints [B,T,22,3].  With lengths (1 <= lengths[b] <= T): packed joints
 * [total_frames,22,3] of the clips' own frames.  The absolute mode then has no dependence between frames and runs one thread
 * per packed frame; the relative mode keeps one thread per clip and stops at lengths[b]. */
ROHM_API int rohm_joints_from_traj(rohm_ctx* ctx, const float* x, int channels_last, const float* mean, const float* stdv,
                                   int B, int T, const int* lengths, const int* clip_off, int64_t total_frames,
                                   int relative, float* joints, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Sliding windows over whole recordings (dataloader_video.py:160-183, dataloader_amass.py:105-131 and :319-341)
 * ---------------------------------------------------------------------------------------------------------- */

/* R recordings packed frame after frame (recording r holds rows rec_off[r] .. rec_off[r+1]-1 of global_orient [.,3],
 * transl [.,3], betas [.,10], body_pose [.,63] axis-angle and the 22-joint world positions joints [.,22,3], z up) ->
 * windows of clip_len frames (3..160) with stride clip_len - overlap (overlap 0..2): window k of a recording starts at
 * k * (clip_len - overlap) and is cut while it ends inside the recording, so a recording shorter than clip_len gives none.
 * rec_off_host (host) and rec_off (device) hold the same R + 1 offsets.  *n_windows (host) receives the window count W; if
 * W > max_windows nothing is launched and ROHM_ERR_INVALID is returned.  Outputs, W rows each: win_rec / win_start (int32:
 * recording and first frame), transf [W,4,4] (cano_seq_smplx's transf_matrix, world -> canonical), repr_traj / repr_pose
 * [W, clip_len-1, 294]: get_repr_smplx of the canonical window (motion_representation.py:47-110, :187-282;
 * update_globalRT_for_smplx with delta_T = pelvis - transl) z-scored with traj_mean / traj_std and pose_mean / pose_std
 * [294].  Frames outside every window are never read. */
ROHM_API int rohm_window_encode(rohm_ctx* ctx, const float* global_orient, const float* transl, const float* betas,
                                const float* body_pose, const float* joints, const int* rec_off_host, const int* rec_off,
                                int R, int clip_len, int overlap, const float* traj_mean, const float* traj_std,
                                const float* pose_mean, const float* pose_std, int max_windows, int* n_windows,
                                int* win_rec, int* win_start, float* transf, float* repr_traj, float* repr_pose,
                                void* stream);

/* Input noise on the windows' canonical SMPL-X parameters (dataloader_amass.py:156-192, input_noise with sep_noise False).
 * global_orient .. joints, rec_off (device int[R+1]), win_rec / win_start and transf [W,4,4] are the inputs and outputs of
 * the rohm_window_encode call that cut these W windows of clip_len frames.  Noise, window-major like the reference's
 * preset-noise pickle: noise_transl [W,clip_len,3] (metres), noise_betas [W,clip_len,10], noise_global_orient
 * [W,clip_len,3] and noise_body_pose [W,clip_len,21,3] (degrees, added to scipy's extrinsic 'zxy' Euler angles of each
 * canonical rotation; the round trip rotvec -> angles -> + n -> rotvec runs in float64 and follows scipy's gimbal-lock
 * rule).  Output noisy_params [W*clip_len, 79]: rows of global_orient 3 | transl 3 | betas 10 | body_pose 63, float32
 * axis-angle, window-major (row w * clip_len + t). */
ROHM_API int rohm_window_param_noise(rohm_ctx* ctx, const float* global_orient, const float* transl, const float* betas,
                                     const float* body_pose, const float* joints, const int* rec_off, const int* win_rec,
                                     const int* win_start, const float* transf, int W, int clip_len,
                                     const float* noise_transl, const float* noise_betas, const float* noise_global_orient,
                                     const float* noise_body_pose, float* noisy_params, void* stream);

/* rohm_window_encode on windows that are already canonical (the noisy windows, which the reference does not
 * re-canonicalise): params [W*clip_len, 79] as rohm_window_param_noise writes them and joints [W*clip_len,22,3], both
 * window-major -> repr_traj / repr_pose [W, clip_len-1, 294], get_repr_smplx of each window z-scored with traj_mean /
 * traj_std and pose_mean / pose_std, computed by the same row code as rohm_window_encode. */
ROHM_API int rohm_window_encode_canonical(rohm_ctx* ctx, const float* params, const float* joints, int W, int clip_len,
                                          const float* traj_mean, const float* traj_std, const float* pose_mean,
                                          const float* pose_std, float* repr_traj, float* repr_pose, void* stream);

/* The inverse: joints [W*(clip_len-2),22,3] (each window's clip_len-2 pose frames in its canonical frame, as
 * reconstruct_outputs returns them) -> world [total_frames,22,3] packed by recording (rec_off, device int[R+1]), pose frame t
 * of window w at row rec_off[win_rec[w]] + win_start[w] + t, mapped by the inverse of transf[w] (eval_prox_egobody.py:177-182).
 * covered [total_frames] (bytes) is 1 on those rows; every other row of both outputs is 0. */
ROHM_API int rohm_window_to_world(rohm_ctx* ctx, const float* joints, const int* win_rec, const int* win_start,
                                  const float* transf, int W, int clip_len, const int* rec_off, int64_t total_frames,
                                  float* world, unsigned char* covered, void* stream);

/* The video loader's windows (dataloader_video.py, DataloaderVideo for PROX and EgoBody): the recordings' per-frame
 * SMPL-X fits and their FK joints are in each recording's camera frame; cam [R,12] holds rows of [A | b], the camera ->
 * z-up scene map (PROX: cam2world; EgoBody, whose scene is y-up: Q cam2world with Q = Rx(+90 deg), (x, y, z) -> (x, -z,
 * y), which turns cano_seq_smplx_egobody into cano_seq_smplx, DESIGN §4.14), and y_up = 1 for EgoBody.  floor [R]: a preset
 * floor height per recording, 0 for the window minimum (the reference's `if preset_floor_height:`).  Windows are cut as
 * rohm_window_encode cuts them, and repr_traj / repr_pose are computed by its row code.  transf [W,4,4] is the
 * reference's scene -> canonical transf_matrix (T_z Q for y_up).  Further outputs per window frame, including the last,
 * window-major: cano_joints and scene_joints [W*clip_len,22,3] (canonical; scene frame, y up for y_up) and cano_params
 * [W*clip_len,79] (the canonical SMPL-X parameters, rows as rohm_window_param_noise writes them). */
ROHM_API int rohm_window_encode_video(rohm_ctx* ctx, const float* global_orient, const float* transl, const float* betas,
                                      const float* body_pose, const float* joints, const int* rec_off_host,
                                      const int* rec_off, int R, int clip_len, int overlap, const float* cam,
                                      const float* floor, int y_up, const float* traj_mean, const float* traj_std,
                                      const float* pose_mean, const float* pose_std, int max_windows, int* n_windows,
                                      int* win_rec, int* win_start, float* transf, float* repr_traj, float* repr_pose,
                                      float* cano_joints, float* scene_joints, float* cano_params, void* stream);

/* The video loader's 2-D inputs of W windows (dataloader_video.py:441-484): keypoints25 [N,25,3] (OpenPose BODY_25 x, y,
 * confidence per packed recording frame, zeros where no person was found) and depth_mask [N,25] (mask_joint.npy, SMPL-X
 * joint order).  conf64 [R] (bytes, device): 1 where the recording's keypoint array is float64 in the loader (some frame
 * had no person), so that conf > 0.2 and PROX's flip are evaluated in float64; 0 for float32.  undistort = 1 (PROX):
 * x -> 1919 - x, cv2.undistortPoints with P = camera_mtx (camera_mtx [R,3,3] and dist [R,14], zero-padded distortion,
 * float64; 5 fixed iterations), flipped back.  Outputs, window-major: keypoints [W*clip_len,22,3] (SMPL topology),
 * mask_joint_vis [W*clip_len,22] and mask_vec_vis [W*clip_len,294]. */
ROHM_API int rohm_window_keypoints(rohm_ctx* ctx, const float* keypoints25, const float* depth_mask,
                                   const unsigned char* conf64, const double* camera_mtx, const double* dist,
                                   int undistort, const int* rec_off, const int* win_rec, const int* win_start, int W,
                                   int clip_len, float* keypoints, float* mask_joint_vis, float* mask_vec_vis,
                                   void* stream);

/* joints [N,22,3] (packed recording frames) mapped by their recording's cam [R,12] (rows of [A | b]) and gathered into
 * the W windows' frames: out [W*clip_len,22,3] (EgoBody's ground-truth joints in the scene frame, dataloader_video.py
 * :312-314). */
ROHM_API int rohm_window_scene_joints(rohm_ctx* ctx, const float* joints, const float* cam, const int* rec_off,
                                      const int* win_rec, const int* win_start, int W, int clip_len, float* out,
                                      void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Evaluation metrics (eval_amass_full.py:71-147, eval_prox_egobody.py:172-272), rohm_b200/metrics.py
 * ------------------------------------------------------------------------------------------------------------ */

/* B clips packed frame after frame: clip b is rows [frame_off[b], frame_off[b+1]) (device int64 [B+1]) of gt / rec
 * [N,22,3] (rec_ric_data_clean / rec_ric_data_rec_from_smpl) and of repr_clean / repr_rec [N,repr_width] (the contact
 * labels are the last 4 channels).  A (frame, joint) is occluded when bit j of occ_joints is set and occ_lo <= t < occ_hi
 * (clamped to the clip).  Per clip: h0 [B] (the NaN-propagating minimum z of gt).  Per packed row: mpjpe [N,22], accerr
 * [N,22] (rows t >= T-2 of a clip are 0), skate_gt / skate_rec [N] (row T-1 is 0), contact [N,4] matches, pene_freq [N,2]
 * and pene_dist [N,2] (toes 10, 11).  sums [B,5] float64 (mpjpe, visible, occluded, accel error, pene dist) and counts
 * [B,11] int64 (mpjpe n, visible n, occluded n, contact matches, contact n, skating gt, skating rec, skating n, accel n,
 * pene freq, pene n), each in a fixed order. */
ROHM_API int rohm_eval_amass(rohm_ctx* ctx, const float* gt, const float* rec, const float* repr_clean,
                             const float* repr_rec, int repr_width, const int64_t* frame_off, int B, unsigned occ_joints,
                             int occ_lo, int occ_hi, float* h0, float* mpjpe, float* accerr, unsigned char* skate_gt,
                             unsigned char* skate_rec, unsigned char* contact, unsigned char* pene_freq,
                             float* pene_dist, double* sums, int64_t* counts, void* stream);

/* W video windows of T frames: rec [W,T,22,3] canonical joints, mapped to the scene by the float64 inverse of transf
 * [W,4,4] rounded to float32; floor [R] per recording (win_rec [W] device int32); y_up = 1 for EgoBody (height y,
 * horizontal xz), 0 for PROX (z; xy).  Optional ground truth gt [W,gt_frames,22,3] and visibility mask_vis
 * [W,mask_frames,22] (first T frames used; the mask needs gt); without gt, accerr / gmpjpe / mpjpe may be NULL.  Outputs:
 * skate [W,T-1], acc and accerr [W,T-2] (per frame, the mean over joints), gmpjpe and mpjpe [W,T,22], pene_freq and
 * pene_dist [W,T]; sums [W,10] float64 (acc, acc error, gmpjpe, mpjpe, vis num, vis den, occ num, occ den, pene freq,
 * pene dist) and counts [W,1] int64 (skating frames). */
ROHM_API int rohm_eval_video(rohm_ctx* ctx, const float* rec, int T, const float* transf, const float* gt, int gt_frames,
                             const float* mask_vis, int mask_frames, const int* win_rec, const float* floor, int W,
                             int y_up, unsigned char* skate, float* acc, float* accerr, float* gmpjpe, float* mpjpe,
                             float* pene_freq, float* pene_dist, double* sums, int64_t* counts, void* stream);

/* Group sums of per-item rows sums [n,ks] / counts [n,kc]: group g sums items order[group_off[g] .. group_off[g+1]) in
 * that order (device int32), row n_groups of out_sums [n_groups+1,ks] / out_counts [n_groups+1,kc] sums the groups in
 * order. */
ROHM_API int rohm_eval_reduce(rohm_ctx* ctx, const double* sums, int ks, const int64_t* counts, int kc, const int* order,
                              const int* group_off, int n_groups, double* out_sums, int64_t* out_counts, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ROHM_B200_H_ */
