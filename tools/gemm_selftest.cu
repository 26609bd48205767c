// Standalone numerics + timing check of the wgmma 3xTF32 GEMM (rohm_b200/csrc/gemm.cu) against a CPU fp64
// reference.  Build:  make -C tools   Run on an H100:  tools/gemm_selftest
// Cases: plain linear layers (PoseNet shapes), ragged K/N tails, multi-segment shifted reads (Conv1d k=5 over a
// padded-clip layout), stride-2 reads (Downsample1d), GroupNorm statistics, hi/lo split outputs.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "../rohm_b200/csrc/gemm.cuh"

using namespace rohm;

#define CK(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e_ = (x);                                                                       \
    if (e_ != cudaSuccess) {                                                                    \
      printf("CUDA error %s at %s:%d: %s\n", cudaGetErrorName(e_), __FILE__, __LINE__, #x);     \
      exit(2);                                                                                  \
    }                                                                                           \
  } while (0)

static std::mt19937 rng(1234);
static void fill(std::vector<float>& v, float scale = 1.0f) {
  std::normal_distribution<float> d(0.0f, scale);
  for (auto& x : v) x = d(rng);
}
template <class T>
static T* dev(const std::vector<T>& h) {
  T* d;
  CK(cudaMalloc(&d, h.size() * sizeof(T)));
  CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}
static float* dev_zero(size_t n) {
  float* d;
  CK(cudaMalloc(&d, n * sizeof(float)));
  CK(cudaMemset(d, 0, n * sizeof(float)));
  return d;
}
static std::vector<float> host(const float* d, size_t n) {
  std::vector<float> h(n);
  CK(cudaMemcpy(h.data(), d, n * sizeof(float), cudaMemcpyDeviceToHost));
  return h;
}
struct Split {
  float *hi, *lo;
};
static Split split(const float* d, size_t n) {
  Split s;
  s.hi = dev_zero(n);
  s.lo = dev_zero(n);
  CK(launch_split_tf32(d, s.hi, s.lo, (int64_t)n, 0));
  return s;
}

static int failures = 0;
static void report(const char* name, double maxerr, double maxref, double tol) {
  const bool ok = maxerr <= tol && std::isfinite(maxerr);
  printf("%-44s max_abs_err %.3e (max |ref| %.3e) tol %.1e  %s\n", name, maxerr, maxref, tol, ok ? "OK" : "FAIL");
  if (!ok) ++failures;
}

// ------------------------------------------------------------------------------------------------
// Case 1: plain linear  C = act(A W^T + b) + R
// ------------------------------------------------------------------------------------------------
static void case_linear(int M, int N, int K, int block_n, int act, bool with_res, bool timing) {
  const int ldk = (K + 3) / 4 * 4;            // 16-byte row pitch
  const int Kp = (K + 31) / 32 * 32;          // weights are stored K-padded to the 32-wide k-block
  const int Np = (N + block_n - 1) / block_n * block_n;
  std::vector<float> A((size_t)M * ldk, 0.f), W((size_t)Np * Kp, 0.f), b(N), R((size_t)M * N);
  {
    std::normal_distribution<float> d(0.f, 1.f);
    for (int m = 0; m < M; ++m)
      for (int k = 0; k < K; ++k) A[(size_t)m * ldk + k] = d(rng);
    const float ws = 1.0f / std::sqrt((float)K);
    for (int n = 0; n < N; ++n)
      for (int k = 0; k < K; ++k) W[(size_t)n * Kp + k] = d(rng) * ws;
  }
  fill(b);
  fill(R);
  float *dA = dev(A), *dW = dev(W), *db = dev(b), *dR = dev(R);
  Split sA = split(dA, A.size()), sW = split(dW, W.size());
  float* dC = dev_zero((size_t)M * N);
  float* dCh = dev_zero((size_t)M * N);
  float* dCl = dev_zero((size_t)M * N);

  for (int passes : {3, 1}) {
    GemmParams p{};
    if (make_tmap_2d(&p.a_hi[0], sA.hi, M, K, ldk, kGemmBlockM) || make_tmap_2d(&p.a_lo[0], sA.lo, M, K, ldk, kGemmBlockM) ||
        make_tmap_2d(&p.b_hi, sW.hi, Np, Kp, Kp, block_n) || make_tmap_2d(&p.b_lo, sW.lo, Np, Kp, Kp, block_n)) {
      printf("tensor map encode failed\n");
      exit(2);
    }
    p.num_segs = 1;
    p.seg_kblocks[0] = Kp / kGemmBlockK;
    p.seg_row_shift[0] = 0;
    p.seg_row_mul[0] = 1;
    p.bias = db;
    p.residual = with_res ? dR : nullptr;
    p.ldr = N;
    p.out = dC, p.ldo = N;
    p.out_hi = dCh, p.out_lo = dCl, p.lds = N;
    p.act = act;
    p.M = M, p.N = N;
    p.out_row_mul = 1, p.out_row_add = 0;
    CK(cudaMemset(dC, 0, (size_t)M * N * 4));
    CK(launch_gemm(p, M, N, block_n, passes, 0));
    CK(cudaDeviceSynchronize());
    auto C = host(dC, (size_t)M * N);
    auto Ch = host(dCh, (size_t)M * N);
    auto Cl = host(dCl, (size_t)M * N);
    double maxerr = 0, maxref = 0, maxsplit = 0;
    // check a subset of rows to keep the CPU side quick
    const int step = M > 600 ? 7 : 1;
    for (int m = 0; m < M; m += step)
      for (int n = 0; n < N; ++n) {
        double acc = 0;
        for (int k = 0; k < K; ++k) acc += (double)A[(size_t)m * ldk + k] * (double)W[(size_t)n * Kp + k];
        acc += b[n];
        if (act == kActGelu) acc = 0.5 * acc * (1.0 + std::erf(acc / std::sqrt(2.0)));
        if (act == kActSilu) acc = acc / (1.0 + std::exp(-acc));
        if (act == kActMish) acc = acc * std::tanh(std::log1p(std::exp(acc)));
        if (with_res) acc += R[(size_t)m * N + n];
        const double got = C[(size_t)m * N + n];
        maxerr = std::fmax(maxerr, std::fabs(got - acc));
        maxref = std::fmax(maxref, std::fabs(acc));
        maxsplit = std::fmax(maxsplit, std::fabs((double)Ch[(size_t)m * N + n] + (double)Cl[(size_t)m * N + n] - got));
      }
    char name[128];
    snprintf(name, sizeof name, "linear M%d N%d K%d bn%d act%d passes%d", M, N, K, block_n, act, passes);
    report(name, maxerr, maxref, passes == 3 ? 2e-5 : 2e-2);
    snprintf(name, sizeof name, "  hi+lo == out (split epilogue)");
    report(name, maxsplit, maxref, 1e-5);

    if (timing) {
      cudaEvent_t e0, e1;
      CK(cudaEventCreate(&e0));
      CK(cudaEventCreate(&e1));
      for (int i = 0; i < 5; ++i) CK(launch_gemm(p, M, N, block_n, passes, 0));
      CK(cudaEventRecord(e0));
      const int iters = 50;
      for (int i = 0; i < iters; ++i) CK(launch_gemm(p, M, N, block_n, passes, 0));
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      const double us = ms * 1000.0 / iters;
      const double flops = 2.0 * M * N * K;
      printf("    timing: %.2f us/launch  -> %.1f TFLOP/s algorithmic (x%d tensor passes)\n", us, flops / us * 1e-6, passes);
    }
  }
  cudaFree(dA), cudaFree(dW), cudaFree(db), cudaFree(dR), cudaFree(dC), cudaFree(dCh), cudaFree(dCl);
  cudaFree(sA.hi), cudaFree(sA.lo), cudaFree(sW.hi), cudaFree(sW.lo);
}



// CTA 0's two timelines of the lean variants (EPI 0 / 1 / 3; gemm.cu debug_ts slots), first four tiles: MMA warpgroups --
// tile i published in acc_s; epilogue warpgroup -- prologue of tile i done (ready), acc_full observed (start), tile i stored (done).  ns since
// kernel start.
static void print_role_timeline(const unsigned long long* h) {
  printf("      MMA: first_full %llu | tile published:", h[3] - h[0]);
  for (int i = 16; i < 20 && h[i] != 0; ++i) printf(" %llu", h[i] - h[0]);
  printf("\n      EPI: ready/start/done per tile:");
  for (int i = 0; i < 4 && h[28 + i] != 0; ++i) printf(" %llu/%llu/%llu", h[20 + i] - h[0], h[24 + i] - h[0], h[28 + i] - h[0]);
  printf(" | end %llu\n", h[7] - h[0]);
}

// ------------------------------------------------------------------------------------------------
// Case 1b: the same linear layer on fp16 hi/lo pairs (kKindF16): A split as is, W scaled by a power of two into the
// middle of the fp16 range, accumulator scaled back in the epilogue.  a_scale stresses the fp16 range of the activations.
// ------------------------------------------------------------------------------------------------
#include <cuda_fp16.h>
static bool g_multicast = false;  // A-operand multicast across CTA pairs (gemm_enable_multicast) in the fp16 cases below
static void case_linear_f16(int M, int N, int K, int block_n, int act, bool with_res, bool timing, float a_scale,
                            int tma_mode = 0) {
  const int BK = gemm_block_k(kKindF16);
  const int ldk = (K + 7) / 8 * 8;  // 16-byte row pitch in halves
  const int Kp = (K + BK - 1) / BK * BK;
  const int Np = (N + block_n - 1) / block_n * block_n;
  std::vector<float> A((size_t)M * ldk, 0.f), W((size_t)Np * Kp, 0.f), b(N), R((size_t)M * N);
  float wmax = 0.f;
  {
    std::normal_distribution<float> d(0.f, 1.f);
    for (int m = 0; m < M; ++m)
      for (int k = 0; k < K; ++k) A[(size_t)m * ldk + k] = d(rng) * a_scale;
    const float ws = 1.0f / std::sqrt((float)K);
    for (int n = 0; n < N; ++n)
      for (int k = 0; k < K; ++k) wmax = std::fmax(wmax, std::fabs(W[(size_t)n * Kp + k] = d(rng) * ws));
  }
  fill(b);
  fill(R);
  int e2;
  std::frexp(wmax, &e2);                       // wmax = f * 2^e2, f in [0.5, 1)
  const float w_scale = std::ldexp(1.0f, 14 - e2);  // scaled max in [2^13, 2^14)
  float *dA = dev(A), *dW = dev(W), *db = dev(b), *dR = dev(R);
  __half *Ah, *Al, *Wh, *Wl, *dCh, *dCl;
  CK(cudaMalloc(&Ah, A.size() * 2));
  CK(cudaMalloc(&Al, A.size() * 2));
  CK(cudaMalloc(&Wh, W.size() * 2));
  CK(cudaMalloc(&Wl, W.size() * 2));
  CK(cudaMalloc(&dCh, (size_t)M * N * 2));
  CK(cudaMalloc(&dCl, (size_t)M * N * 2));
  CK(launch_split_f16(dA, Ah, Al, (int64_t)A.size(), 1.0f, 0));
  CK(launch_split_f16(dW, Wh, Wl, (int64_t)W.size(), w_scale, 0));
  float* dC = dev_zero((size_t)M * N);
  GemmParams p{};
  if (make_tmap_2d(&p.a_hi[0], Ah, M, K, ldk, kGemmBlockM, 1, kKindF16) || make_tmap_2d(&p.a_lo[0], Al, M, K, ldk, kGemmBlockM, 1, kKindF16) ||
      make_tmap_2d(&p.b_hi, Wh, Np, Kp, Kp, block_n, 1, kKindF16) || make_tmap_2d(&p.b_lo, Wl, Np, Kp, Kp, block_n, 1, kKindF16)) {
    printf("tensor map encode failed (f16)\n");
    exit(2);
  }
  p.num_segs = 1, p.seg_kblocks[0] = Kp / BK, p.seg_row_mul[0] = 1;
  p.bias = db, p.residual = with_res ? dR : nullptr, p.ldr = N;
  p.out = dC, p.ldo = N;
  const bool split_out = (N % 4) == 0;
  if (split_out) p.out_hi = dCh, p.out_lo = dCl, p.lds = N;
  p.act = act, p.M = M, p.N = N, p.out_row_mul = 1;
  p.acc_scale = 1.0f / w_scale;
  if (tma_mode == 1) p.out_hi = nullptr, p.out_lo = nullptr;  // fp32 out through the TMA-store epilogue
  if (tma_mode == 2) p.out = nullptr;                           // fp16 pair through the TMA-store epilogue
  if (tma_mode != 0) {
    if (gemm_enable_tma_store(&p, M, kKindF16) != 0 || !p.tma_store) {
      printf("gemm_enable_tma_store refused an eligible launch\n");
      exit(2);
    }
  }
  if (g_multicast && gemm_enable_multicast(&p, Ah, Al, M, K, ldk, N, block_n, kKindF16) != 0) {
    printf("gemm_enable_multicast failed\n");
    exit(2);
  }
  CK(cudaMemset(dCh, 0, (size_t)M * N * 2));
  CK(cudaMemset(dCl, 0, (size_t)M * N * 2));
  CK(launch_gemm(p, M, N, block_n, 3, 0, false, kKindF16));
  CK(cudaDeviceSynchronize());
  auto C = host(dC, (size_t)M * N);
  std::vector<__half> Ch((size_t)M * N), Cl((size_t)M * N);
  CK(cudaMemcpy(Ch.data(), dCh, Ch.size() * 2, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(Cl.data(), dCl, Cl.size() * 2, cudaMemcpyDeviceToHost));
  double maxerr = 0, maxref = 0, maxsplit = 0;
  const int step = M > 600 ? 7 : 1;
  for (int m = 0; m < M; m += step)
    for (int n = 0; n < N; ++n) {
      double acc = 0;
      for (int k = 0; k < K; ++k) acc += (double)A[(size_t)m * ldk + k] * (double)W[(size_t)n * Kp + k];
      acc += b[n];
      if (act == kActGelu) acc = 0.5 * acc * (1.0 + std::erf(acc / std::sqrt(2.0)));
      if (act == kActSilu) acc = acc / (1.0 + std::exp(-acc));
      if (with_res) acc += R[(size_t)m * N + n];
      const double pair = (double)__half2float(Ch[(size_t)m * N + n]) + (double)__half2float(Cl[(size_t)m * N + n]);
      const double got = tma_mode == 2 ? pair : C[(size_t)m * N + n];
      maxerr = std::fmax(maxerr, std::fabs(got - acc));
      maxref = std::fmax(maxref, std::fabs(acc));
      if (split_out && tma_mode == 0) maxsplit = std::fmax(maxsplit, std::fabs(pair - got));
    }
  char name[160];
  snprintf(name, sizeof name, "f16x2 linear M%d N%d K%d bn%d act%d a_scale %g%s%s", M, N, K, block_n, act, a_scale,
           tma_mode == 1 ? " [TMA store fp32]" : tma_mode == 2 ? " [TMA store fp16 pair]" : "", p.multicast_a ? " [A multicast]" : "");
  report(name, maxerr, maxref, (tma_mode == 2 ? 2.5e-5 : 2e-5) * std::fmax(1.0f, a_scale));
  if (tma_mode == 0) report("  hi+lo == out (fp16 split epilogue)", maxsplit, maxref, 4e-6 * std::fmax(1.0, maxref));
  if (timing) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int i = 0; i < 5; ++i) CK(launch_gemm(p, M, N, block_n, 3, 0, false, kKindF16));
    CK(cudaEventRecord(e0));
    const int iters = 50;
    for (int i = 0; i < iters; ++i) CK(launch_gemm(p, M, N, block_n, 3, 0, false, kKindF16));
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    const double us = ms * 1000.0 / iters;
    printf("    timing: %.2f us/launch  -> %.1f TFLOP/s algorithmic (fp16 hi/lo, 3 tensor passes)\n", us, 2.0 * M * N * K / us * 1e-6);
    unsigned long long* dts;
    CK(cudaMalloc(&dts, 32 * sizeof(unsigned long long)));
    // flags 1 / 2: developer experiments that break the result (epilogue drains the accumulator only / stages without storing) -- they
    // show how much of the main loop's steady-state slowdown comes from the concurrent epilogue of the previous tile
    for (int flags = 0; flags < (tma_mode == 2 && N >= 1024 ? 3 : 1); ++flags) {
      p.debug_flags = flags;
      p.debug_ts = nullptr;
      for (int i = 0; i < 3; ++i) CK(launch_gemm(p, M, N, block_n, 3, 0, false, kKindF16));
      CK(cudaEventRecord(e0));
      for (int i = 0; i < iters; ++i) CK(launch_gemm(p, M, N, block_n, 3, 0, false, kKindF16));
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaEventElapsedTime(&ms, e0, e1));
      CK(cudaMemset(dts, 0, 32 * sizeof(unsigned long long)));
      p.debug_ts = dts;
      CK(launch_gemm(p, M, N, block_n, 3, 0, false, kKindF16));
      CK(launch_gemm(p, M, N, block_n, 3, 0, false, kKindF16));
      CK(cudaDeviceSynchronize());
      unsigned long long h[32];
      CK(cudaMemcpy(h, dts, sizeof h, cudaMemcpyDeviceToHost));
      printf("    [debug_flags %d: %.2f us/launch] CTA0 timeline (ns): setup %llu | first_tma %llu | tile0 epi start %llu | tile0 epi done %llu | "
             "all tiles published %llu | last epi done %llu | stores done %llu\n",
             flags, ms * 1000.0 / iters, h[1] - h[0], h[2] - h[0], h[5] - h[0], h[6] - h[0], h[12] - h[0], h[13] - h[0], h[14] - h[0]);
      print_role_timeline(h);
    }
    p.debug_flags = 0;
    p.debug_ts = nullptr;
    cudaFree(dts);
  }
  cudaFree(dA), cudaFree(dW), cudaFree(db), cudaFree(dR), cudaFree(dC), cudaFree(dCh), cudaFree(dCl);
  cudaFree(Ah), cudaFree(Al), cudaFree(Wh), cudaFree(Wl);
}

// ------------------------------------------------------------------------------------------------
// Case 1c: LayerNorm folding (GemmParams::stats_out / a_stats), three chained launches on [M, 512] rows:
//   (A) producer:  u1 = R + A1 W1^T + b1            (in place over the residual pair, writes partial row statistics S1)
//   (B) consumer:  y  = LN(u1) W2^T + b2             (raw pair u1 as the A operand, gamma folded into W2, epilogue correction)
//   (C) producer:  u2 = LN(u1) + A3 W3^T + b3        (residual passed through the LayerNorm on the fly, writes S2)
// ------------------------------------------------------------------------------------------------
struct F16Weights {
  __half *hi = nullptr, *lo = nullptr;
  float scale = 1.f;
  int Kp = 0;
};
static F16Weights pack_f16(const std::vector<float>& W, int N, int K) {
  const int BK = gemm_block_k(kKindF16);
  F16Weights o;
  o.Kp = (K + BK - 1) / BK * BK;
  std::vector<float> Wp((size_t)N * o.Kp, 0.f);
  float wmax = 0.f;
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) wmax = std::fmax(wmax, std::fabs(Wp[(size_t)n * o.Kp + k] = W[(size_t)n * K + k]));
  int e2;
  std::frexp(wmax, &e2);
  o.scale = std::ldexp(1.0f, 14 - e2);
  float* d = dev(Wp);
  CK(cudaMalloc(&o.hi, Wp.size() * 2));
  CK(cudaMalloc(&o.lo, Wp.size() * 2));
  CK(launch_split_f16(d, o.hi, o.lo, (int64_t)Wp.size(), o.scale, 0));
  CK(cudaDeviceSynchronize());
  cudaFree(d);
  return o;
}
static void make_linear(GemmParams& p, const __half* Ah, const __half* Al, int M, int K, int lda, const F16Weights& w, int N, int bn) {
  p = GemmParams{};
  const int BK = gemm_block_k(kKindF16);
  if (make_tmap_2d(&p.a_hi[0], Ah, M, K, lda, kGemmBlockM, 1, kKindF16) || make_tmap_2d(&p.a_lo[0], Al, M, K, lda, kGemmBlockM, 1, kKindF16) ||
      make_tmap_2d(&p.b_hi, w.hi, N, w.Kp, w.Kp, bn, 1, kKindF16) || make_tmap_2d(&p.b_lo, w.lo, N, w.Kp, w.Kp, bn, 1, kKindF16)) {
    printf("tensor map encode failed (ln)\n");
    exit(2);
  }
  p.num_segs = 1, p.seg_kblocks[0] = w.Kp / BK, p.seg_row_mul[0] = 1;
  p.M = M, p.N = N, p.out_row_mul = 1, p.acc_scale = 1.0f / w.scale, p.ln_eps = 1e-5f;
  if (g_multicast && gemm_enable_multicast(&p, Ah, Al, M, K, lda, N, bn, kKindF16) != 0) {
    printf("gemm_enable_multicast failed (ln)\n");
    exit(2);
  }
}
static void case_linear_ln(int M, int K, bool timing) {
  const int D = 512, N2 = 1024;
  std::normal_distribution<float> nd(0.f, 1.f);
  auto randv = [&](size_t n, float sc, float off = 0.f) {
    std::vector<float> v(n);
    for (auto& x : v) x = off + sc * nd(rng);
    return v;
  };
  auto A1 = randv((size_t)M * K, 1.f), A3 = randv((size_t)M * K, 1.f), R = randv((size_t)M * D, 1.5f, 0.7f);
  auto W1 = randv((size_t)D * K, 1.f / std::sqrt((float)K)), W3 = randv((size_t)D * K, 1.f / std::sqrt((float)K));
  auto W2 = randv((size_t)N2 * D, 1.f / std::sqrt((float)D));
  auto b1 = randv(D, 1.f), b2 = randv(N2, 1.f), b3 = randv(D, 1.f), gam = randv(D, 0.1f, 1.f), bet = randv(D, 0.1f);
  // folded consumer weights
  std::vector<float> W2f((size_t)N2 * D), c2(N2), d2(N2);
  for (int n = 0; n < N2; ++n) {
    double sc = 0, sd = 0;
    for (int k = 0; k < D; ++k) {
      W2f[(size_t)n * D + k] = gam[k] * W2[(size_t)n * D + k];
      sc += W2f[(size_t)n * D + k];
      sd += (double)bet[k] * W2[(size_t)n * D + k];
    }
    c2[n] = (float)sc, d2[n] = (float)(b2[n] + sd);
  }
  const F16Weights w1 = pack_f16(W1, D, K), w2 = pack_f16(W2f, N2, D), w3 = pack_f16(W3, D, K);
  float *dA1 = dev(A1), *dA3 = dev(A3), *dR = dev(R), *db1 = dev(b1), *db3 = dev(b3), *dc2 = dev(c2), *dd2 = dev(d2);
  float *dg = dev(gam), *dbe = dev(bet);
  __half *A1h, *A1l, *A3h, *A3l, *Xh, *Xl;
  for (__half** q : {&A1h, &A1l, &A3h, &A3l}) CK(cudaMalloc(q, (size_t)M * K * 2));
  CK(cudaMalloc(&Xh, (size_t)M * D * 2));
  CK(cudaMalloc(&Xl, (size_t)M * D * 2));
  CK(launch_split_f16(dA1, A1h, A1l, (int64_t)M * K, 1.0f, 0));
  CK(launch_split_f16(dA3, A3h, A3l, (int64_t)M * K, 1.0f, 0));
  float2 *S1, *S2;
  CK(cudaMalloc(&S1, (size_t)M * 8 * sizeof(float2)));
  CK(cudaMalloc(&S2, (size_t)M * 8 * sizeof(float2)));
  float* dY = dev_zero((size_t)M * N2);
  GemmParams pa, pb, pc;
  make_linear(pa, A1h, A1l, M, K, K, w1, D, 128);
  pa.bias = db1, pa.out_hi = Xh, pa.out_lo = Xl, pa.lds = D, pa.stats_out = S1;
  make_linear(pb, Xh, Xl, M, D, D, w2, N2, 128);
  pb.bias = dd2, pb.a_stats = S1, pb.a_corr = dc2, pb.out = dY, pb.ldo = N2;
  make_linear(pc, A3h, A3l, M, K, K, w3, D, 128);
  pc.bias = db3, pc.out_hi = Xh, pc.out_lo = Xl, pc.lds = D, pc.stats_out = S2, pc.res_stats = S1, pc.res_gamma = dg, pc.res_beta = dbe;
  for (GemmParams* q : {&pa, &pb, &pc})
    if (gemm_enable_tma_store(q, M, kKindF16) != 0 || !q->tma_store) {
      printf("gemm_enable_tma_store refused a LayerNorm-folding launch\n");
      exit(2);
    }
  auto read_pair = [&](std::vector<double>& out) {
    std::vector<__half> h((size_t)M * D), l((size_t)M * D);
    CK(cudaMemcpy(h.data(), Xh, h.size() * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(l.data(), Xl, l.size() * 2, cudaMemcpyDeviceToHost));
    out.resize(h.size());
    for (size_t i = 0; i < h.size(); ++i) out[i] = (double)__half2float(h[i]) + (double)__half2float(l[i]);
  };
  CK(launch_split_f16(dR, Xh, Xl, (int64_t)M * D, 1.0f, 0));
  CK(launch_gemm(pa, M, D, 128, 3, 0, false, kKindF16));
  CK(cudaDeviceSynchronize());
  std::vector<double> u1g, u2g;
  read_pair(u1g);
  CK(launch_gemm(pb, M, N2, 128, 3, 0, false, kKindF16));
  CK(launch_gemm(pc, M, D, 128, 3, 0, false, kKindF16));
  CK(cudaDeviceSynchronize());
  read_pair(u2g);
  auto Y = host(dY, (size_t)M * N2);
  double ea = 0, eb = 0, ec = 0, ra = 0, rb = 0, rcm = 0;
  const int step = M > 600 ? 11 : 1;
  std::vector<double> u1(D), x(D);
  for (int m = 0; m < M; m += step) {
    double mean = 0;
    for (int n = 0; n < D; ++n) {
      double acc = 0;
      for (int k = 0; k < K; ++k) acc += (double)A1[(size_t)m * K + k] * W1[(size_t)n * K + k];
      u1[n] = acc + b1[n] + R[(size_t)m * D + n];
      mean += u1[n];
      ea = std::fmax(ea, std::fabs(u1g[(size_t)m * D + n] - u1[n])), ra = std::fmax(ra, std::fabs(u1[n]));
    }
    mean /= D;
    double var = 0;
    for (int n = 0; n < D; ++n) var += (u1[n] - mean) * (u1[n] - mean);
    const double rstd = 1.0 / std::sqrt(var / D + 1e-5);
    for (int n = 0; n < D; ++n) x[n] = (u1[n] - mean) * rstd * gam[n] + bet[n];
    for (int n = 0; n < N2; ++n) {
      double acc = b2[n];
      for (int k = 0; k < D; ++k) acc += x[k] * W2[(size_t)n * D + k];
      eb = std::fmax(eb, std::fabs(Y[(size_t)m * N2 + n] - acc)), rb = std::fmax(rb, std::fabs(acc));
    }
    for (int n = 0; n < D; ++n) {
      double acc = 0;
      for (int k = 0; k < K; ++k) acc += (double)A3[(size_t)m * K + k] * W3[(size_t)n * K + k];
      const double ref = x[n] + acc + b3[n];
      ec = std::fmax(ec, std::fabs(u2g[(size_t)m * D + n] - ref)), rcm = std::fmax(rcm, std::fabs(ref));
    }
  }
  char name[160];
  snprintf(name, sizeof name, "LN folding M%d K%d: (A) producer u = res + A W^T + b", M, K);
  report(name, ea, ra, 2e-5);
  report("  (B) consumer y = LN(u) W2^T + b2 via folded weights + epilogue correction", eb, rb, 3e-5);
  report("  (C) producer u2 = LN(u) + A W^T + b (residual normalised on the fly)", ec, rcm, 3e-5);
  if (timing) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const int iters = 20;
    for (GemmParams* q : {&pc, &pb}) {
      for (int i = 0; i < 3; ++i) CK(launch_gemm(*q, M, q->N, 128, 3, 0, false, kKindF16));
      CK(cudaEventRecord(e0));
      for (int i = 0; i < iters; ++i) CK(launch_gemm(*q, M, q->N, 128, 3, 0, false, kKindF16));
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("    timing %s: %.2f us/launch\n", q == &pc ? "(C) producer" : "(B) consumer N=1024", ms * 1000.0 / iters);
    }
    unsigned long long* dts;
    CK(cudaMalloc(&dts, 32 * sizeof(unsigned long long)));
    CK(cudaMemset(dts, 0, 32 * sizeof(unsigned long long)));
    pc.debug_ts = dts;
    CK(launch_gemm(pc, M, D, 128, 3, 0, false, kKindF16));
    CK(launch_gemm(pc, M, D, 128, 3, 0, false, kKindF16));
    CK(cudaDeviceSynchronize());
    unsigned long long h[32];
    CK(cudaMemcpy(h, dts, sizeof h, cudaMemcpyDeviceToHost));
    printf("    (C) CTA0 timeline (ns): setup %llu | first_tma %llu | tile0 epi start %llu | acc added %llu | stats written %llu | "
           "tile0 epi done %llu | end %llu\n",
           h[1] - h[0], h[2] - h[0], h[5] - h[0], h[8] - h[0], h[9] - h[0], h[6] - h[0], h[7] - h[0]);
    print_role_timeline(h);
    cudaFree(dts);
  }
  for (float* q : {dA1, dA3, dR, db1, db3, dc2, dd2, dg, dbe, dY}) cudaFree(q);
  for (__half* q : {A1h, A1l, A3h, A3l, Xh, Xl, w1.hi, w1.lo, w2.hi, w2.lo, w3.hi, w3.lo}) cudaFree(q);
  cudaFree(S1), cudaFree(S2);
}

// ------------------------------------------------------------------------------------------------
// Case 2: Conv1d over a padded-clip channels-last layout, as TrajNet uses it.
//   x: [B, Tp_in, Cin] with the first T_in rows of each clip real, others zero.
//   y[b, t, co] = bias[co] + sum_{j<ks} sum_ci W[co, ci, j] * x[b, t*stride + j - pad, ci]
//   Weight matrix for the GEMM: [Cout, ks * Cin_p] with tap-major K (Cin padded to 32).
// ------------------------------------------------------------------------------------------------
static void case_conv(int B, int T_in, int Tp_in, int Cin, int Cout, int ks, int stride, int pad, int block_n, int groups) {
  const int T_out = (T_in + 2 * pad - ks) / stride + 1;
  const int Tp_out = Tp_in / stride;
  const int Cin_p = (Cin + 31) / 32 * 32;
  const int ldx = (Cin + 3) / 4 * 4;
  const int Np = (Cout + block_n - 1) / block_n * block_n;
  const int Kt = ks * Cin_p;
  std::vector<float> x((size_t)B * Tp_in * ldx, 0.f), W((size_t)Np * Kt, 0.f), Wt((size_t)Cout * Cin * ks), bias(Cout);
  std::normal_distribution<float> d(0.f, 1.f);
  for (int b = 0; b < B; ++b)
    for (int t = 0; t < T_in; ++t)
      for (int c = 0; c < Cin; ++c) x[((size_t)b * Tp_in + t) * ldx + c] = d(rng);
  const float ws = 1.0f / std::sqrt((float)(Cin * ks));
  for (auto& w : Wt) w = d(rng) * ws;
  for (int co = 0; co < Cout; ++co)
    for (int ci = 0; ci < Cin; ++ci)
      for (int j = 0; j < ks; ++j) W[(size_t)co * Kt + j * Cin_p + ci] = Wt[((size_t)co * Cin + ci) * ks + j];
  fill(bias);
  float *dx = dev(x), *dW = dev(W), *db = dev(bias);
  Split sx = split(dx, x.size()), sW = split(dW, W.size());
  const int Mrows = B * Tp_out;
  float* dy = dev_zero((size_t)Mrows * Cout);
  double* dstats;
  CK(cudaMalloc(&dstats, sizeof(double) * B * groups * 2));
  CK(cudaMemset(dstats, 0, sizeof(double) * B * groups * 2));

  GemmParams p{};
  for (int j = 0; j < ks; ++j) {
    if (make_tmap_2d(&p.a_hi[j], sx.hi, (int64_t)B * Tp_in, Cin, ldx, kGemmBlockM, stride) ||
        make_tmap_2d(&p.a_lo[j], sx.lo, (int64_t)B * Tp_in, Cin, ldx, kGemmBlockM, stride)) {
      printf("tensor map encode failed (conv A)\n");
      exit(2);
    }
    p.seg_kblocks[j] = Cin_p / kGemmBlockK;
    p.seg_row_shift[j] = j - pad;
    p.seg_row_mul[j] = stride;
  }
  if (make_tmap_2d(&p.b_hi, sW.hi, Np, Kt, Kt, block_n) || make_tmap_2d(&p.b_lo, sW.lo, Np, Kt, Kt, block_n)) {
    printf("tensor map encode failed (conv B)\n");
    exit(2);
  }
  p.num_segs = ks;
  p.bias = db;
  p.out = dy, p.ldo = Cout;
  p.act = kActNone;
  p.M = Mrows, p.N = Cout;
  p.out_row_mul = 1, p.out_row_add = 0;
  p.clip_rows = Tp_out, p.clip_valid = T_out;
  p.gn_stats = dstats, p.gn_groups = groups, p.gn_group_size = Cout / groups;
  if (gemm_enable_tma_store(&p, Mrows, kKindTf32) != 0 || !p.tma_store) {  // masks + statistics through the TMA-store path
    printf("gemm_enable_tma_store refused the convolution\n");
    exit(2);
  }
  CK(launch_gemm(p, Mrows, Cout, block_n, 3, 0));
  CK(cudaDeviceSynchronize());
  auto y = host(dy, (size_t)Mrows * Cout);
  std::vector<double> stats(B * groups * 2);
  CK(cudaMemcpy(stats.data(), dstats, stats.size() * 8, cudaMemcpyDeviceToHost));

  double maxerr = 0, maxref = 0, maxpad = 0, maxstat = 0;
  std::vector<double> rs(B * groups * 2, 0.0);
  for (int b = 0; b < B; ++b)
    for (int t = 0; t < Tp_out; ++t)
      for (int co = 0; co < Cout; ++co) {
        const double got = y[((size_t)b * Tp_out + t) * Cout + co];
        if (t >= T_out) {
          maxpad = std::fmax(maxpad, std::fabs(got));
          continue;
        }
        double acc = bias[co];
        for (int j = 0; j < ks; ++j) {
          const int ti = t * stride + j - pad;
          if (ti < 0 || ti >= T_in) continue;
          for (int ci = 0; ci < Cin; ++ci)
            acc += (double)Wt[((size_t)co * Cin + ci) * ks + j] * (double)x[((size_t)b * Tp_in + ti) * ldx + ci];
        }
        maxerr = std::fmax(maxerr, std::fabs(got - acc));
        maxref = std::fmax(maxref, std::fabs(acc));
        const int g = co / (Cout / groups);
        rs[(b * groups + g) * 2] += acc;
        rs[(b * groups + g) * 2 + 1] += acc * acc;
      }
  for (size_t i = 0; i < rs.size(); ++i) maxstat = std::fmax(maxstat, std::fabs(rs[i] - stats[i]) / (1.0 + std::fabs(rs[i])));
  char name[160];
  snprintf(name, sizeof name, "conv B%d T%d/%d Cin%d Cout%d k%d s%d bn%d", B, T_in, Tp_in, Cin, Cout, ks, stride, block_n);
  report(name, maxerr, maxref, ks * Cin > 2048 ? 1e-4 : 2e-5);
  report("  pad rows written as zero", maxpad, 0, 0.0);
  report("  GroupNorm sum/sumsq (relative)", maxstat, 1, ks * Cin > 2048 ? 2e-4 : 1e-5);
  cudaFree(dx), cudaFree(dW), cudaFree(db), cudaFree(dy), cudaFree(dstats);
  cudaFree(sx.hi), cudaFree(sx.lo), cudaFree(sW.hi), cudaFree(sW.lo);
}


// ------------------------------------------------------------------------------------------------
// Fixed-cost microbenchmark: where do the non-MMA microseconds of a launch go?
// ------------------------------------------------------------------------------------------------
static void bench_fixed(int M, int N, int K, int outputs /*0 none, 1 fp32, 2 hi/lo, 3 all*/, bool with_res, int passes) {
  const int Kp = (K + 31) / 32 * 32;
  std::vector<float> A((size_t)M * Kp, 0.5f), W((size_t)N * Kp, 0.25f), b(N, 0.1f), R((size_t)M * N, 1.0f);
  float *dA = dev(A), *dW = dev(W), *db = dev(b), *dR = dev(R);
  Split sA = split(dA, A.size()), sW = split(dW, W.size());
  float* dC = dev_zero((size_t)M * N);
  float* dCh = dev_zero((size_t)M * N);
  float* dCl = dev_zero((size_t)M * N);
  GemmParams p{};
  make_tmap_2d(&p.a_hi[0], sA.hi, M, Kp, Kp, kGemmBlockM);
  make_tmap_2d(&p.a_lo[0], sA.lo, M, Kp, Kp, kGemmBlockM);
  make_tmap_2d(&p.b_hi, sW.hi, N, Kp, Kp, 128);
  make_tmap_2d(&p.b_lo, sW.lo, N, Kp, Kp, 128);
  p.num_segs = 1, p.seg_kblocks[0] = Kp / kGemmBlockK, p.seg_row_mul[0] = 1;
  p.bias = db;
  p.residual = with_res ? dR : nullptr, p.ldr = N;
  if (outputs & 1) p.out = dC, p.ldo = N;
  if (outputs & 2) p.out_hi = dCh, p.out_lo = dCl, p.lds = N;
  p.M = M, p.N = N, p.out_row_mul = 1;
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int i = 0; i < 5; ++i) CK(launch_gemm(p, M, N, 128, passes, 0));
  CK(cudaEventRecord(e0));
  const int iters = 100;
  for (int i = 0; i < iters; ++i) CK(launch_gemm(p, M, N, 128, passes, 0));
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  float ms;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  printf("fixed-cost M%d N%d K%-5d outputs=%d res=%d passes=%d : %.2f us/launch\n", M, N, K, outputs, (int)with_res, passes,
         ms * 1000.0 / iters);
  {
    unsigned long long* dts;
    CK(cudaMalloc(&dts, 32 * sizeof(unsigned long long)));
    p.debug_ts = dts;
    CK(launch_gemm(p, M, N, 128, passes, 0));
    CK(launch_gemm(p, M, N, 128, passes, 0));
    CK(cudaDeviceSynchronize());
    unsigned long long h[16];
    CK(cudaMemcpy(h, dts, sizeof h, cudaMemcpyDeviceToHost));
    printf("    CTA0 timeline (ns since kernel start): setup_done %llu | first_tma %llu | first_full %llu | mma_issued %llu | "
           "epi_start %llu | epi_done %llu | end %llu\n", h[1] - h[0], h[2] - h[0], h[3] - h[0], h[4] - h[0], h[5] - h[0],
           h[6] - h[0], h[7] - h[0]);
    printf("      epilogue chunk0 of warp2: tmem_ld done %llu | math done %llu | staged %llu | stored %llu\n", h[8] - h[0],
           h[9] - h[0], h[10] - h[0], h[11] - h[0]);
    p.debug_ts = nullptr;
    cudaFree(dts);
  }
  cudaFree(dA), cudaFree(dW), cudaFree(db), cudaFree(dR), cudaFree(dC), cudaFree(dCh), cudaFree(dCl);
  cudaFree(sA.hi), cudaFree(sA.lo), cudaFree(sW.hi), cudaFree(sW.lo);
}

__global__ void empty_kernel() {}

int main() {
  int devcount = 0;
  CK(cudaGetDeviceCount(&devcount));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s  sm_%d%d  SMs %d\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount);

  {
    // launch-only floor: an empty kernel back to back
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int i = 0; i < 10; ++i) empty_kernel<<<132, 384>>>();
    CK(cudaEventRecord(e0));
    for (int i = 0; i < 200; ++i) empty_kernel<<<132, 384>>>();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("empty kernel back-to-back: %.2f us/launch\n", ms * 1000.0 / 200);
  }
  for (int K : {32, 128, 512, 1024, 2048}) bench_fixed(4640, 512, K, 1, false, 3);
  bench_fixed(4640, 512, 32, 0, false, 3);
  bench_fixed(4640, 512, 32, 3, true, 3);
  bench_fixed(4640, 512, 512, 0, false, 3);
  bench_fixed(4640, 512, 512, 3, true, 3);
  bench_fixed(128, 128, 32, 1, false, 3);
  bench_fixed(128, 128, 512, 1, false, 3);
  bench_fixed(4640, 1536, 512, 1, false, 3);
  bench_fixed(4640, 1536, 32, 1, false, 3);

  // PoseNet shapes at B=32, S=145 (M = 4640)
  case_linear(4640, 512, 512, 128, kActNone, true, true);    // out-proj + residual
  case_linear(4640, 1536, 512, 128, kActNone, false, true);  // QKV
  case_linear(4640, 1024, 512, 128, kActGelu, false, true);  // FFN1 + GELU
  case_linear(4640, 512, 1024, 128, kActNone, true, true);   // FFN2 + residual
  case_linear(4640, 512, 294, 128, kActNone, true, false);   // input embedding (K tail via TMA OOB)
  case_linear(4640, 272, 512, 96, kActNone, false, true);    // output head (N tail)
  // the same shapes on fp16 hi/lo operands
  case_linear_f16(4640, 512, 512, 128, kActNone, true, true, 1.0f);
  case_linear_f16(4640, 1536, 512, 128, kActNone, false, true, 1.0f);
  case_linear_f16(4640, 1024, 512, 128, kActGelu, false, true, 1.0f);
  case_linear_f16(4640, 512, 1024, 128, kActNone, true, true, 1.0f);
  case_linear_f16(4640, 512, 294, 128, kActNone, true, false, 1.0f);
  case_linear_f16(4640, 272, 512, 96, kActNone, false, true, 1.0f);
  // TMA-store epilogue (PoseNet QKV / out-proj / FFN shapes, plus ragged M and N edges that mix both store paths)
  case_linear_f16(4640, 1536, 512, 128, kActNone, false, true, 1.0f, 2);
  case_linear_f16(4640, 512, 512, 128, kActNone, false, true, 1.0f, 1);
  case_linear_f16(4640, 1024, 512, 128, kActGelu, false, true, 1.0f, 2);
  case_linear_f16(4640, 512, 1024, 128, kActNone, false, true, 1.0f, 1);
  case_linear_f16(4640, 272, 512, 96, kActNone, false, true, 1.0f, 1);
  // the PoseNet shapes again with the A operand multicast across CTA pairs
  g_multicast = true;
  case_linear_f16(4640, 1536, 512, 128, kActNone, false, true, 1.0f, 2);
  case_linear_f16(4640, 1024, 512, 128, kActGelu, false, true, 1.0f, 2);
  case_linear_f16(4640, 512, 1024, 128, kActNone, false, true, 1.0f, 1);
  case_linear_f16(18560, 1536, 512, 128, kActNone, false, true, 1.0f, 2);
  case_linear_f16(145, 512, 512, 128, kActNone, false, false, 1.0f, 1);
  case_linear_f16(34, 1536, 512, 128, kActNone, false, false, 1.0f, 2);
  case_linear_ln(4640, 512, true);
  case_linear_ln(34, 1024, false);
  g_multicast = false;
  // fused residual + LayerNorm epilogue: PoseNet out-proj / FFN2 shapes, a one-stripe case and ragged row counts
  case_linear_ln(4640, 512, true);
  case_linear_ln(4640, 1024, true);
  case_linear_ln(18560, 512, true);   // 128 clips: 145 stripes -> 3.9 persistent rounds
  case_linear_ln(128, 512, false);
  case_linear_ln(34, 512, false);      // ragged last row group (per-thread store path)
  case_linear_ln(1000, 1024, false);
  case_linear_f16(145, 512, 512, 128, kActNone, false, false, 1.0f, 1);
  case_linear_f16(333, 1536, 512, 128, kActNone, false, false, 1.0f, 2);
  case_linear_f16(300, 512, 512, 128, kActNone, false, false, 300.0f);   // large activations
  case_linear_f16(300, 512, 512, 128, kActNone, false, false, 1e-3f);    // lo halves all subnormal
  case_linear_f16(77, 64, 40, 64, kActSilu, false, false, 1.0f);
  case_linear_f16(33, 13, 32, 32, kActNone, false, false, 1.0f);
  // small / ragged
  case_linear(300, 272, 294, 96, kActNone, false, false);
  case_linear(77, 64, 40, 64, kActSilu, false, false);
  case_linear(200, 128, 128, 128, kActMish, false, false);
  case_linear(33, 13, 32, 32, kActNone, false, false);
  // TrajNet-style convolutions over padded clips
  case_conv(3, 18, 22, 64, 64, 5, 1, 2, 64, 8);
  case_conv(2, 144, 176, 13, 64, 5, 1, 2, 64, 8);
  case_conv(2, 36, 44, 256, 256, 5, 1, 2, 128, 8);
  case_conv(3, 72, 88, 128, 128, 3, 2, 1, 128, 8);  // Downsample1d
  case_conv(2, 9, 11, 1024, 512, 5, 1, 2, 128, 8);
  case_conv(2, 144, 176, 32, 32, 5, 1, 2, 32, 8);

  printf(failures ? "SELFTEST FAILED (%d)\n" : "SELFTEST PASSED\n", failures);
  return failures ? 1 : 0;
}
