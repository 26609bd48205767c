"""The segmented hi/lo GEMM (rohm_b200/csrc/gemm.cu) launched directly through tests/native/libkernel_probe.so and compared
with float64 references computed on the device from the hi + lo values the kernel was fed.

Error bound (DESIGN.md section 2, test_kernel_arithmetic_model.py): per output,
    |got - ref| <= c 2^-20 (|A| |W|^T + |bias|) + 2^-25 sum_k |w|
with c = 2 for the fp16 pairs and for TF32 x3 (three products, only lo*lo dropped); single-pass TF32 rounds both operands
to 11 bits, so its bound is 2^-10 (|A| |W|^T) + the same terms.  An activation adds its own rounding, 2^-21 (1 + |y|), and
scales the bound by at most 1.25 (the largest slope of GELU / SiLU / Mish); a residual or the final fp32 store adds
2^-23 |y|.  Large row counts are checked on a seeded subset of rows."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_probe as kp
from arith_model import gemm_f16x2

pytestmark = pytest.mark.gpu

F16, TF32 = kp.KIND_F16, kp.KIND_TF32
C_PAIR = 2.0            # c of the bound for fp16 pairs and TF32 x3
C_ONE_PASS = 2.0 ** 10  # TF32 x1: c 2^-20 = 2^-10


@pytest.fixture(scope="module")
def dev(cuda_device):
    kp.lib()  # a missing probe library fails every test of the module
    return cuda_device


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _randn(shape, seed, dev, scale=1.0):
    return (torch.randn(*shape, generator=_gen(seed)) * scale).to(dev)


def _rows(M, seed):
    """All rows of small problems, a seeded subset (always with the first and last row) of large ones."""
    if M <= 1024:
        return torch.arange(M)
    r = torch.randperm(M, generator=_gen(seed))[:384]
    return torch.unique(torch.cat([r, torch.tensor([0, M - 1])]))


def _bound(abs_aw, abs_b, w_abs_sum, passes=3):
    c = C_PAIR if passes == 3 else C_ONE_PASS
    return c * 2.0 ** -20 * (abs_aw + abs_b) + 2.0 ** -25 * w_abs_sum


def _act64(y, act):
    if act == kp.ACT_GELU:
        return 0.5 * y * (1.0 + torch.erf(y / math.sqrt(2.0)))
    if act == kp.ACT_SILU:
        return y / (1.0 + torch.exp(-y))
    if act == kp.ACT_MISH:
        return y * torch.tanh(F.softplus(y))
    return y


def _check(got, ref, tol, what):
    got = got.double()
    assert bool(torch.isfinite(got).all()), what
    err = (got - ref).abs()
    ratio = float((err / tol).max())
    assert ratio <= 1.0, f"{what}: max |err| / bound = {ratio:.3f} (max |err| {float(err.max()):.3e})"
    return ratio


def _pair_matches(hi, lo, out, what):
    """The stored hi/lo split of an output equals the fp32 output to the split's own precision."""
    pair = kp.pair_value(hi, lo)
    o = out.double()
    if hi.dtype == torch.float32:  # TF32 pair: lo = v - hi exactly
        assert torch.equal(pair, o), what
    else:  # fp16 pair: 2 x 11 bits, lo halves below 2^-14 are subnormal
        assert float(((pair - o).abs() - (2.0 ** -21 * o.abs() + 2.0 ** -25)).max()) <= 0.0, what


def _linear(dev, kind, M, N, K, block_n, seed, a_scale=1.0, w_scale=None):
    a = _randn((M, K), seed, dev, a_scale)
    w = _randn((N, K), seed + 1, dev, (1.0 / math.sqrt(K)) if w_scale is None else w_scale)
    return kp.Operand(kind, a), kp.Weight(kind, [w], block_n), a, w


def _ref_linear(A, W, rows, bias=None):
    a, w = A.value[rows.to(A.value.device)], W.parts[0]
    ref = a @ w.T
    aw = a.abs() @ w.abs().T
    b = torch.zeros(W.N, dtype=torch.float64, device=a.device) if bias is None else bias.double()
    return ref + b, aw, b.abs()[None, :], w.abs().sum(1)[None, :]


LINEAR_CASES = [
    # kind, passes, block_n, M, N, K
    (F16, 3, 128, 4640, 1536, 512),   # PoseNet QKV
    (F16, 3, 96, 4640, 272, 512),     # output head: N tail
    (F16, 3, 128, 18560, 512, 512),   # 128 clips: the persistent scheduler runs several rounds
    (F16, 3, 64, 129, 200, 294),      # input embedding K tail, one row past a tile
    (F16, 3, 32, 1, 13, 40),
    (F16, 3, 128, 127, 1000, 1024),
    (F16, 3, 96, 34, 272, 5120),
    (F16, 3, 64, 128, 130, 294),
    (TF32, 3, 128, 4640, 512, 1024),
    (TF32, 3, 96, 300, 272, 294),
    (TF32, 3, 32, 34, 13, 40),
    (TF32, 3, 64, 129, 100, 5120),
    (TF32, 3, 128, 18560, 256, 512),
    (TF32, 3, 128, 4640, 1536, 512),
    (TF32, 1, 128, 4640, 512, 512),
    (TF32, 1, 96, 300, 272, 294),
    (TF32, 1, 64, 127, 272, 294),
    (TF32, 1, 32, 1, 13, 40),
]


@pytest.mark.parametrize("kind,passes,block_n,M,N,K", LINEAR_CASES)
def test_linear_with_bias_matches_float64(dev, kind, passes, block_n, M, N, K):
    """fp32 out and the hi/lo split out of one launch, column bias, NaN in the A row-pitch padding."""
    A, W, _, _ = _linear(dev, kind, M, N, K, block_n, 100 + M + N + K)
    bias = _randn((N,), 7, dev)
    out = torch.full((M, N), 777.0, device=dev)
    dt = torch.float16 if kind == F16 else torch.float32
    oh, ol = torch.empty(M, N, dtype=dt, device=dev), torch.empty(M, N, dtype=dt, device=dev)
    rc, _ = kp.gemm(kind, W, [A.seg(W.kblocks[0])], M, N, passes=passes, out=out, out_hi=oh, out_lo=ol, bias=bias)
    assert rc == 0
    torch.cuda.synchronize()
    rows = _rows(M, 5)
    ref, aw, ab, ws = _ref_linear(A, W, rows, bias)
    tol = _bound(aw, ab, ws, passes) + 2.0 ** -23 * ref.abs()
    _check(out[rows.to(dev)], ref, tol, "fp32 out")
    _check(kp.pair_value(oh, ol)[rows.to(dev)], ref, tol + 2.0 ** -21 * ref.abs() + 2.0 ** -25, "hi + lo out")
    _pair_matches(oh, ol, out, "hi + lo == out")


@pytest.mark.parametrize("kind", [F16, TF32])
@pytest.mark.parametrize("act", [kp.ACT_NONE, kp.ACT_GELU, kp.ACT_SILU, kp.ACT_MISH])
@pytest.mark.parametrize("with_res", [False, True])
def test_epilogue_activation_and_residual(dev, kind, act, with_res):
    M, N, K = 300, 200, 294
    A, W, _, _ = _linear(dev, kind, M, N, K, 64, 11 + act)
    bias = _randn((N,), 8, dev)
    res = _randn((M, N), 9, dev) if with_res else None
    out = torch.full((M, N), 777.0, device=dev)
    rc, _ = kp.gemm(kind, W, [A.seg(W.kblocks[0])], M, N, out=out, bias=bias, residual=res, act=act)
    assert rc == 0
    torch.cuda.synchronize()
    rows = torch.arange(M)
    pre, aw, ab, ws = _ref_linear(A, W, rows, bias)
    ref = _act64(pre, act)
    tol = _bound(aw, ab, ws) * (1.25 if act else 1.0) + (2.0 ** -21 * (1.0 + ref.abs()) if act else 0.0)
    if with_res:
        ref = ref + res.double()
    _check(out, ref, tol + 2.0 ** -23 * ref.abs(), f"act {act} residual {with_res}")


@pytest.mark.parametrize("kind,form", [(F16, "fp32"), (F16, "pair"), (TF32, "fp32")])
@pytest.mark.parametrize("M,N,block_n", [(4640, 1536, 128), (333, 272, 96), (145, 512, 128), (34, 104, 64)])
def test_tma_store_epilogue_with_ragged_edges(dev, kind, form, M, N, block_n):
    """The bulk-store epilogue; chunks on a ragged M or N edge take the per-thread path in the same launch."""
    A, W, _, _ = _linear(dev, kind, M, N, 512, block_n, 21 + M)
    bias = _randn((N,), 4, dev)
    out = oh = ol = None
    if form == "fp32":
        out = torch.full((M, N), 777.0, device=dev)
    else:
        oh, ol = torch.full((M, N), 77.0, dtype=torch.float16, device=dev), torch.zeros(M, N, dtype=torch.float16, device=dev)
    rc, g = kp.gemm(kind, W, [A.seg(W.kblocks[0])], M, N, out=out, out_hi=oh, out_lo=ol, bias=bias, tma_store=True)
    assert rc == 0 and g.tma_store == 1
    torch.cuda.synchronize()
    rows = _rows(M, 6)
    ref, aw, ab, ws = _ref_linear(A, W, rows, bias)
    tol = _bound(aw, ab, ws) + 2.0 ** -23 * ref.abs()
    got = out if form == "fp32" else kp.pair_value(oh, ol)
    _check(got[rows.to(dev)], ref, tol + (2.0 ** -21 * ref.abs() + 2.0 ** -25 if form == "pair" else 0.0), form)


@pytest.mark.parametrize("w_scale", [1e-6, 3e-3, 4e4])
def test_weight_scale_is_undone_exactly_by_acc_scale(dev, w_scale):
    """fp16 pairs store w 2^s with 2^s chosen per matrix; acc_scale = 2^-s scales the accumulator back in the epilogue."""
    M, N, K = 200, 128, 512
    A, W, _, _ = _linear(dev, F16, M, N, K, 128, 31, w_scale=w_scale)
    assert W.scale == 2.0 ** round(math.log2(W.scale)) and W.scale != 1.0
    out = torch.zeros(M, N, device=dev)
    assert kp.gemm(F16, W, [A.seg(W.kblocks[0])], M, N, out=out)[0] == 0
    torch.cuda.synchronize()
    ref, aw, ab, ws = _ref_linear(A, W, torch.arange(M))
    _check(out, ref, _bound(aw, ab, ws) + 2.0 ** -23 * ref.abs(), f"w_scale {w_scale}")


# ---------------------------------------------------------------------------------------------------------------------------
# convolutions over padded clips (TrajNet): channels-last rows, clip b at rows [b Tp, b Tp + T), pad rows zero
# ---------------------------------------------------------------------------------------------------------------------------
def _clips(B, T, Tp, C, seed, dev):
    x = torch.zeros(B, Tp, C, device=dev)
    x[:, :T] = _randn((B, T, C), seed, dev)
    return x


def _conv_setup(dev, kind, B, T, Tp, cins, Cout, ks, stride, block_n, seed):
    """Conv1d(k, stride, pad = k // 2) over the channel concat of len(cins) sources; segments tap-major.  The returned
    operands own the memory the segments point to: keep them alive until the launch has completed."""
    pad = ks // 2
    srcs = [_clips(B, T, Tp, c, seed + i, dev) for i, c in enumerate(cins)]
    ops = [kp.Operand(kind, s.reshape(B * Tp, -1)) for s in srcs]
    Wt = _randn((Cout, sum(cins), ks), seed + 10, dev, 1.0 / math.sqrt(sum(cins) * ks))
    parts, segs_spec = [], []
    for j in range(ks):
        off = 0
        for i, c in enumerate(cins):
            parts.append(Wt[:, off:off + c, j])
            segs_spec.append((i, j - pad))
            off += c
    W = kp.Weight(kind, parts, block_n)
    segs = [ops[i].seg(W.kblocks[n], shift, stride) for n, (i, shift) in enumerate(segs_spec)]
    # the weight values the kernel multiplies, back in Conv1d layout; inputs as the kernel reads them
    W64 = torch.zeros(Cout, sum(cins), ks, dtype=torch.float64, device=dev)
    for n, (i, shift) in enumerate(segs_spec):
        off = sum(cins[:i])
        W64[:, off:off + cins[i], shift + pad] = W.parts[n]
    x64 = torch.cat([o.value.reshape(B, Tp, -1)[:, :T] for o in ops], dim=2).permute(0, 2, 1)
    return W, segs, W64, x64, pad, ops


LEVELS = [(144, 176, 13, 64), (72, 88, 128, 128), (36, 44, 256, 256), (18, 22, 512, 512), (9, 11, 1024, 512)]


@pytest.mark.parametrize("kind", [F16, TF32])
@pytest.mark.parametrize("level", range(5))
def test_conv_k5_masks(dev, kind, level):
    """k = 5 taps (row shifts -2..+2) at the TrajNet level shapes, pad rows exactly 0; levels 1 and 3 read a two-source
    channel concat (the decoder's skip connections)."""
    T, Tp, Cin, Cout = LEVELS[level]
    B = 3
    cins = [Cin // 2, Cin - Cin // 2] if level in (1, 3) else [Cin]
    block_n = 64 if Cout <= 64 else 128
    W, segs, W64, x64, pad, ops = _conv_setup(dev, kind, B, T, Tp, cins, Cout, 5, 1, block_n, 40 + level)
    bias = _randn((Cout,), 3, dev)
    out = torch.full((B * Tp, Cout), 777.0, device=dev)
    rc, g = kp.gemm(kind, W, segs, B * Tp, Cout, out=out, bias=bias, clip_rows=Tp, clip_valid=T, tma_store=True)
    assert rc == 0 and g.tma_store == 1
    torch.cuda.synchronize()
    y = out.reshape(B, Tp, Cout)
    assert bool((y[:, T:] == 0).all()), "pad rows must be written as exact zeros"
    ref = F.conv1d(x64, W64, bias.double(), padding=pad).permute(0, 2, 1)
    aw = F.conv1d(x64.abs(), W64.abs(), padding=pad).permute(0, 2, 1)
    ws = W64.abs().sum((1, 2))
    _check(y[:, :T], ref, _bound(aw, bias.double().abs(), ws) + 2.0 ** -23 * ref.abs(), "conv")


@pytest.mark.parametrize("kind", [F16, TF32])
@pytest.mark.parametrize("level", range(4))
def test_downsample_k3_stride2(dev, kind, level):
    """Downsample1d: k = 3, stride 2, pad 1 (row_mul 2 through the tensor map's traversal stride), level L -> L + 1."""
    T, Tp, C, _ = LEVELS[level]
    C = max(C, 32)
    B = 3
    W, segs, W64, x64, pad, ops = _conv_setup(dev, kind, B, T, Tp, [C], C, 3, 2, 128 if C >= 128 else 64, 60 + level)
    To, Tpo = T // 2, Tp // 2
    bias = _randn((C,), 2, dev)
    out = torch.full((B * Tpo, C), 777.0, device=dev)
    assert kp.gemm(kind, W, segs, B * Tpo, C, out=out, bias=bias, clip_rows=Tpo, clip_valid=To)[0] == 0
    torch.cuda.synchronize()
    y = out.reshape(B, Tpo, C)
    assert bool((y[:, To:] == 0).all())
    ref = F.conv1d(x64, W64, bias.double(), stride=2, padding=pad).permute(0, 2, 1)
    aw = F.conv1d(x64.abs(), W64.abs(), stride=2, padding=pad).permute(0, 2, 1)
    _check(y[:, :To], ref, _bound(aw, bias.double().abs(), W64.abs().sum((1, 2))) + 2.0 ** -23 * ref.abs(), "downsample")


@pytest.mark.parametrize("kind", [F16, TF32])
@pytest.mark.parametrize("level", [0, 2, 3])
def test_conv_transpose_from_two_phase_launches(dev, kind, level):
    """ConvTranspose1d(k4, s2, p1) from level L + 1 to L: output row 2t + phase; phase 0 sums taps 1 (row t) and 3 (row
    t - 1), phase 1 taps 0 (row t + 1) and 2 (row t); out_row_mul = 2, out_row_add = phase."""
    T, Tp, C, _ = LEVELS[level + 1]
    Cin, Cout, B = C, max(LEVELS[level][3], 64), 3
    x = _clips(B, T, Tp, Cin, 80 + level, dev)
    A = kp.Operand(kind, x.reshape(B * Tp, Cin))
    Wt = _randn((Cin, Cout, 4), 81 + level, dev, 1.0 / math.sqrt(2 * Cin))
    out = torch.full((B * 2 * Tp, Cout), 777.0, device=dev)
    bias = _randn((Cout,), 5, dev)
    W64 = torch.zeros(Cin, Cout, 4, dtype=torch.float64, device=dev)
    for phase, taps in ((0, ((1, 0), (3, -1))), (1, ((0, 1), (2, 0)))):
        W = kp.Weight(kind, [Wt[:, :, k].T.contiguous() for k, _ in taps], 64)
        for n, (k, _) in enumerate(taps):
            W64[:, :, k] = W.parts[n].T
        segs = [A.seg(W.kblocks[n], shift) for n, (_, shift) in enumerate(taps)]
        rc, _ = kp.gemm(kind, W, segs, B * Tp, Cout, out=out, bias=bias, clip_rows=Tp, clip_valid=T, out_row_mul=2,
                        out_row_add=phase)
        assert rc == 0
    torch.cuda.synchronize()
    y = out.reshape(B, 2 * Tp, Cout)
    assert bool((y[:, 2 * T:] == 0).all())
    x64 = A.value.reshape(B, Tp, Cin)[:, :T].permute(0, 2, 1)
    ref = F.conv_transpose1d(x64, W64, bias.double(), stride=2, padding=1).permute(0, 2, 1)
    aw = F.conv_transpose1d(x64.abs(), W64.abs(), stride=2, padding=1).permute(0, 2, 1)
    ws = W64.abs().sum((0, 2)) / 2  # each output sums two of the four taps
    _check(y[:, :2 * T], ref, _bound(aw, bias.double().abs(), ws) + 2.0 ** -23 * ref.abs(), "conv transpose")


# ---------------------------------------------------------------------------------------------------------------------------
# split-K (TrajNet deep levels): split s stores its fp32 partial at rows m + s * split_row_stride
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [F16, TF32])
@pytest.mark.parametrize("level", [3, 4])
@pytest.mark.parametrize("splits", [2, 3, 5, 8])
def test_split_k_partials(dev, kind, level, splits):
    T, Tp, Cin, Cout = LEVELS[level]
    B = 4
    W, segs, W64, x64, pad, ops = _conv_setup(dev, kind, B, T, Tp, [Cin], Cout, 5, 1, 128, 90 + level)
    M = B * Tp
    stride = -(-M // 128) * 128
    out = torch.full((splits * stride, Cout), 777.0, device=dev)
    outs = []
    for _ in range(2):
        rc, _ = kp.gemm(kind, W, segs, M, Cout, out=out, clip_rows=Tp, clip_valid=T, k_splits=splits,
                        split_row_stride=stride)
        assert rc == 0
        torch.cuda.synchronize()
        outs.append(out.clone())
    assert torch.equal(outs[0], outs[1]), "split-K must be deterministic"
    parts = outs[0].reshape(splits, stride, Cout)[:, :M]
    acc = parts[0].clone()
    for s in range(1, splits):  # the consumer's order
        acc = acc + parts[s]
    y = acc.reshape(B, Tp, Cout)
    assert bool((parts.reshape(splits, B, Tp, Cout)[:, :, T:] == 0).all())
    ref = F.conv1d(x64, W64, padding=pad).permute(0, 2, 1)
    aw = F.conv1d(x64.abs(), W64.abs(), padding=pad).permute(0, 2, 1)
    tol = _bound(aw, 0.0, W64.abs().sum((1, 2))) + splits * 2.0 ** -23 * aw
    _check(y[:, :T], ref, tol, f"split-K {splits}")


@pytest.mark.parametrize("kind", [F16, TF32])
def test_split_k_refusals_launch_nothing(dev, kind):
    """launch_cfg refuses an empty last K range and partial rows that would overlap, before launching."""
    T, Tp, Cin, Cout = LEVELS[3]
    B = 2
    W, segs, _, _, _, ops = _conv_setup(dev, kind, B, T, Tp, [64], 128, 5, 1, 128, 99)
    iters = sum(W.kblocks)
    M = B * Tp
    out = torch.full((16 * 128, 128), 777.0, device=dev)
    bad = next(s for s in range(2, 16) if (s - 1) * (-(-iters // s)) >= iters)
    rc, _ = kp.gemm(kind, W, segs, M, 128, out=out, clip_rows=Tp, clip_valid=T, k_splits=bad, split_row_stride=128)
    assert rc == kp.CUDA_ERROR_INVALID_VALUE
    rc, _ = kp.gemm(kind, W, segs, M, 128, out=out, clip_rows=Tp, clip_valid=T, k_splits=2, split_row_stride=M - 1)
    assert rc == kp.CUDA_ERROR_INVALID_VALUE
    torch.cuda.synchronize()
    assert bool((out == 777.0).all())


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [34, 128, 1000, 4640, 18560])
def test_layernorm_folding_chain(dev, M):
    """(A) producer u1 = R + A1 W1^T + b1 in place over the residual pair, with per-row partial statistics;
    (B) consumer y = LN(u1) W2^T + b2 through gamma-folded weights and the epilogue correction;
    (C) producer u2 = LN(u1) + A3 W3^T + b3 with the residual normalised on the fly."""
    D, N2, K = 512, 1024, 512
    A1, W1, a1, _ = _linear(dev, F16, M, D, K, 128, 200)
    A3, W3, a3, _ = _linear(dev, F16, M, D, K, 128, 202)
    R = _randn((M, D), 204, dev, 1.5) + 0.7
    W2 = _randn((N2, D), 205, dev, 1.0 / math.sqrt(D))
    b1, b2, b3 = _randn((D,), 206, dev), _randn((N2,), 207, dev), _randn((D,), 208, dev)
    gam, bet = _randn((D,), 209, dev, 0.1) + 1.0, _randn((D,), 210, dev, 0.1)
    W2f = (gam[None, :] * W2).contiguous()
    c2 = W2f.double().sum(1).float()
    d2 = (b2.double() + W2.double() @ bet.double()).float()
    W2p = kp.Weight(F16, [W2f], 128)
    Xh, Xl = kp.split(F16, R)
    S1 = torch.zeros(M, 16, device=dev)
    S2 = torch.zeros(M, 16, device=dev)
    Y = torch.zeros(M, N2, device=dev)
    rc, g = kp.gemm(F16, W1, [A1.seg(W1.kblocks[0])], M, D, out_hi=Xh, out_lo=Xl, bias=b1, stats_out=S1, tma_store=True)
    assert rc == 0 and g.tma_store == 1
    torch.cuda.synchronize()
    u1g = kp.pair_value(Xh, Xl)
    X = kp.Operand(F16, torch.zeros(M, D, device=dev))
    X.hi, X.lo = Xh, Xl  # the consumer reads the pair in place
    rc, g = kp.gemm(F16, W2p, [X.seg(W2p.kblocks[0])], M, N2, out=Y, bias=d2, a_stats=S1, a_corr=c2, tma_store=True)
    assert rc == 0
    rc, g = kp.gemm(F16, W3, [A3.seg(W3.kblocks[0])], M, D, out_hi=Xh, out_lo=Xl, bias=b3, stats_out=S2, res_stats=S1,
                    res_gamma=gam, res_beta=bet, tma_store=True)
    assert rc == 0
    torch.cuda.synchronize()
    u2g = kp.pair_value(Xh, Xl)
    Rv = kp.pair_value(*kp.split(F16, R))
    u1 = A1.value @ W1.parts[0].T + b1.double() + Rv
    aw1 = A1.value.abs() @ W1.parts[0].abs().T + b1.double().abs() + Rv.abs()
    tol1 = C_PAIR * 2.0 ** -20 * aw1 + 2.0 ** -21 * u1.abs() + 2.0 ** -24
    _check(u1g, u1, tol1, "(A) producer")
    # LayerNorm of the stored pair (the consumers see what was stored)
    mean = u1g.mean(1, keepdim=True)
    var = ((u1g - mean) ** 2).mean(1, keepdim=True)
    xn = (u1g - mean) / torch.sqrt(var + 1e-5)
    x = xn * gam.double() + bet.double()
    y = x @ W2.double().T + b2.double()
    # the folded form cancels mean * c_n in fp32: error scale rstd (|u| |W'| + |mean| |c|) and |x| |W|
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    ayw = rstd * (u1g.abs() @ W2f.double().abs().T + mean.abs() * c2.double().abs()[None, :]) + x.abs() @ W2.double().abs().T
    _check(Y, y, 4.0 * 2.0 ** -20 * ayw + 2.0 ** -23 * y.abs() + 1e-7, "(B) consumer")
    u2 = x + A3.value @ W3.parts[0].T + b3.double()
    aw3 = x.abs() + A3.value.abs() @ W3.parts[0].abs().T + b3.double().abs()
    _check(u2g, u2, 4.0 * 2.0 ** -20 * aw3 + 2.0 ** -21 * u2.abs() + 2.0 ** -24, "(C) producer")


# ---------------------------------------------------------------------------------------------------------------------------
# fp16 range: the kernel computes exactly the CPU arithmetic model of the fp16 pairs (tests/arith_model.py)
# ---------------------------------------------------------------------------------------------------------------------------
def _model_case(dev, a, w, block_n=128):
    M, K = a.shape
    N = w.shape[0]
    A, W = kp.Operand(F16, a), kp.Weight(F16, [w], block_n)
    out = torch.zeros(M, N, device=dev)
    assert kp.gemm(F16, W, [A.seg(W.kblocks[0])], M, N, out=out)[0] == 0
    torch.cuda.synchronize()
    model = torch.from_numpy(gemm_f16x2(a.cpu().numpy(), w.cpu().numpy())).double().to(dev)
    aw = a.double().abs() @ w.double().abs().T
    # the model rounds each accumulator once; the tensor core truncates every addition into its fp32 accumulator, up to one
    # ulp of the running sum per 16-wide k-step (biased, so it adds up linearly), plus the final add of the two accumulators
    tol = (K / 16 + 2) * 2.0 ** -23 * aw + 2.0 ** -24 * model.abs()
    return A, W, out, model, aw, tol


@pytest.mark.parametrize("a_scale", [1.0, 1e-3, 300.0, 1.3e5])
def test_f16_kernel_equals_the_cpu_model(dev, a_scale):
    """Activations at 1e-3 (lo halves subnormal), 300 and up to 1.3e5 (inside the pair's range |x| < 131024: above 65504 the
    hi half saturates and the lo half carries the rest, so the reference is the model, not fp32 grade)."""
    M, N, K = 256, 192, 512
    if a_scale > 65504.0:  # uniform up to the limit
        a = ((torch.rand(M, K, generator=_gen(300)) * 2.0 - 1.0) * a_scale).to(dev)
    else:
        a = _randn((M, K), 300, dev, a_scale)
    w = _randn((N, K), 301, dev, 1.0 / math.sqrt(K))
    A, W, out, model, aw, tol = _model_case(dev, a, w)
    _check(out, model, tol + 1e-30, f"model, a_scale {a_scale}")
    if a_scale <= 300.0:
        ref = a.double() @ W.parts[0].T
        _check(out, ref, _bound(aw, 0.0, W.parts[0].abs().sum(1)[None, :]) + 2.0 ** -23 * ref.abs(), "float64")


def test_weight_outlier_loses_lo_bits_as_the_model_says(dev):
    """One weight 1e3 times the rest: the per-matrix scale is set by the outlier, the small weights sit 2^10 lower in the
    fp16 range and the smallest of them lose lo bits to the subnormals.  The kernel must still equal the model."""
    M, N, K = 256, 128, 512
    a = _randn((M, K), 310, dev)
    w = _randn((N, K), 311, dev, 1.0 / math.sqrt(K))
    w[5, 17] = 1e3 * float(w.abs().max())
    A, W, out, model, aw, tol = _model_case(dev, a, w)
    _check(out, model, tol, "model, outlier weight")


@pytest.mark.parametrize("kind", [F16, TF32])
def test_nan_row_stays_in_its_row(dev, kind):
    """A NaN in one A row turns exactly that output row to NaN; every other row of its 128-row tile is unchanged bit for bit."""
    M, N, K = 300, 256, 512
    a = _randn((M, K), 400, dev)
    w = _randn((N, K), 401, dev, 1.0 / math.sqrt(K))
    W = kp.Weight(kind, [w], 128)
    outs = []
    for poison in (False, True):
        x = a.clone()
        if poison:
            x[130, 77] = float("nan")
        A = kp.Operand(kind, x)
        out = torch.zeros(M, N, device=dev)
        assert kp.gemm(kind, W, [A.seg(W.kblocks[0])], M, N, out=out, bias=_randn((N,), 402, dev))[0] == 0
        torch.cuda.synchronize()
        outs.append(out)
    assert bool(torch.isnan(outs[1][130]).all())
    keep = torch.ones(M, dtype=torch.bool)
    keep[130] = False
    assert torch.equal(outs[0][keep.to(dev)], outs[1][keep.to(dev)])
    assert bool(torch.isfinite(outs[0]).all())
