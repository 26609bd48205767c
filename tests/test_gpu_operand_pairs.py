"""The operand pairs every kernel hands to the next one, and the GEMM epilogue activations, at the edges of their range.

Pairs (DESIGN.md section 2, tests/arith_model.py): the fp16 pair of an fp32 value x is hi = rn_f16(x) saturated to +-65504
(NaN stays NaN) and lo = rn_f16(x - hi) unsaturated, so it is finite exactly when |x| < 131024 and +-inf beyond, with the
scalar (ptx::split_f16) and packed (split_f16x2 / split_f16x4) forms bit-identical except for NaN payloads.  The helpers
themselves (through tests/native/libkernel_probe.so's probe_pair_forms) and every kernel path that writes a pair are held to
the CPU model bit for bit, the model applied to the fp32 value the path computed; for NaN only the class is compared.

Activations: the GEMM epilogues run on x = fp32(a_m + b_n), a_m one exactly pair-representable A column, W all ones (exact
through the weight scale 2^13) and b_n the bias, so x is known exactly on the host.  Bounds against float64:
  * GELU (gemm.cu gelu_erf): the fitted form's 2.5e-7 maximum error plus the rounding of the output, 2^-24 |y|; below
    x = -6.5 the clamp takes the tail |x| Phi(-|x|) as |x| 2^Q(6.5), which adds up to 3.6e-11 |x|.
  * SiLU, x / (1 + expf(-x)): expf is within 2 ulp (CUDA C Programming Guide, single-precision function accuracy), the add
    and the IEEE division round once each, and the condition number of 1 + e in e is below 1: relative 2^-22 + 2^-23 < 2^-21.
  * Mish, x tanhf(log1pf(expf(x))) (x tanhf(x) above 20): expf 2 ulp, log1pf 1 ulp, tanhf 2 ulp, the product 1/2 ulp, and
    the condition numbers of log1p(e) in e and of tanh(s) in s are below 1: relative 11 x 2^-24.
  SiLU and Mish add an absolute 2^-118: where expf over- or underflows (|x| > 87) both results are below 104 x 2^-126.
A non-finite input must give a non-finite output: NaN stays NaN, +-inf never becomes a finite value."""
import math

import numpy as np
import pytest
import torch
from scipy.special import expit, ndtr

import kernel_probe as kp
from arith_model import split_f16, split_tf32

pytestmark = pytest.mark.gpu

f16, f32, f64 = np.float16, np.float32, np.float64
F16 = kp.KIND_F16
# fp32 values of every class of the fp16 pair: finite above 65504, the largest finite pair, the edge, +-inf pairs, NaN
EDGES = [1.2e5, 131008.0, 131023.99, 131024.0, 2e5, 65504.0, 65519.996, 65520.0, 3.4028235e38, math.inf]
EDGES = [f32(v) for v in EDGES] + [f32(-v) for v in EDGES] + [f32(math.nan)]


@pytest.fixture(scope="module")
def dev(cuda_device):
    kp.lib()  # a missing probe library fails every test of the module
    return cuda_device


def _np(t):
    return t.detach().cpu().numpy()


def _same(got, want, what, x=None):
    """got equals want bit for bit where want is not NaN, and is NaN where want is."""
    got, want = np.asarray(got).ravel(), np.asarray(want, dtype=got.dtype).ravel()
    ut = np.uint16 if got.dtype == f16 else np.uint32
    nan = np.isnan(want)
    bad = np.where(nan, ~np.isnan(got), got.view(ut) != want.view(ut))
    if bad.any():
        i = np.flatnonzero(bad)[:6]
        src = "" if x is None else f" x={np.asarray(x).ravel()[i].tolist()}"
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ;{src} got {got[i].tolist()} want {want[i].tolist()}")


def _pair_is_model(x, hi, lo, what):
    """The stored fp16 pair (device tensors) of the fp32 values x (numpy) is the model's pair of x."""
    x = np.asarray(x, dtype=f32).ravel()
    mh, ml = split_f16(x)
    _same(_np(hi).ravel(), mh.astype(f16), f"{what}: hi", x)
    _same(_np(lo).ravel(), ml.astype(f16), f"{what}: lo", x)


# ---------------------------------------------------------------------------------------------------------------------------
# the helpers of ptx.cuh
# ---------------------------------------------------------------------------------------------------------------------------
def _helper_inputs():
    e = [0.0, -0.0, 1e-45, 2e-45, 1.1754942e-38, 1.1754944e-38, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -24, 1.5 * 2.0 ** -24,
         2.0 ** -14 - 2.0 ** -24, 2.0 ** -14, 2.0 ** -14 + 2.0 ** -25,
         1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -22, 1.0 + 2.0 ** -11 + 3 * 2.0 ** -22,  # hi / lo ties
         2048.0 + 1.0, 2048.0 + 3.0, 1.0 + 2.0 ** -13, 1.0 + 2.0 ** -12 + 2.0 ** -13,                             # TF32 ties
         65504.0, 65519.996, 65520.0, 131008.0, 131023.99, 131024.0, 2e5, 1e30, 3.4028235e38, 3.4028e38,
         2.0 ** 128 * (1.0 - 2.0 ** -12), 2.0 ** 128 * (1.0 - 2.0 ** -11), math.inf]
    lo, hi = np.array([2.0 ** -24, 2.0 ** -14], dtype=f32).view(np.uint32)
    x = np.concatenate([np.array(e, dtype=f32), np.arange(1, 1024, dtype=np.uint16).view(f16).astype(f32),  # fp16 subnormals
                        np.arange(lo, hi + 1, 331, dtype=np.uint32).view(f32)])  # fp32 values that split into them
    x = np.concatenate([x, -x])
    nans = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FBFFFFF, 0x7FC01234, 0xFF812345, 0x7FFFFFFF], dtype=np.uint32)
    rnd = np.random.default_rng(11).integers(0, 2 ** 32, size=2 ** 20, dtype=np.uint64).astype(np.uint32)
    x = np.concatenate([x, nans.view(f32), rnd.view(f32)])
    return np.concatenate([x, np.zeros(-len(x) % 4, dtype=f32)])


def test_pair_helpers_match_the_model_bit_for_bit(dev):
    """split_f16, split_f16x2, split_f16x4 and the TF32 pair against tests/arith_model.py: zeros, fp32 and fp16 subnormals,
    rounding ties of hi and lo, the fp16 pair's range edges, FLT_MAX and the TF32 top binade, +-inf, quiet and payload NaNs,
    and 2^20 random bit patterns.  The scalar and packed forms agree bit for bit on every non-NaN input."""
    x = _helper_inputs()
    hi, lo, t_hi, t_lo = kp.pair_forms(torch.from_numpy(x).to(dev))
    torch.cuda.synchronize()
    hi, lo = _np(hi), _np(lo)
    mh, ml = split_f16(x)
    for form, name in enumerate(("split_f16", "split_f16x2", "split_f16x4")):
        _same(hi[form], mh.astype(f16), f"{name} hi", x)
        _same(lo[form], ml.astype(f16), f"{name} lo", x)
    finite_class = ~np.isnan(x)
    for form in (1, 2):
        assert (hi[form][finite_class].view(np.uint16) == hi[0][finite_class].view(np.uint16)).all()
        assert (lo[form][finite_class].view(np.uint16) == lo[0][finite_class].view(np.uint16)).all()
    th, tl = split_tf32(x)
    _same(_np(t_hi), th, "TF32 hi", x)
    _same(_np(t_lo), tl, "TF32 lo", x)


# ---------------------------------------------------------------------------------------------------------------------------
# GEMM epilogues: x = fp32(a_m + b_n) through one pair-exact A column and a weight of ones
# ---------------------------------------------------------------------------------------------------------------------------
def _exact_gemm(dev, a, N, block_n):
    """A [M, 1] (a: pair-exact float32) and W [N, 1] of ones: the accumulator times acc_scale is a_m exactly."""
    hi, lo = split_f16(a)
    assert (hi.astype(f64) + lo.astype(f64) == a.astype(f64)).all(), "A column not exactly pair-representable"
    A = kp.Operand(F16, torch.from_numpy(a[:, None].copy()).to(dev))
    W = kp.Weight(F16, [torch.ones(N, 1, device=dev)], block_n)
    return A, W


def _edge_bias(N, seed):
    """Bias columns cycling through EDGES, with random normal values between them."""
    b = np.random.default_rng(seed).standard_normal(N).astype(f32) * 3.0
    b[::3] = [EDGES[i % len(EDGES)] for i in range(len(b[::3]))]
    return b


def _edge_rows(M, seed):
    """Pair-exact A values: 0 (the bias alone) and small multiples of 2^-6."""
    a = (np.random.default_rng(seed).integers(-256, 257, size=M) / 64.0).astype(f32)
    a[::5] = 0.0
    return a


def test_gemm_pair_stores_follow_the_model(dev):
    """Every pair-writing path of the GEMM epilogue on values of every class: the dense pair store next to the fp32 output
    (packed split on full 32-column chunks, scalar split on the ragged N tail), the same with a residual, and the TMA-store
    path (packed split on full 32-row groups, the per-thread paths on the ragged last row group and N tail)."""
    M, N = 300, 200
    a = _edge_rows(M, 1)
    b = _edge_bias(N, 2)
    A, W = _exact_gemm(dev, a, N, 64)
    bias = torch.from_numpy(b).to(dev)
    with np.errstate(invalid="ignore", over="ignore"):
        x = a[:, None] + b[None, :]
    seg = [A.seg(W.kblocks[0])]

    out = torch.full((M, N), 777.0, device=dev)
    oh, ol = torch.empty(M, N, dtype=torch.float16, device=dev), torch.empty(M, N, dtype=torch.float16, device=dev)
    rc, g = kp.gemm(F16, W, seg, M, N, out=out, out_hi=oh, out_lo=ol, bias=bias)
    assert rc == 0 and g.tma_store == 0
    torch.cuda.synchronize()
    _same(_np(out), x, "fp32 out == fp32(a + b)", x)
    _pair_is_model(_np(out), oh, ol, "dense pair store")

    r = np.random.default_rng(3).standard_normal((M, N)).astype(f32)
    r[::7, ::3] = np.resize(np.array(EDGES, dtype=f32), r[::7, ::3].shape)
    out.fill_(777.0)
    rc, g = kp.gemm(F16, W, seg, M, N, out=out, out_hi=oh, out_lo=ol, bias=bias, residual=torch.from_numpy(r).to(dev))
    assert rc == 0
    torch.cuda.synchronize()
    with np.errstate(invalid="ignore", over="ignore"):
        _same(_np(out), x + r, "fp32 out with residual", x)
    _pair_is_model(_np(out), oh, ol, "dense pair store with residual")

    oh.fill_(77.0), ol.fill_(0.0)
    rc, g = kp.gemm(F16, W, seg, M, N, out_hi=oh, out_lo=ol, bias=bias, tma_store=True)
    assert rc == 0 and g.tma_store == 1
    torch.cuda.synchronize()
    _pair_is_model(x, oh, ol, "TMA-store pair")


@pytest.mark.parametrize("M", [128, 100])
def test_layernorm_producer_pairs_follow_the_model(dev, M):
    """The LayerNorm-folding producer (stats_out) writes u = residual pair + acc 2^-s + bias in place: with a zero residual
    u = fp32(a + b), stored through the packed split of stage_pair_chunk on full 32-row groups and the scalar split on a
    ragged last group (M = 100)."""
    N = 512
    a = _edge_rows(M, 4)
    b = _edge_bias(N, 5)
    A, W = _exact_gemm(dev, a, N, 128)
    with np.errstate(invalid="ignore", over="ignore"):
        u = f32(0.0) + (a[:, None] + b[None, :])
    oh, ol = torch.zeros(M, N, dtype=torch.float16, device=dev), torch.zeros(M, N, dtype=torch.float16, device=dev)
    stats = torch.zeros(M, 16, device=dev)
    rc, g = kp.gemm(F16, W, [A.seg(W.kblocks[0])], M, N, out_hi=oh, out_lo=ol, bias=torch.from_numpy(b).to(dev),
                    stats_out=stats, tma_store=True)
    assert rc == 0 and g.tma_store == 1
    torch.cuda.synchronize()
    _pair_is_model(u, oh, ol, f"LayerNorm producer, M = {M}")


def test_group_norm_pairs_follow_the_model(dev):
    """gn_mish_split_kernel with f16 = 1 writes the fp32 output and its pair (store_act4, packed split) in one launch; r1
    brings values of every class into the output."""
    B, T, C = 2, 48, 64
    g = torch.Generator().manual_seed(12)
    rnd = lambda *s: torch.randn(*s, generator=g).to(dev)
    rows = B * T
    r1 = torch.randn(rows * C, generator=g)
    r1[::5] = torch.tensor(np.resize(np.array(EDGES, dtype=f32), r1[::5].shape))
    out = torch.full((rows * C,), 777.0, device=dev)
    hi, lo = torch.empty(rows * C, dtype=torch.float16, device=dev), torch.empty(rows * C, dtype=torch.float16, device=dev)
    rc = kp.group_norm(rnd(1, rows * C), 1, rows * C, rnd(C), 1.0 + 0.2 * rnd(C), 0.3 * rnd(C), None, 0, r1.to(dev), None, out,
                       hi, lo, C, T, T, B, 1, 1)
    torch.cuda.synchronize()
    assert rc == 0
    o = _np(out)
    assert (np.isnan(o) == np.isnan(r1.numpy())).all() and np.isinf(o).sum() >= np.isinf(r1.numpy()).sum()
    _pair_is_model(o, hi, lo, "GroupNorm pair store")


# ---------------------------------------------------------------------------------------------------------------------------
# attention: one non-finite V element
# ---------------------------------------------------------------------------------------------------------------------------
D, H, DH = 512, 4, 128
POISON_CLIP, POISON_TOKEN, POISON_HEAD, POISON_CH = 2, 5, 1, 17
UNIFORM = {"simt_f16": (kp.ATTN_SIMT, F16), "simt_tf32": (kp.ATTN_SIMT, kp.KIND_TF32), "mma_tf32": (kp.ATTN_MMA_TF32, kp.KIND_TF32),
           "mma_f16": (kp.ATTN_MMA_F16, F16), "wgmma": (kp.ATTN_WGMMA, F16), "stream": (kp.ATTN_WGMMA_STREAM, F16)}


def _attend(dev, qkv, kind, which, B, S, clip_off=None, clip_ids=None):
    rows = qkv.shape[0]
    if kind == F16:
        hi, lo = kp.split(F16, qkv)
        cdt = torch.float16
    else:
        hi, lo, cdt = qkv, None, torch.float32
    ctx_hi = torch.full((rows, D), 7.0, dtype=cdt, device=dev)
    ctx_lo = torch.full((rows, D), 7.0, dtype=cdt, device=dev)
    rc = kp.attention(hi, lo, ctx_hi, ctx_lo, B, S, D, H, 1.0 / math.sqrt(DH), kind, which, clip_off=clip_off,
                      clip_ids=clip_ids)
    torch.cuda.synchronize()
    assert rc == 0, rc
    return ctx_hi, ctx_lo


def _poison_check(name, clean, bad, c0, c1, value):
    """Rows [c0, c1) are the poisoned clip: its poisoned context column is non-finite (NaN for a NaN V), every other element
    of the launch keeps its bits."""
    col = POISON_HEAD * DH + POISON_CH
    ch = kp.pair_value(*bad)[c0:c1, col]
    if math.isnan(value):
        assert bool(torch.isnan(ch).all()), f"{name}: NaN in V must give NaN context, got {ch[:4].tolist()}"
    else:
        assert not bool(torch.isfinite(ch).any()), f"{name}: {value} in V gave finite context values {ch[:4].tolist()}"
    keep = torch.ones_like(bad[0], dtype=torch.bool)
    keep[c0:c1, col] = False
    bits = torch.int16 if bad[0].dtype == torch.float16 else torch.int32
    for a, b in zip(clean, bad):
        assert torch.equal(a.view(bits)[keep], b.view(bits)[keep]), f"{name}: {value} in V changed other context bits"


@pytest.mark.parametrize("value", [math.inf, -math.inf, math.nan])
@pytest.mark.parametrize("name", list(UNIFORM))
def test_non_finite_v_reaches_the_context_in_every_kernel(dev, name, value):
    """One +inf, -inf or NaN V element of clip 2 (uniform clips of 64 tokens) makes that clip's context column non-finite
    in every kernel and stores it as a non-finite pair; the tensor-core kernels may turn inf into NaN through 0 x inf."""
    which, kind = UNIFORM[name]
    B, S = 4, 64
    g = torch.Generator().manual_seed(13)
    qkv = torch.randn(B * S + 5, 3 * D, generator=g)
    clean = _attend(dev, qkv.to(dev), kind, which, B, S)
    qkv[POISON_CLIP * S + POISON_TOKEN, 2 * D + POISON_HEAD * DH + POISON_CH] = value
    bad = _attend(dev, qkv.to(dev), kind, which, B, S)
    _poison_check(name, clean, bad, POISON_CLIP * S, (POISON_CLIP + 1) * S, value)


@pytest.mark.parametrize("value", [math.inf, -math.inf, math.nan])
@pytest.mark.parametrize("which", [kp.ATTN_WGMMA, kp.ATTN_WGMMA_STREAM])
def test_non_finite_v_reaches_the_context_on_packed_clips(dev, which, value):
    """The same on packed clips of different lengths, listed out of order."""
    tokens = [40, 17, 100, 64, 3]
    off = np.concatenate([[0], np.cumsum(tokens)]).tolist()
    g = torch.Generator().manual_seed(14)
    qkv = torch.randn(off[-1] + 5, 3 * D, generator=g)
    clip_off = torch.tensor(off, dtype=torch.int32, device=dev)
    ids = torch.tensor([3, 0, 2, 4, 1], dtype=torch.int32, device=dev)
    args = dict(clip_off=clip_off, clip_ids=ids)
    clean = _attend(dev, qkv.to(dev), F16, which, len(tokens), max(tokens), **args)
    qkv[off[POISON_CLIP] + POISON_TOKEN, 2 * D + POISON_HEAD * DH + POISON_CH] = value
    bad = _attend(dev, qkv.to(dev), F16, which, len(tokens), max(tokens), **args)
    _poison_check(f"packed {which}", clean, bad, off[POISON_CLIP], off[POISON_CLIP + 1], value)


# ---------------------------------------------------------------------------------------------------------------------------
# activation sweeps against float64
# ---------------------------------------------------------------------------------------------------------------------------
def _ulps(v, k):
    v = f32(v)
    out = [v]
    lo = hi = v
    for _ in range(k):
        lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
        out += [lo, hi]
    return out


SPECIAL = sorted({float(s) for v in (6.5, 20.0) for s in _ulps(v, 3)} | {1e4, 1e30})
SPECIAL = [f32(v) for v in SPECIAL] + [f32(-v) for v in SPECIAL] + [f32(math.inf), f32(-math.inf), f32(math.nan)]


def _sweep_operands():
    """Rows a_m: [-16, 16) in steps of 2^-5 and the pair-exact specials (6.5 and 20 a few ulp either side, 1e4); columns
    b_n: offsets n 2^-15 in [0, 2^-5) and the specials again as plain fp32 biases (with a_m = 0 they are x exactly)."""
    a = np.arange(-512, 512, dtype=f64) / 32.0
    a_sp = [v for v in SPECIAL if np.isfinite(v) and abs(v) < 2e4]
    a = np.concatenate([a, a_sp]).astype(f32)
    b = np.concatenate([np.arange(1024, dtype=f64) * 2.0 ** -15, SPECIAL]).astype(f32)
    b = np.concatenate([b, np.zeros(-len(b) % 4 + 4, dtype=f32)])  # N % 4 == 0, with a ragged 32-column tail
    with np.errstate(invalid="ignore", over="ignore"):
        x = a[:, None] + b[None, :]
    return a, b, x


def _act_ref(x, act):
    x = x.astype(f64)
    with np.errstate(invalid="ignore", over="ignore"):
        if act == kp.ACT_GELU:
            return x * ndtr(x)
        if act == kp.ACT_SILU:
            return x * expit(x)
        return x * np.tanh(np.logaddexp(0.0, x))


def _act_tol(x, ref, act):
    x = x.astype(f64)
    if act == kp.ACT_GELU:
        return 2.5e-7 + 2.0 ** -24 * np.abs(ref) + np.where(x < -6.5, 3.6e-11 * np.abs(x), 0.0)
    rel = 2.0 ** -21 if act == kp.ACT_SILU else 11 * 2.0 ** -24
    return rel * np.abs(ref) + 2.0 ** -118


def _check_act(x, got, act, what):
    x, got = x.ravel(), np.asarray(got, dtype=f32).ravel()
    fin = np.isfinite(x)
    assert (np.isnan(got[np.isnan(x)])).all(), f"{what}: NaN input gave a non-NaN output"
    assert not np.isfinite(got[np.isinf(x)]).any(), f"{what}: an infinite input gave a finite output"
    ref = _act_ref(x[fin], act)
    err = np.abs(got[fin].astype(f64) - ref)
    ratio = err / _act_tol(x[fin], ref, act)
    i = int(np.argmax(ratio))
    assert ratio[i] <= 1.0, (f"{what}: max |err| / bound = {ratio[i]:.3f} at x = {x[fin][i]!r} "
                             f"(got {got[fin][i]!r}, float64 {ref[i]!r})")


@pytest.mark.parametrize("act,general", [(kp.ACT_GELU, False), (kp.ACT_GELU, True), (kp.ACT_SILU, True),
                                         (kp.ACT_MISH, True)])
def test_epilogue_activation_sweep_against_float64(dev, act, general):
    """About 1.1M points through the lean (GELU) or the general epilogue (clip rows set), on the TMA-store and the dense /
    per-thread store paths, which must agree bit for bit; the identity epilogue first shows x arrives exactly."""
    a, b, x = _sweep_operands()
    M, N = x.shape
    A, W = _exact_gemm(dev, a, N, 128)
    seg = [A.seg(W.kblocks[0])]
    bias = torch.from_numpy(b).to(dev)
    clip = dict(clip_rows=M, clip_valid=M) if general else {}
    out = torch.empty(M, N, device=dev)
    assert kp.gemm(F16, W, seg, M, N, out=out, bias=bias)[0] == 0
    torch.cuda.synchronize()
    _same(_np(out), x, "identity epilogue: x = fp32(a + b)")
    outs = []
    for tma in (True, False):
        out = torch.full((M, N), 777.0, device=dev)
        rc, g = kp.gemm(F16, W, seg, M, N, out=out, bias=bias, act=act, tma_store=tma, **clip)
        assert rc == 0 and g.tma_store == int(tma)
        torch.cuda.synchronize()
        outs.append(out)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "TMA-store and per-thread stores differ"
    _check_act(x, _np(outs[0]), act, f"act {act} ({'general' if general else 'lean'} epilogue)")


def test_group_norm_mish_sweep_against_float64(dev):
    """gn_mish_split_kernel's mish_f over the same points: zero partials make every group's normalised value 0, so the
    kernel's Mish input is the channel's beta exactly (one row, 64 channels per group)."""
    _, _, x = _sweep_operands()
    x = x.ravel()
    C = -(-x.size // 64) * 64
    beta = np.zeros(C, dtype=f32)
    beta[:x.size] = x
    gen = torch.Generator().manual_seed(15)
    gamma = (1.0 + 0.2 * torch.randn(C, generator=gen)).to(dev)
    out = torch.full((C,), 777.0, device=dev)
    hi, lo = torch.empty(C, dtype=torch.float16, device=dev), torch.empty(C, dtype=torch.float16, device=dev)
    zeros = torch.zeros(C, device=dev)
    rc = kp.group_norm(zeros[None], 1, C, zeros, gamma, torch.from_numpy(beta).to(dev), None, 0, None, None, out, hi, lo, C,
                       1, 1, 1, 1, 1, groups=C // 64)
    torch.cuda.synchronize()
    assert rc == 0
    o = _np(out)
    _check_act(x, o[:x.size], kp.ACT_MISH, "GroupNorm mish_f")
    _pair_is_model(o, hi, lo, "GroupNorm pair store of the sweep")
