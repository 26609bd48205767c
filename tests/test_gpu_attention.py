"""The four attention kernels (rohm_b200/csrc/attention.cu) launched directly through tests/native/libkernel_probe.so and
compared with float64 softmax(scale Q K^T) V built from the hi + lo values the kernels read.

Every launch runs four clips of which clips 1 and 3 hold NaN in all their Q / K / V rows, and the row capacity past B * S
holds NaN too: a kernel must read nothing outside its clip.  The context buffer starts as a sentinel: every row of the
clips is written, nothing past B * S is.

Tolerance per output (i, d), relative to the output's natural scale sum_j p_ij |v_jd|:
    |got - ref| <= (C_OUT 2^-18 + 2 x 2^-20 L_i) sum_j p_ij |v_jd|,   L_i = scale max_j sum_k |q_ik| |k_jk|
The first term covers the hi/lo split of P and of the context and the fp32 softmax; the second the error of the logits,
which the exponential turns into a relative error of p (2^-20 per |q| |k| product, the three-product bound of the GEMM)."""
import math

import pytest
import torch

import kernel_probe as kp

pytestmark = pytest.mark.gpu

F16, TF32 = kp.KIND_F16, kp.KIND_TF32
C_OUT = 4.0
B, D = 4, 512
POISONED = (1, 3)
SENTINEL = 60000.0  # exact in fp16, and above every |output| of these inputs (|v| <= 1e4)
S_TC = [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 144, 145, 159, 160]
S_SIMT = [161, 200, 256]
# name: (kernel, operand kind, head dims it serves)
KERNELS = {"wgmma": (kp.ATTN_WGMMA, F16, (128,)), "mma_f16": (kp.ATTN_MMA_F16, F16, (128, 64)),
           "mma_tf32": (kp.ATTN_MMA_TF32, TF32, (128, 64)), "simt_f16": (kp.ATTN_SIMT, F16, (128, 64)),
           "simt_tf32": (kp.ATTN_SIMT, TF32, (128, 64))}
REGIMES = ["flat", "sharp_last", "sharp_first", "identical", "big_v"]


@pytest.fixture(scope="module")
def dev(cuda_device):
    kp.lib()  # a missing probe library fails every test of the module
    return cuda_device


def _qkv(S, dh, regime, seed):
    """fp32 Q, K, V [B, S, H, dh] of a logit regime (CPU, seeded)."""
    H = D // dh
    g = torch.Generator().manual_seed(seed)
    scale = 1.0 / math.sqrt(dh)
    q = torch.randn(B, S, H, dh, generator=g)
    k = torch.randn(B, S, H, dh, generator=g)
    v = torch.randn(B, S, H, dh, generator=g)
    if regime.startswith("sharp"):
        # near one-hot rows: logits of the target key about 80 after scaling, the others spread around 0
        t = S - 1 if regime == "sharp_last" else 0
        kt = k[:, t:t + 1]
        beta = 80.0 / (scale * (kt * kt).sum(-1, keepdim=True))
        q = beta * kt + 0.3 * q
    elif regime == "identical":
        k = k[:, :1].expand(B, S, H, dh).clone()
    elif regime == "big_v":
        v = (torch.rand(B, S, H, dh, generator=g) * 2.0 - 1.0) * 1e4
    return q, k, v, scale


def _launch(dev, which, kind, S, dh, regime, seed):
    H = D // dh
    q, k, v, scale = _qkv(S, dh, regime, seed)
    rows = B * S + 37
    qkv = torch.full((rows, 3 * D), float("nan"))
    qkv[:B * S] = torch.cat([t.reshape(B * S, D) for t in (q, k, v)], dim=1)
    for b in POISONED:
        qkv[b * S:(b + 1) * S] = float("nan")
    qkv = qkv.to(dev)
    if kind == F16:
        hi, lo = kp.split(F16, qkv)
        planes = torch.stack([hi, lo])  # one buffer, as the engine keeps them
        planes[:, B * S:] = float("nan")
        for b in POISONED:
            planes[:, b * S:(b + 1) * S] = float("nan")
        qkv_hi, qkv_lo = planes[0], planes[1]
        value = kp.pair_value(qkv_hi, qkv_lo)
        cdt = torch.float16
    else:
        qkv_hi, qkv_lo, value, cdt = qkv, None, qkv.double(), torch.float32
    ctx_hi = torch.full((rows, D), SENTINEL, dtype=cdt, device=dev)
    ctx_lo = torch.full((rows, D), SENTINEL, dtype=cdt, device=dev)
    rc = kp.attention(qkv_hi, qkv_lo, ctx_hi, ctx_lo, B, S, D, H, scale, kind, which)
    torch.cuda.synchronize()
    return rc, value, ctx_hi, ctx_lo, scale


def _reference(value, S, dh, scale):
    H = D // dh
    x = value[:B * S].reshape(B, S, 3, H, dh)
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    logits = scale * torch.einsum("bihd,bjhd->bhij", q, k)
    p = torch.softmax(logits, dim=-1)
    o = torch.einsum("bhij,bjhd->bihd", p, v)
    scale_o = torch.einsum("bhij,bjhd->bihd", p, v.abs())
    L = scale * torch.einsum("bihd,bjhd->bhij", q.abs(), k.abs()).amax(-1)  # [B, H, S]
    tol = (C_OUT * 2.0 ** -18 + 2.0 * 2.0 ** -20 * L.permute(0, 2, 1)[..., None]) * scale_o
    return o.reshape(B, S, D), tol.reshape(B, S, D)


def _split_ok(hi, lo):
    """The stored context pair is a proper split: hi carries the value to its own precision, |lo| <= half an ulp of hi."""
    h = hi.float()
    _, e = torch.frexp(h)
    bits = 11  # significant bits of fp16 and of TF32
    half_ulp = torch.where(h == 0, torch.full_like(h, 2.0 ** -25), torch.ldexp(torch.ones_like(h), e - bits - 1))
    ok = lo.float().abs() <= half_ulp * (1.0 + 2.0 ** -10)
    if hi.dtype == torch.float32:
        ok &= (hi.view(torch.int32) & 0x1FFF) == 0
    return bool(ok.all())


def _check(dev, name, S, dh, regime):
    which, kind, _ = KERNELS[name]
    seed = 1000 * S + dh + REGIMES.index(regime)
    rc, value, ctx_hi, ctx_lo, scale = _launch(dev, which, kind, S, dh, regime, seed)
    assert rc == 0, (name, S, dh, rc)
    # only the clips' rows are written
    assert bool((ctx_hi[B * S:] == SENTINEL).all()) and bool((ctx_lo[B * S:] == SENTINEL).all()), "wrote past B * S"
    got = kp.pair_value(ctx_hi, ctx_lo)[:B * S].reshape(B, S, D)
    written = (ctx_hi[:B * S] != SENTINEL).reshape(B, S, D)
    assert bool(written.all()), "a row of the clips was not written"
    ref, tol = _reference(value, S, dh, scale)
    good = [b for b in range(B) if b not in POISONED]
    for b in good:
        assert bool(torch.isfinite(got[b]).all()), f"NaN from another clip leaked into clip {b} (S={S})"
        ratio = float(((got[b] - ref[b]).abs() / tol[b]).max())
        assert ratio <= 1.0, f"{name} S={S} dh={dh} {regime}: clip {b} max |err| / bound = {ratio:.3f}"
    rows = torch.cat([torch.arange(b * S, (b + 1) * S) for b in good]).to(dev)
    assert _split_ok(ctx_hi[rows], ctx_lo[rows]), "context hi/lo split"


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name,dh", [("wgmma", 128), ("mma_f16", 128), ("mma_f16", 64), ("mma_tf32", 128),
                                     ("mma_tf32", 64)])
def test_tensor_core_kernels_against_float64(dev, name, dh, regime):
    for S in S_TC:
        _check(dev, name, S, dh, regime)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name", ["simt_f16", "simt_tf32"])
def test_simt_kernel_against_float64(dev, name, regime):
    """The SIMT kernel serves clips of more than 160 tokens (and is correct on short ones too); head dim 128 up to the
    shared memory limit (about 210 tokens), head dim 64 up to 256."""
    for S in [1, 17, 160] + S_SIMT:
        for dh in (64, 128):
            if dh == 128 and S > 200:
                continue
            _check(dev, name, S, dh, regime)


def test_kernels_outside_their_domain_are_refused(dev):
    """A forced kernel that cannot run the launch returns cudaErrorInvalidValue without launching."""
    cases = [("wgmma", 64, 64), ("wgmma", 161, 128), ("mma_f16", 161, 128), ("mma_tf32", 161, 64), ("simt_f16", 256, 128)]
    for name, S, dh in cases:
        which, kind, _ = KERNELS[name]
        rc, _, ctx_hi, ctx_lo, _ = _launch(dev, which, kind, S, dh, "flat", 5)
        assert rc == kp.CUDA_ERROR_INVALID_VALUE, (name, S, dh, rc)
        assert bool((ctx_hi == SENTINEL).all()) and bool((ctx_lo == SENTINEL).all())
    # the kernel kinds: an fp16 kernel on fp32 Q|K|V and the reverse
    for name, kind in (("wgmma", TF32), ("mma_f16", TF32), ("mma_tf32", F16)):
        which = KERNELS[name][0]
        rc, _, _, _, _ = _launch(dev, which, kind, 16, 128, "flat", 6)
        assert rc == kp.CUDA_ERROR_INVALID_VALUE, (name, kind, rc)


@pytest.mark.parametrize("kind", [F16, TF32])
def test_automatic_choice_matches_the_forced_kernel(dev, kind):
    """kAttnAuto takes the wgmma kernel (fp16 pairs, head dim 128, <= 160 tokens), else the mma.sync kernel of the kind,
    else the SIMT kernel: bit-identical to forcing that kernel."""
    for S, dh in ((145, 128), (145, 64), (200, 64)):
        if S > 160:
            forced = kp.ATTN_SIMT
        elif kind == F16:
            forced = kp.ATTN_WGMMA if dh == 128 else kp.ATTN_MMA_F16
        else:
            forced = kp.ATTN_MMA_TF32
        outs = []
        for which in (kp.ATTN_AUTO, forced):
            rc, _, hi, lo, _ = _launch(dev, which, kind, S, dh, "flat", 9)
            assert rc == 0
            outs.append((hi, lo))
        bits = torch.int16 if kind == F16 else torch.int32  # bit patterns: the poisoned clips' NaN rows compare too
        assert all(torch.equal(a.view(bits), b.view(bits)) for a, b in zip(outs[0], outs[1])), (S, dh)
