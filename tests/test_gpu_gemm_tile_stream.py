"""Long tile sequences per CTA through the lean GEMM variants (rohm_b200/csrc/gemm.cu, EPI 0 / 1 / 3), whose MMA and
epilogue warpgroups hand every accumulator tile over through acc_full / acc_empty mbarriers.  At M = 16384 (128 row
stripes) a CTA runs 11-12 QKV tiles, 7-8 FFN1 tiles and 4 LayerNorm-producer tiles, so both barriers flip phase over odd
and even counts; M = 16384 + 32 adds a ragged last stripe.  Launched through tests/native/libkernel_probe.so and compared
with float64 on a seeded subset of rows, with the bounds of test_gpu_gemm.py; two launches must agree bit for bit."""
import math

import pytest
import torch

import kernel_probe as kp

pytestmark = pytest.mark.gpu

F16 = kp.KIND_F16
D, K = 512, 512


@pytest.fixture(scope="module")
def dev(cuda_device):
    kp.lib()
    return cuda_device


def _randn(shape, seed, dev, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(dev)


def _rows(M, seed):
    r = torch.randperm(M, generator=torch.Generator().manual_seed(seed))[:384]
    return torch.unique(torch.cat([r, torch.arange(M - 40, M), torch.tensor([0])]))


def _check(got, ref, tol, what):
    got = got.double()
    assert bool(torch.isfinite(got).all()), what
    ratio = float(((got - ref).abs() / tol).max())
    assert ratio <= 1.0, f"{what}: max |err| / bound = {ratio:.3f}"


def _folded(W, gam, bet, b):
    """A LayerNorm consumer's weight with gamma folded in, its c_n and d_n (GemmParams::a_stats)."""
    Wf = (gam[None, :] * W).contiguous()
    return Wf, Wf.double().sum(1).float(), (b.double() + W.double() @ bet.double()).float()


def _producer(dev, M, A, W, b, R):
    """u = R + A W^T + b, written in place over the fp16 pair of R; returns (pair, stats)."""
    Xh, Xl = kp.split(F16, R)
    S = torch.zeros(M, 16, device=dev)
    rc, g = kp.gemm(F16, W, [A.seg(W.kblocks[0])], M, D, out_hi=Xh, out_lo=Xl, bias=b, stats_out=S, tma_store=True)
    assert rc == 0 and g.tma_store == 1
    return Xh, Xl, S


def _ln(u, gam, bet):
    mean = u.mean(1, keepdim=True)
    var = ((u - mean) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    return (u - mean) * rstd * gam.double() + bet.double(), mean, rstd


@pytest.mark.parametrize("M", [16384, 16384 + 32])
def test_long_tile_streams_match_float64_and_repeat_bitwise(dev, M):
    """EPI 3 producer (u1 = R + A1 W1^T + b1) -> EPI 0 LayerNorm consumer QKV (N = 1536, fp16 pair out) and EPI 1
    consumer FFN1 (N = 1024, exact GELU, fp32 out) -> EPI 3 producer with the residual normalised on the fly."""
    A1 = kp.Operand(F16, _randn((M, K), 300, dev))
    A3 = kp.Operand(F16, _randn((M, K), 301, dev))
    W1 = kp.Weight(F16, [_randn((D, K), 302, dev, 1.0 / math.sqrt(K))], 128)
    W3 = kp.Weight(F16, [_randn((D, K), 303, dev, 1.0 / math.sqrt(K))], 128)
    Wq, Wf = _randn((1536, D), 304, dev, 1.0 / math.sqrt(D)), _randn((1024, D), 305, dev, 1.0 / math.sqrt(D))
    b1, b3, bq, bf = _randn((D,), 306, dev), _randn((D,), 307, dev), _randn((1536,), 308, dev), _randn((1024,), 309, dev)
    gam, bet = _randn((D,), 310, dev, 0.1) + 1.0, _randn((D,), 311, dev, 0.1)
    R = _randn((M, D), 312, dev, 1.5) + 0.7
    Wqf, cq, dq = _folded(Wq, gam, bet, bq)
    Wff, cf, df = _folded(Wf, gam, bet, bf)
    WqP, WfP = kp.Weight(F16, [Wqf], 128), kp.Weight(F16, [Wff], 128)

    runs = []
    for _ in range(2):
        Xh, Xl, S1 = _producer(dev, M, A1, W1, b1, R)
        X = kp.Operand(F16, torch.zeros(1, D, device=dev))
        X.hi, X.lo, X.rows = Xh, Xl, M  # the consumers read the stored pair in place
        Qh, Ql = torch.empty(M, 1536, dtype=torch.float16, device=dev), torch.empty(M, 1536, dtype=torch.float16, device=dev)
        rc, g = kp.gemm(F16, WqP, [X.seg(WqP.kblocks[0])], M, 1536, out_hi=Qh, out_lo=Ql, bias=dq, a_stats=S1, a_corr=cq,
                        tma_store=True)
        assert rc == 0 and g.tma_store == 1
        Y = torch.empty(M, 1024, device=dev)
        rc, g = kp.gemm(F16, WfP, [X.seg(WfP.kblocks[0])], M, 1024, out=Y, bias=df, a_stats=S1, a_corr=cf,
                        act=kp.ACT_GELU, tma_store=True)
        assert rc == 0 and g.tma_store == 1
        u1g = kp.pair_value(Xh, Xl)
        Uh, Ul, S2 = Xh.clone(), Xl.clone(), torch.zeros(M, 16, device=dev)  # (C) overwrites its residual u1 in place
        rc, g = kp.gemm(F16, W3, [A3.seg(W3.kblocks[0])], M, D, out_hi=Uh, out_lo=Ul, bias=b3, stats_out=S2, res_stats=S1,
                        res_gamma=gam, res_beta=bet, tma_store=True)
        assert rc == 0
        torch.cuda.synchronize()
        runs.append((u1g, S1, Qh, Ql, Y, Uh, Ul, S2))
    for a, b in zip(*runs):
        assert torch.equal(a, b), "two launches differ"

    u1g, S1, Qh, Ql, Y, Uh, Ul, S2 = runs[0]
    rows = _rows(M, 17).to(dev)
    Rv = kp.pair_value(*kp.split(F16, R))[rows]
    a1, a3 = A1.value[rows], A3.value[rows]
    w1, w3 = W1.parts[0], W3.parts[0]
    u1 = a1 @ w1.T + b1.double() + Rv
    aw1 = a1.abs() @ w1.abs().T + b1.double().abs() + Rv.abs()
    u1s = u1g[rows]
    _check(u1s, u1, 2.0 * 2.0 ** -20 * aw1 + 2.0 ** -21 * u1.abs() + 2.0 ** -24, "EPI 3 producer")
    x, mean, rstd = _ln(u1s, gam, bet)
    for name, W, Wfold, c, b, got, act in (("EPI 0 QKV", Wq, Wqf, cq, bq, kp.pair_value(Qh, Ql)[rows], False),
                                           ("EPI 1 FFN1", Wf, Wff, cf, bf, Y[rows], True)):
        y = x @ W.double().T + b.double()
        ayw = rstd * (u1s.abs() @ Wfold.double().abs().T + mean.abs() * c.double().abs()[None, :]) + x.abs() @ W.double().abs().T
        tol = 4.0 * 2.0 ** -20 * ayw + 2.0 ** -23 * y.abs() + 1e-7
        if act:
            y = 0.5 * y * (1.0 + torch.erf(y / math.sqrt(2.0)))
            tol = 1.25 * tol + 2.0 ** -21 * (1.0 + y.abs())
        else:
            tol = tol + 2.0 ** -21 * y.abs() + 2.0 ** -25
        _check(got, y, tol, name)
    u2 = x + a3 @ w3.T + b3.double()
    aw3 = x.abs() + a3.abs() @ w3.abs().T + b3.double().abs()
    _check(kp.pair_value(Uh, Ul)[rows], u2, 4.0 * 2.0 ** -20 * aw3 + 2.0 ** -21 * u2.abs() + 2.0 ** -24,
           "EPI 3 producer, residual through LayerNorm")
