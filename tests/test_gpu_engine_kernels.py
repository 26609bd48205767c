"""GPU: the denoiser engines' small kernels (rohm_b200/csrc/engine_kernels.cu) through the kernel probe, against float64
and bit-level references at their edges.

* layernorm_kernel<D> (PoseNet's LayerNorm in the tf32 precisions and without LayerNorm folding) for every d_model it is
  instantiated for.
* fold_ln_kernel: the gamma-folded weight and the c / d vectors of the folded-LayerNorm GEMM epilogue.
* trajnet_time_kernel: TrajNet's time path, evaluated directly and gathered from the table the kernel builds.
* sum_split_kernel: bias plus the split-K partials of the downsampling convolutions, uniform and packed clips.

Every launch writes into sentinel-filled buffers longer than its output; nothing past the output may change, and a
repeated launch must give the same bits.  Each float64 comparison prints its worst error / bound ratio."""
import math

import numpy as np
import pytest
import torch

import kernel_probe as kp
from arith_model import split_f16, split_tf32
from rohm_b200 import synthetic
from rohm_b200.trajnet import TrajNet

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # fp32 unit roundoff
UD = 2.0 ** -53  # float64 unit roundoff
SENTINEL = 1234.0  # exact in fp16 too
EXTRA = 64  # elements past every output that must keep the sentinel


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _launch_twice(shapes, launch):
    """Runs launch(*buffers) on two fresh sets of sentinel-filled buffers, each (n, dtype) of n + EXTRA elements.  Asserts
    that the launch returned 0, left the EXTRA elements alone and that both runs gave the same bits; returns the first
    run's buffers cut to their n elements."""
    runs = []
    for _ in range(2):
        bufs = [torch.full((n + EXTRA,), SENTINEL, dtype=dt, device="cuda") for n, dt in shapes]
        rc = launch(*bufs)
        torch.cuda.synchronize()
        assert rc == 0, rc
        for (n, _), b in zip(shapes, bufs):
            assert bool((b[n:].float() == SENTINEL).all()), "wrote past the output"
        runs.append(bufs)
    for a, b in zip(*runs):
        assert torch.equal(_bits(a), _bits(b)), "a repeated launch changed bits"
    return [b[:n] for (n, _), b in zip(shapes, runs[0])]


def _assert_pair_model(out, hi, lo, f16):
    """hi / lo are the arith_model split of the fp32 `out`, bit for bit (float32 values of the halves for fp16)."""
    h, l = (split_f16 if f16 else split_tf32)(out.cpu().numpy())
    for got, want in ((hi, h), (lo, l)):
        got = got.float().cpu().numpy()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "operand pair differs from the model"


def _mish(x):
    return x * torch.tanh(torch.nn.functional.softplus(x))


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
def _ln_reference(x, gamma, beta, D):
    """float64 LayerNorm (eps 1e-5) of the fp32 rows x (= fl(in + res), as torch adds them) and the per-element bound of
    the kernel's fp32 arithmetic.

    Derivation (u = 2^-24; k = D / 128 + 7, the depth of the kernel's sum: pairs within a float4, D / 128 float4s per lane,
    5 shuffle levels):
      mean: fp32 sum of D terms, |dsum| <= k u sum|x|; times 1/D (exact) and rounded: dm <= k u mean|x| + u |mean|
      a = x - mean (fp32):   |da| <= dm + u |a|
      sq = sum a^2 (fp32):   a square and k adds per term, and dm shifts every a (their sum is ~0): sq (k + 3) u + D dm^2
      v = sq / D + eps:      two more roundings, and 1e-5f differs from 1e-5 by < u eps: dv <= var (k + 5) u + dm^2 + u eps
      rstd = rsqrtf(v):      2 ulp (4 u) plus half the relative error of v: drel = 4 u + dv / (2 v)
      y = a rstd gamma + beta (two products and a sum): |dy| <= |gamma| rstd (|a| (drel + 2 u) + |da|) + u |y|
    The bound is twice that sum, for the terms second order in u."""
    x = x.double()
    g, b = gamma.double().view(1, D), beta.double().view(1, D)
    k = D // 128 + 7
    mean = x.mean(dim=1, keepdim=True)
    a = x - mean
    var = (a * a).mean(dim=1, keepdim=True)
    v = var + 1e-5
    rstd = 1.0 / torch.sqrt(v)
    y = a * rstd * g + b
    dm = k * U * x.abs().mean(dim=1, keepdim=True) + U * mean.abs()
    da = dm + U * a.abs()
    dv = var * (k + 5) * U + dm * dm + U * 1e-5
    drel = 4 * U + dv / (2 * v)
    bound = 2 * (g.abs() * rstd * (a.abs() * (drel + 2 * U) + da) + U * y.abs())
    return y, bound


def _ln_rows(D, gen):
    """in, res [rows, D] fp32 (CPU) with the row kinds the kernel must get right, 42 rows (not a multiple of the 8 rows of
    one CTA): 0-12 random, 13-20 |mean| >> std (mean 1e3, std 0.1), 21-28 variance near eps (std 3e-3), 29-41 constant
    (in + res = c exactly, so every sum the kernel forms is exact and the output must be beta)."""
    rnd = lambda *s: torch.randn(*s, generator=gen)
    res = rnd(42, D)
    x = torch.cat([2.0 * rnd(13, D) + 0.3,
                   1e3 + 0.1 * rnd(8, D),
                   -0.7 + 3e-3 * rnd(8, D)])
    consts = torch.tensor([0.0, 1.5, -3.25, 1000.0, 0.125, -7.0, 2.0, -0.5, 96.0, 0.75, -1024.0, 5.5, 3.0])
    inp = torch.cat([x - res[:29], consts.view(-1, 1) - 0.5 + torch.zeros(13, D)])
    res[29:] = 0.5
    return inp, res


def _ln_launch(D, x, res, gamma, beta, rows, f16, alias=False):
    """layernorm_kernel<D> of x + res (res None: x alone; alias: res passed as the output buffer, as the engine does)."""
    dt = torch.float16 if f16 else torch.float32
    n = rows * D

    def launch(out, hi, lo):
        if alias:
            out[:n] = res.reshape(-1)
        return kp.layernorm(D, x, out if alias else res, gamma, beta, out, hi, lo, rows, f16)

    return [t.view(rows, D) for t in _launch_twice([(n, torch.float32), (n, dt), (n, dt)], launch)]


@pytest.mark.parametrize("D", [128, 256, 512, 1024])
def test_layernorm_matches_float64(cuda_device, D):
    """layernorm_kernel<D> with fp16 and tf32 pairs, with the residual, without it and with the output aliasing it: the
    fp32 output within the derived bound of a float64 LayerNorm of fl(in + res), constant rows exactly beta, the pair the
    arith_model split of the fp32 output bit for bit, and the aliased launch bit-identical to the plain one."""
    gen = torch.Generator().manual_seed(D)
    inp, res = _ln_rows(D, gen)
    rows = inp.shape[0]
    gamma = (1.0 + 0.3 * torch.randn(D, generator=gen)).to(cuda_device)
    beta = (0.2 * torch.randn(D, generator=gen)).to(cuda_device)
    inp, res = inp.to(cuda_device).contiguous(), res.to(cuda_device).contiguous()
    worst = 0.0
    for f16 in (1, 0):
        for with_res in (True, False):
            out, hi, lo = _ln_launch(D, inp, res if with_res else None, gamma, beta, rows, f16)
            x = inp + res if with_res else inp  # torch's fp32 add, the kernel's first step
            ref, bound = _ln_reference(x, gamma, beta, D)
            err = (out.double() - ref).abs()
            assert bool((err <= bound).all()), (f16, with_res, float(err.max()), float((err / bound).max()))
            worst = max(worst, float((err / bound).max()))
            # rows 29-41 are constant either way (c, or c - 0.5 without the residual), and every sum of them is exact
            assert torch.equal(out[29:], beta.view(1, D).expand(13, D)), "a constant row must give beta"
            _assert_pair_model(out, hi, lo, f16)
            if with_res:
                aliased = _ln_launch(D, inp, res, gamma, beta, rows, f16, alias=True)
                for a, b in zip(aliased, (out, hi, lo)):
                    assert torch.equal(_bits(a), _bits(b)), "out aliasing res changed the result"
    print(f"LayerNorm D={D}: worst error / bound = {worst:.3f}")


@pytest.mark.parametrize("D", [128, 1024])
@pytest.mark.parametrize("rows", [1, 7, 13])
def test_layernorm_nan_row_stays_in_its_row(cuda_device, D, rows):
    """A NaN in one row makes that row NaN in every output; every other row, in the same CTA or not, keeps its bits."""
    gen = torch.Generator().manual_seed(rows * D)
    x = torch.randn(rows, D, generator=gen).to(cuda_device)
    res = torch.randn(rows, D, generator=gen).to(cuda_device)
    gamma = (1.0 + 0.3 * torch.randn(D, generator=gen)).to(cuda_device)
    beta = (0.2 * torch.randn(D, generator=gen)).to(cuda_device)
    r = rows // 2
    bad = x.clone()
    bad[r, D // 3] = float("nan")
    for f16 in (1, 0):
        clean = _ln_launch(D, x, res, gamma, beta, rows, f16)
        poisoned = _ln_launch(D, bad, res, gamma, beta, rows, f16)
        keep = torch.arange(rows, device=cuda_device) != r
        for c, p in zip(clean, poisoned):
            assert bool(torch.isnan(p[r].float()).all()), "the NaN row must be NaN throughout"
            assert torch.equal(_bits(c[keep]), _bits(p[keep])), "a NaN leaked into another row"


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm folding
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [512, 1024, 700, 200])
def test_fold_ln_matches_float64(cuda_device, K):
    """fold_ln_kernel on a [N, K] weight: Wf is torch's fp32 gamma * W bit for bit; c and d are within the bound of the
    float64 sums.

    Derivation (u = 2^-24, ud = 2^-53): each thread adds ceil(K / 256) terms in double, the 256 thread sums meet in an
    8-level tree, so |d sum| <= (ceil(K / 256) + 8) ud sum|term|; the products beta_k w are exact in double, d adds the
    bias (one more ud) and each result is rounded to fp32 (u |result|).  The float64 reference sums err by up to
    K ud sum|term| themselves.  The bound is twice u |ref| + (ceil(K / 256) + 9 + K) ud sum|term|."""
    gen = torch.Generator().manual_seed(K)
    N = 100
    rnd = lambda *s: torch.randn(*s, generator=gen).to(cuda_device)
    W, gamma, beta, bias = 0.05 * rnd(N, K), 1.0 + 0.2 * rnd(K), 0.3 * rnd(K), 0.1 * rnd(N)
    Wf, c, d = _launch_twice([(N * K, torch.float32), (N, torch.float32), (N, torch.float32)],
                             lambda Wf, c, d: kp.fold_ln(W, gamma, beta, bias, Wf, c, d))
    assert torch.equal(_bits(Wf.view(N, K)), _bits(gamma.view(1, K) * W)), "Wf must be torch's gamma * W"
    g = (math.ceil(K / 256) + 9 + K) * UD
    terms_c = Wf.view(N, K).double()
    terms_d = beta.double().view(1, K) * W.double()
    c_ref, d_ref = terms_c.sum(dim=1), bias.double() + terms_d.sum(dim=1)
    bc = 2 * (U * c_ref.abs() + g * terms_c.abs().sum(dim=1))
    bd = 2 * (U * d_ref.abs() + g * (bias.double().abs() + terms_d.abs().sum(dim=1)))
    worst = 0.0
    for got, ref, bound in ((c, c_ref, bc), (d, d_ref, bd)):
        err = (got.double() - ref).abs()
        assert bool((err <= bound).all()), (float(err.max()), float((err / bound).max()))
        worst = max(worst, float((err / bound).max()))
    print(f"fold_ln K={K}: worst error / bound = {worst:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# TrajNet time path
# ---------------------------------------------------------------------------------------------------------------------
TIME_DIM = 32
TABLE_ROWS = 1024  # trajnet.cu kTimeTableRows
TIMESTEPS = [0, 1, 2, 499, 998, 999, 1023, 1024, 1025, 4999, -1]


@pytest.fixture(scope="module")
def time_weights(cuda_device):
    """The time MLP and the stacked per-block time projections of the mid_dim 512 TrajNet + TrajControl, stacked as
    rohm_trajnet_create stacks them (every block with a time projection, its Linear(32, Cout) rows one after another)."""
    m = TrajNet(time_dim=TIME_DIM, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=True,
                device=torch.device("cpu"), dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
    sd = synthetic.synth_state_dict(m, 2)
    blocks = [k[:-len("time_mlp.1.weight")] for k in sd
              if k.endswith("time_mlp.1.weight") and k[:-len("1.weight")] + "3.weight" not in sd]
    w = {"w1": sd["time_mlp.1.weight"], "b1": sd["time_mlp.1.bias"], "w3": sd["time_mlp.3.weight"],
         "b3": sd["time_mlp.3.bias"], "wcat": torch.cat([sd[p + "time_mlp.1.weight"] for p in blocks]),
         "bcat": torch.cat([sd[p + "time_mlp.1.bias"] for p in blocks])}
    assert w["wcat"].shape[1] == TIME_DIM and w["bcat"].numel() % 4 == 0
    return {k: v.float().contiguous().to(cuda_device) for k, v in w.items()}


def _time_reference(t, w):
    """float64 time path of the int64 timesteps t and the per-element bound of the kernel's fp32 arithmetic.

    The sinusoid argument is the fp32 product t * f torch forms (oracle.trajnet_oracle.sinusoidal_pos_emb), f_j =
    exp(-j ln(1e4) / 15) in fp32.  Derivation (u = 2^-24, x_j = j ln(1e4) / 15):
      f:      the kernel's fp32 logf / division / product (4 u |x|) and expf (2 ulp) against torch's cast / product (2 u |x|)
              and exp (1 ulp): |df| <= f (8 u x_j + 8 u)
      arg a:  |da| <= |t| |df| + 2 u |a| (the two products' roundings)
      e:      sinf / cosf, 2 ulp: |de| <= |da| + 4 u |e|
      h = mish(W1 e + b1): an fmaf chain of K = 32 terms, K u (|b1| + sum |w1| |e|), plus sum |w1| |de|; mish: |mish'| <=
              1.1, and its fp32 evaluation adds <= 8 u |mish| + 4 u
      m = mish(W3 h + b3): the same with K = 128
      tp = Wcat m + bcat: K = 32 chain, sum |wcat| |dm| + K u (|bcat| + sum |wcat| |m|)
    The bound is twice that, for the terms second order in u."""
    half = TIME_DIM // 2
    f = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
    a = t.cpu().to(torch.float32)[:, None] * f[None, :]
    xj = torch.arange(half, dtype=torch.float64) * (math.log(10000) / (half - 1))
    df = f.double() * (8 * U * xj + 8 * U)
    da = t.cpu().double().abs()[:, None] * df[None, :] + 2 * U * a.double().abs()
    a = a.double()
    e = torch.cat([a.sin(), a.cos()], dim=1)
    de = torch.cat([da, da], dim=1) + 4 * U * e.abs()
    w = {k: v.double().cpu() for k, v in w.items()}

    def linear(x, dx, W, b):
        y = x @ W.T + b
        dy = dx @ W.abs().T + W.shape[1] * U * (b.abs() + x.abs() @ W.abs().T)
        return y, dy

    def mish(y, dy):
        m = _mish(y)
        return m, 1.1 * dy + 8 * U * m.abs() + 4 * U

    h, dh = mish(*linear(e, de, w["w1"], w["b1"]))
    m, dm = mish(*linear(h, dh, w["w3"], w["b3"]))
    tp, dtp = linear(m, dm, w["wcat"], w["bcat"])
    return tp, 2 * dtp


def _time_launch(w, t, ctas, table=None):
    total = w["bcat"].numel()
    (tp,) = _launch_twice([(t.numel() * total, torch.float32)],
                          lambda tp: kp.trajnet_time(t, ctas, TIME_DIM, w["w1"], w["b1"], w["w3"], w["b3"], w["wcat"],
                                                     w["bcat"], tp, table, TABLE_ROWS if table is not None else 0))
    return tp.view(t.numel(), total)


def test_trajnet_time_direct_matches_float64(cuda_device, time_weights):
    """The direct evaluation (no table) at timesteps inside, at the edges of and outside the table, against the float64
    SinusoidalPosEmb -> Linear -> Mish -> Linear -> Mish -> stacked projections, within the derived bound; one and eight
    CTAs per clip give the same bits."""
    t = torch.tensor(TIMESTEPS, dtype=torch.int64, device=cuda_device)
    got = _time_launch(time_weights, t, 8)
    assert torch.equal(_bits(_time_launch(time_weights, t, 1)), _bits(got)), "gridDim.y changed the bits"
    ref, bound = _time_reference(t, time_weights)
    err = (got.double().cpu() - ref).abs()
    for i, ti in enumerate(TIMESTEPS):
        assert bool((err[i] <= bound[i]).all()), (ti, float(err[i].max()), float((err[i] / bound[i]).max()))
    print(f"TrajNet time path: worst error / bound = {float((err / bound).max()):.3f}")


def test_trajnet_time_table_gather_equals_direct(cuda_device, time_weights):
    """The table built by the kernel itself for t = 0 .. 1023 (as rohm_trajnet_create builds it, eight CTAs per row):
    a gather for every t < 1024 equals the direct evaluation bit for bit, and t outside [0, 1024) takes the direct
    evaluation although a table is passed; with one and with eight CTAs per clip."""
    all_t = torch.arange(TABLE_ROWS, dtype=torch.int64, device=cuda_device)
    table = _time_launch(time_weights, all_t, 8)
    t = torch.tensor(TIMESTEPS + list(range(0, TABLE_ROWS, 37)), dtype=torch.int64, device=cuda_device)
    direct = _time_launch(time_weights, t, 8)
    inside = (t >= 0) & (t < TABLE_ROWS)
    assert torch.equal(_bits(direct[inside]), _bits(table[t[inside]])), "table row differs from the direct evaluation"
    for ctas in (1, 8):
        gathered = _time_launch(time_weights, t, ctas, table)
        assert torch.equal(_bits(gathered), _bits(direct)), ctas


# ---------------------------------------------------------------------------------------------------------------------
# Split-K sum
# ---------------------------------------------------------------------------------------------------------------------
LEVEL_C = [64, 128, 256, 512, 512]  # output channels of a level's rows (any multiple of 4 serves)


def _split_layout(packed, L):
    """(rows, Tp, T, real-row mask) of a level-L activation: packed clips of 16, 32 and 4992 frames, each taking
    (n + 32) >> L rows with its n >> L real rows first; or two uniform clips of 144 frames."""
    if packed:
        lengths = [16, 4992, 32]
        mask = torch.cat([torch.arange((n + 32) >> L) < (n >> L) for n in lengths])
        T = max(lengths)
    else:
        T = 144
        mask = (torch.arange((T + 32) >> L) < (T >> L)).repeat(2)
    return mask.numel(), (T + 32) >> L, T >> L, mask


@pytest.mark.parametrize("splits", [1, 2, 3, 8])
@pytest.mark.parametrize("packed", [False, True])
def test_sum_split_is_torchs_sum_in_split_order(cuda_device, splits, packed):
    """At every pyramid level, fp16 and tf32 pairs, with the fp32 output and / or the pair: real rows are torch's fp32
    ((bias + p0) + p1) + ... bit for bit, pad rows +0.0 in every form (their partials hold NaN, which must not be read),
    and the pair is the arith_model split of the fp32 sum bit for bit."""
    gen = torch.Generator().manual_seed(splits * 10 + packed)
    for L in range(5):
        rows, Tp, T, mask = _split_layout(packed, L)
        C = LEVEL_C[L]
        n = rows * C
        real = mask.to(cuda_device).view(rows, 1)
        part = (torch.randn(splits, rows, C, generator=gen) * torch.tensor([1.0, 30.0, 1e-3, 7.0] * 2)[:splits].view(
            splits, 1, 1)).to(cuda_device)
        part = torch.where(real, part, torch.full_like(part, float("nan")))
        bias = torch.randn(C, generator=gen).to(cuda_device)
        ref = bias.view(1, C).expand(rows, C)
        for s in range(splits):
            ref = ref + part[s]
        ref = torch.where(real, ref, torch.zeros_like(ref))
        row_mask = mask.to(torch.uint8).to(cuda_device) if packed else None
        for f16 in (1, 0):
            dt = torch.float16 if f16 else torch.float32
            for want_out, want_pair in ((True, True), (True, False), (False, True)):
                def launch(out, hi, lo):
                    return kp.sum_split(part, splits, rows * C, bias, out if want_out else None, hi if want_pair else None,
                                        lo if want_pair else None, C, Tp, T, rows, f16, row_mask)

                out, hi, lo = _launch_twice([(n, torch.float32), (n, dt), (n, dt)], launch)
                if want_out:
                    assert torch.equal(_bits(out.view(rows, C)), _bits(ref)), (L, f16, "not torch's sum in split order")
                else:
                    assert bool((out == SENTINEL).all())
                if want_pair:
                    _assert_pair_model(ref.reshape(-1), hi, lo, f16)
                else:
                    assert bool((hi.float() == SENTINEL).all()) and bool((lo.float() == SENTINEL).all())
