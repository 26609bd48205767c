"""Long clips (more than 160 tokens, up to the 5000-row positional table) on fp16 pairs with head dim 128: the streaming
wgmma attention kernel (kAttnWgmmaStream, rohm_b200/csrc/attention.cu) against float64, the automatic kernel choice, and
PoseNet forward / sampling / guidance on long clips through the public API against the oracle.

Kernel tolerance per output (i, d), relative to the output's natural scale sum_j p_ij |v_jd| (test_gpu_attention.py's
bound plus two terms for the online softmax):
    |got - ref| <= (C_OUT 2^-18 + 2 x 2^-20 L_i + 2^-21 L_i + n_blocks 2^-21) sum_j p_ij |v_jd|
* n_blocks 2^-21, n_blocks = ceil(S / 64): per 64-key block the kernel folds the block's P V (its own accumulator, 12
  wgmma additions relative to the block's share, fewer than the 30 of the 160-key kernel that C_OUT covers) into the
  running O with one fma by the factor a = exp((m_old - m_new) scale): one rounding (2^-24) plus the factor's own error
  (expf, 2 ulp = 2^-23); l = l a + (block sum) takes two roundings plus the same factor error.  7 x 2^-24 < 2^-21.
* 2^-21 L_i: the rounding of each factor's argument (m_old - m_new) scale is relative to its size, and the sizes of the
  arguments telescope over the blocks to (m_final - m_first) scale <= 2 L_i: 2 L_i x 2^-23 on O and again on l.
sharp_first / sharp_last put the row maximum into the first / last key block: the running max is then final at once, or
changes only at the very end, the two extremes of the rescaling."""
import argparse
import math

import pytest
import torch

import kernel_probe as kp
from helpers import NoiseTape, TOL
from oracle import diffusion_oracle as do
from oracle import kinematics_oracle as ko
from oracle import pipeline_oracle, posenet_oracle
from rohm_b200 import _lib, diffusion, synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.posenet import PoseNet
from test_gpu_attention import B, D, POISONED, REGIMES, SENTINEL, _launch, _split_ok

pytestmark = pytest.mark.gpu

F16, TF32 = kp.KIND_F16, kp.KIND_TF32
C_OUT = 4.0
DH = 128
S_STREAM = [1, 63, 64, 65, 128, 129, 160, 161, 212, 213, 256, 257, 1000, 4097, 5000]
SAMPLED_FROM = 1000  # from this clip length on, the float64 reference covers sampled query rows only


@pytest.fixture(scope="module")
def dev(cuda_device):
    kp.lib()  # a missing probe library fails every test of the module
    return cuda_device


def _query_rows(S, seed):
    """All rows of a short clip; of a long one the first, the last, both sides of every 64-query tile boundary and a
    seeded sample (a full float64 P of 4 clips x 4 heads x 5000^2 would be 3.2 GB)."""
    if S < SAMPLED_FROM:
        return torch.arange(S)
    edges = [r for t in range(64, S, 64) for r in (t - 1, t)]
    sample = torch.randperm(S, generator=torch.Generator().manual_seed(seed))[:64].tolist()
    return torch.tensor(sorted(set([0, S - 1] + edges + sample)))


def _reference_rows(value, S, scale, rows):
    """float64 softmax(scale Q K^T) V of the query rows `rows` of every clip -> (out, tol), both [B, len(rows), D]."""
    H = D // DH
    x = value[:B * S].reshape(B, S, 3, H, DH)
    q, k, v = x[:, rows.to(value.device), 0], x[:, :, 1], x[:, :, 2]
    p = torch.softmax(scale * torch.einsum("bihd,bjhd->bhij", q, k), dim=-1)
    o = torch.einsum("bhij,bjhd->bihd", p, v)
    scale_o = torch.einsum("bhij,bjhd->bihd", p, v.abs())
    L = (scale * torch.einsum("bihd,bjhd->bhij", q.abs(), k.abs()).amax(-1)).permute(0, 2, 1)[..., None]  # [B, R, H, 1]
    n_blocks = -(-S // 64)
    tol = (C_OUT * 2.0 ** -18 + (2.0 * 2.0 ** -20 + 2.0 ** -21) * L + n_blocks * 2.0 ** -21) * scale_o
    R = len(rows)
    return o.reshape(B, R, D), tol.reshape(B, R, D)


def _check_stream(dev, S, regime):
    seed = 1000 * S + DH + REGIMES.index(regime)
    rc, value, ctx_hi, ctx_lo, scale = _launch(dev, kp.ATTN_WGMMA_STREAM, F16, S, DH, regime, seed)
    assert rc == 0, (S, rc)
    assert bool((ctx_hi[B * S:] == SENTINEL).all()) and bool((ctx_lo[B * S:] == SENTINEL).all()), "wrote past B * S"
    got = kp.pair_value(ctx_hi, ctx_lo)[:B * S].reshape(B, S, D)
    assert bool((ctx_hi[:B * S] != SENTINEL).all()), "a row of the clips was not written"
    rows = _query_rows(S, seed)
    ref, tol = _reference_rows(value, S, scale, rows)
    good = [b for b in range(B) if b not in POISONED]
    for b in good:
        assert bool(torch.isfinite(got[b]).all()), f"NaN from another clip leaked into clip {b} (S={S})"
        ratio = float(((got[b][rows.to(dev)] - ref[b]).abs() / tol[b]).max())
        assert ratio <= 1.0, f"stream S={S} {regime}: clip {b} max |err| / bound = {ratio:.3f}"
    all_rows = torch.cat([torch.arange(b * S, (b + 1) * S) for b in good]).to(dev)
    assert _split_ok(ctx_hi[all_rows], ctx_lo[all_rows]), "context hi/lo split"


@pytest.mark.parametrize("regime", REGIMES)
def test_streaming_kernel_against_float64(dev, regime):
    for S in S_STREAM:
        _check_stream(dev, S, regime)


def test_automatic_choice_on_fp16_pairs_of_head_dim_128(dev):
    """kAttnAuto: the streaming kernel above 160 tokens, the 160-key wgmma kernel at 160 or fewer (bit for bit)."""
    for S, forced in ((161, kp.ATTN_WGMMA_STREAM), (1000, kp.ATTN_WGMMA_STREAM), (145, kp.ATTN_WGMMA)):
        outs = []
        for which in (kp.ATTN_AUTO, forced):
            rc, _, hi, lo, _ = _launch(dev, which, F16, S, DH, "flat", 19)
            assert rc == 0, (S, which, rc)
            outs.append((hi, lo))
        assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(outs[0], outs[1])), S


def test_streaming_kernel_outside_its_domain_is_refused(dev):
    """TF32 Q|K|V or head dim 64: cudaErrorInvalidValue before any launch, the context buffer untouched."""
    for kind, dh, S in ((TF32, 128, 200), (TF32, 128, 1000), (F16, 64, 200), (F16, 64, 1000)):
        rc, _, ctx_hi, ctx_lo, _ = _launch(dev, kp.ATTN_WGMMA_STREAM, kind, S, dh, "flat", 5)
        assert rc == kp.CUDA_ERROR_INVALID_VALUE, (kind, dh, S, rc)
        assert bool((ctx_hi == SENTINEL).all()) and bool((ctx_lo == SENTINEL).all())


# ---------------------------------------------------------------------------------------------------------------------
# PoseNet through the public API
# ---------------------------------------------------------------------------------------------------------------------
def _model(dev, ds=None):
    ds = ds if ds is not None else synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, device=dev,
                traj_feat_dim=22)
    sd = {k: v.cpu() for k, v in synthetic.synth_state_dict(m, 1).items()}
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


@pytest.fixture(scope="module")
def posenet(cuda_device):
    return _model(cuda_device)


def _diff(steps, resp, dev):
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(args, diffusion, diffusion.SpacedDiffusionPoseNet, steps, resp, dev)


# 211 / 212 frames: the last clip the SIMT kernel could hold and the first it could not; 255 / 256: the old 256-token limit
@pytest.mark.parametrize("B_,T", [(2, 211), (2, 212), (2, 255), (2, 256), (1, 600), (2, 1000)])
def test_long_clip_forward_matches_oracle(posenet, cuda_device, B_, T):
    m, sd = posenet
    gen = torch.Generator().manual_seed(2000 + B_ * 7 + T)
    x = torch.randn(B_, 294, 1, T, generator=gen)
    cond = synthetic.posenet_batch(B_, T, 5)['cond']
    ts = torch.randint(0, 1000, (B_,), generator=gen)
    ref = posenet_oracle.posenet_forward(sd, x, cond, ts)
    y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    assert float((y - ref).abs().max()) < TOL
    assert torch.equal(y[:, :22], cond[:, :22])  # trajectory channels are a verbatim copy of the condition


def test_longest_clip_against_float64_oracle(posenet, cuda_device):
    """4999 frames + the timestep token fill the 5000-row positional table."""
    m, sd = posenet
    B_, T = 1, 4999
    gen = torch.Generator().manual_seed(4999)
    x = torch.randn(B_, 294, 1, T, generator=gen)
    cond = synthetic.posenet_batch(B_, T, 9)['cond']
    ts = torch.tensor([500])
    ref = posenet_oracle.posenet_forward(sd, x.double(), cond.double(), ts).float()
    y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    err = float((y - ref).abs().max())
    print(f"PoseNet 1 x 4999 frames: max |cuda - float64 oracle| = {err:.3e}")
    assert err < TOL * max(1.0, float(ref.abs().max()) / 10.0)
    assert torch.equal(y[:, :22], cond[:, :22])


def test_clip_longer_than_the_positional_table_is_refused(posenet, cuda_device):
    m, _ = posenet
    T = 5000
    x = torch.zeros(1, 294, 1, T, device=cuda_device)
    m.invalidate_engine()
    with pytest.raises(RohmB200Error, match="sequence_pos_encoder.pe"):
        m({'x_t': x, 'cond': x}, torch.tensor([3], device=cuda_device))
    assert m._engine is None, "the engine must not be built for a clip the positional table cannot hold"


def test_tf32_precision_keeps_its_clip_limit(posenet, cuda_device):
    """tf32x3 attention above 160 tokens is the SIMT kernel: 300 frames are refused, and the message states the rule."""
    m, _ = posenet
    T = 300
    x = torch.zeros(1, 294, 1, T, device=cuda_device)
    m.precision = _lib.PRECISION_TF32X3
    try:
        with pytest.raises(RohmB200Error) as info:
            m({'x_t': x, 'cond': x}, torch.tensor([3], device=cuda_device))
    finally:
        m.precision = None
        m.invalidate_engine()
    msg = str(info.value)
    assert "f16x2" in msg and "head dim 128" in msg and "tf32x3" in msg and "211" in msg, msg


def test_respaced_sampling_at_1000_frames_matches_oracle(posenet, cuda_device):
    """10 respaced steps through eval_losses with a replayed noise tape, against the oracle's p_sample_loop."""
    m, sd = posenet
    B_, T = 2, 1000
    d = _diff(1000, 'ddim10', cuda_device)
    cond = synthetic.posenet_batch(B_, T, 3)['cond']
    tape = NoiseTape(7, cuda_device)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    _, out = d.eval_losses(model=m, batch={'cond': cond.to(cuda_device)}, shape=[B_, 294, 1, T], progress=False,
                           clip_denoised=False, cond_fn_with_grad=False, compute_loss=False)
    tables, tmap = do.create_diffusion('cosine', 1000, 'ddim10')
    ctape = NoiseTape(7)
    x_T = ctape.randn(B_, 294, 1, T)
    ref, _ = do.p_sample_loop(tables, tmap,
                              lambda x, t: posenet_oracle.posenet_forward(sd, x, cond, torch.full((B_,), t, dtype=torch.long)),
                              x_T, lambda i: ctape.randn_like(x_T))
    assert float((out.cpu() - ref).abs().max()) < TOL


def test_fused_sample_step_at_1000_frames_equals_the_unfused_chain(posenet, cuda_device, monkeypatch):
    """One graph launch per step (forward + in-kernel-noise update) == forward, torch.randn_like, gather, update, bit for
    bit, and torch's generator ends in the same state."""
    m, _ = posenet
    B_, T = 2, 1000
    cond = synthetic.posenet_batch(B_, T, 5)['cond'].to(cuda_device)
    gen = torch.cuda.default_generators[cuda_device.index]
    d = _diff(1000, 'ddim6', cuda_device)
    outs, offs = [], []
    for fused in (True, False):
        monkeypatch.setattr(diffusion, "_FUSED_STEP", fused)
        torch.manual_seed(123)
        outs.append(d.p_sample_loop(m, {'cond': cond}, [B_, 294, 1, T], clip_denoised=False))
        offs.append(gen.get_offset())
    assert torch.equal(outs[0], outs[1]) and offs[0] == offs[1]


def test_guided_step_at_1000_frames(cuda_device):
    """One guided 'amass' step (skating guidance) on a 1000-frame clip: the denoiser output against the oracle's, and the
    guided update against the oracle's update at the CUDA path's own x0 (the update is ill-conditioned in x0, see
    test_gpu_pipeline.py::test_guided_tail_at_benchmark_size)."""
    dev = cuda_device
    B_, T, i = 1, 1000, 10
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    m, sd = _model(dev, ds)
    body_o = synthetic.smplx_like_model(0)
    d = _diff(1000, '', dev)
    tables, tmap = do.create_diffusion('cosine', 1000, '')
    init = synthetic.plausible_motion(B_, T, 21, ds)
    tape = NoiseTape(22)
    x = do.q_sample(tables, i, init, tape.randn(B_, 294, 1, T))
    nz = tape.randn(B_, 294, 1, T)
    mean_p, std_p = torch.from_numpy(ds.Mean), torch.from_numpy(ds.Std)
    _, x0_o = pipeline_oracle.posenet_guided_step(tables, tmap, i, x, init, sd, mean_p, std_p, body_o, nz)
    d._randn_like = lambda t_, _n=nz.to(dev): _n
    o = d.p_sample_with_grad(m, {'cond': init.to(dev)}, x.to(dev), d._t_rows(B_, dev)[i], clip_denoised=False,
                             grad_type='amass', _step_index=i)
    x0_c = o['pred_xstart'].cpu()
    assert float((x0_c - x0_o).abs().max()) < TOL
    g_at_c = ko.guide_skating(x0_c, mean_p, std_p, body_o)
    upd_o = do.p_sample_step(tables, i, x, x0_c, nz, [(3e6, g_at_c)] if g_at_c.dim() != 0 else None)
    assert float((o['sample'].cpu() - upd_o).abs().max()) < TOL * max(1.0, float(upd_o.abs().max()))
