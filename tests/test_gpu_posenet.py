"""GPU parity tests (pytest -m gpu): the CUDA path, called through the public drop-in API / the C-ABI, against the CPU
oracle, the reference golden fixtures and size-independent properties.  Tolerance: 1e-4 abs (north_star)."""
import argparse
import ctypes

import numpy as np
import pytest
import torch

from helpers import NoiseTape, TOL, golden
from oracle import diffusion_oracle as do
from oracle import posenet_oracle
from rohm_b200 import _lib, diffusion, ops, synthetic
from rohm_b200.posenet import PoseNet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def posenet(cuda_device):
    ds = synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4,
                device=cuda_device, traj_feat_dim=22)
    sd = synthetic.synth_state_dict(m, 1)
    m.load_state_dict(sd)
    m.to(cuda_device).eval()
    return m, sd


def _diff(steps, resp, dev, cls=diffusion.SpacedDiffusionPoseNet):
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(args, diffusion, cls, steps, resp, dev)


def test_native_library_is_what_runs(cuda_device):
    lib = _lib.load()
    assert isinstance(lib, ctypes.CDLL) and lib.rohm_version() >= 100
    assert _lib.ctx(cuda_device.index) is not None
    with open("/proc/self/maps") as f:
        assert "librohm_b200.so" in f.read()


def test_forward_matches_reference_golden(posenet, cuda_device):
    m, sd = posenet
    g = golden("posenet_forward.npz")
    for c in range(int(g["n_cases"])):
        B, T, s = [int(v) for v in g[f"c{c}_meta"]]
        gen = torch.Generator().manual_seed(s)
        x = torch.randn(B, 294, 1, T, generator=gen)
        cond = synthetic.posenet_batch(B, T, s + 100)['cond']
        ts = torch.from_numpy(g[f"c{c}_timesteps"])
        y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
        err = float((y - torch.from_numpy(g[f"c{c}_out"])).abs().max())
        assert err < TOL, (c, err)


# T + 1 tokens per clip: 128 / 129 straddle a 64-query tile boundary of the wgmma attention kernel, 160 is its largest
# clip, 161 and 201 take the mma.sync / SIMT fallbacks
@pytest.mark.parametrize("B,T", [(1, 1), (2, 7), (3, 143), (5, 144), (2, 127), (2, 128), (3, 159), (1, 160), (2, 200)])
def test_forward_matches_oracle(posenet, cuda_device, B, T):
    m, sd = posenet
    gen = torch.Generator().manual_seed(1000 + B * 7 + T)
    x = torch.randn(B, 294, 1, T, generator=gen)
    cond = synthetic.posenet_batch(B, T, 5)['cond']
    ts = torch.randint(0, 1000, (B,), generator=gen)
    ref = posenet_oracle.posenet_forward(sd, x, cond, ts)
    y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    assert float((y - ref).abs().max()) < TOL
    assert torch.equal(y[:, :22], cond[:, :22])  # trajectory channels are a verbatim copy of the condition


@pytest.mark.parametrize("prec,tol", [(_lib.PRECISION_F16X2, TOL), (_lib.PRECISION_TF32X3, TOL), (_lib.PRECISION_TF32, 5e-2)])
def test_every_precision_mode_against_oracle(posenet, cuda_device, prec, tol):
    """fp16 hi/lo (default) and TF32 hi/lo are both fp32-grade; single-pass TF32 is the documented fast mode.
    Includes large-magnitude inputs (|x| ~ 500, the range guided sampling reaches) for the fp16 range."""
    m, sd = posenet
    B, T = 3, 60
    gen = torch.Generator().manual_seed(4242)
    x = torch.randn(B, 294, 1, T, generator=gen)
    x[1] *= 500.0
    cond = synthetic.posenet_batch(B, T, 9)['cond']
    ts = torch.tensor([0, 500, 999])
    ref = posenet_oracle.posenet_forward(sd, x.double(), cond.double(), ts).float()
    m.precision = prec
    try:
        y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    finally:
        m.precision = None
    assert m._engine.precision == prec
    assert float((y - ref).abs().max()) < tol * max(1.0, float(ref.abs().max()) / 10.0)


def test_mma_sync_attention_fallback_matches_oracle(posenet, cuda_device, monkeypatch):
    """ROHM_B200_TC_ATTENTION=0 routes f16x2 attention to the mma.sync m16n8k16 kernel (also used for head dim 64)."""
    m, sd = posenet
    B, T = 3, 144
    gen = torch.Generator().manual_seed(31337)
    x = torch.randn(B, 294, 1, T, generator=gen)
    cond = synthetic.posenet_batch(B, T, 11)['cond']
    ts = torch.tensor([1, 400, 998])
    ref = posenet_oracle.posenet_forward(sd, x, cond, ts)
    monkeypatch.setenv("ROHM_B200_TC_ATTENTION", "0")
    m.invalidate_engine()
    try:
        y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    finally:
        monkeypatch.delenv("ROHM_B200_TC_ATTENTION")
        m._engine = None
    assert float((y - ref).abs().max()) < TOL


@pytest.mark.parametrize("env", [{"ROHM_B200_TC_ATTENTION": "0"}, {"ROHM_B200_MULTICAST": "1"}, {"ROHM_B200_TMA_STORE": "0"},
                                 {"ROHM_B200_FUSED_LN": "0"}])
def test_engine_switches_match_oracle(posenet, cuda_device, monkeypatch, env):
    """The engines behind the library's switches: ROHM_B200_TC_ATTENTION=0 routes f16x2 attention to the mma.sync m16n8k16
    kernel, ROHM_B200_MULTICAST=1 shares the GEMMs' A tiles across CTA pairs, ROHM_B200_TMA_STORE=0 keeps the per-thread
    store epilogue (and with it the separate LayerNorm kernel), ROHM_B200_FUSED_LN=0 the separate LayerNorm kernel alone.
    32 clips x 145 tokens: 37 row tiles, so the persistent GEMMs run several rounds per launch."""
    m, sd = posenet
    B, T = 32, 144
    gen = torch.Generator().manual_seed(31337)
    x = torch.randn(B, 294, 1, T, generator=gen)
    cond = synthetic.posenet_batch(B, T, 11)['cond']
    ts = torch.randint(0, 1000, (B,), generator=gen)
    ref = posenet_oracle.posenet_forward(sd, x, cond, ts)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    m.invalidate_engine()
    try:
        y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    finally:
        for k in env:
            monkeypatch.delenv(k)
        m.invalidate_engine()
    assert float((y - ref).abs().max()) < TOL


def test_launch_switches_do_not_change_the_result(posenet, cuda_device):
    """Programmatic dependent launch and CUDA-graph replay only change how the kernels are scheduled: the forward must be
    bit-identical with either switched off (rohm_posenet_set_option 1 / 0)."""
    m, _ = posenet
    B, T = 5, 144
    gen = torch.Generator().manual_seed(41)
    x = torch.randn(B, 294, 1, T, generator=gen).to(cuda_device)
    cond = synthetic.posenet_batch(B, T, 3)['cond'].to(cuda_device)
    ts = torch.randint(0, 1000, (B,), generator=gen).to(cuda_device)
    ref = m({'x_t': x, 'cond': cond}, ts).clone()
    eng = m._engine
    try:
        for option in (1, 0):
            assert eng.lib.rohm_posenet_set_option(eng.handle, option, 0) == 0
            assert torch.equal(m({'x_t': x, 'cond': cond}, ts), ref)
            assert eng.lib.rohm_posenet_set_option(eng.handle, option, 1) == 0
            assert torch.equal(m({'x_t': x, 'cond': cond}, ts), ref)
    finally:
        eng.lib.rohm_posenet_set_option(eng.handle, 0, 1)
        eng.lib.rohm_posenet_set_option(eng.handle, 1, 1)


def test_forward_noncontiguous_inputs_and_cond_updates(posenet, cuda_device):
    """The driver builds cond by permute(0,2,1).unsqueeze(-2) (non-contiguous) and edits it in place between rounds."""
    m, sd = posenet
    B, T = 2, 24
    gen = torch.Generator().manual_seed(77)
    base = torch.randn(B, T, 294, generator=gen).to(cuda_device)
    cond = torch.permute(base, (0, 2, 1)).unsqueeze(-2)
    assert not cond.is_contiguous()
    x = torch.randn(B, 294, 1, T, generator=gen)
    ts = torch.tensor([3, 900])
    y1 = m({'x_t': x.to(cuda_device), 'cond': cond}, ts.to(cuda_device)).cpu()
    ref1 = posenet_oracle.posenet_forward(sd, x, cond.cpu(), ts)
    assert float((y1 - ref1).abs().max()) < TOL
    base[:, :, 0:22] += 1.0  # in-place edit of the underlying storage must be picked up
    y2 = m({'x_t': x.to(cuda_device), 'cond': cond}, ts.to(cuda_device)).cpu()
    ref2 = posenet_oracle.posenet_forward(sd, x, cond.cpu(), ts)
    assert float((y2 - ref2).abs().max()) < TOL
    assert float((y2 - y1).abs().max()) > 1e-3


def test_weight_reload_is_picked_up(posenet, cuda_device):
    m, sd = posenet
    B, T = 1, 8
    x = torch.randn(B, 294, 1, T)
    cond = synthetic.posenet_batch(B, T, 1)['cond']
    ts = torch.tensor([10])
    sd2 = {k: v.cpu() for k, v in synthetic.synth_state_dict(m, 2).items()}
    m.load_state_dict(sd2)
    y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    assert float((y - posenet_oracle.posenet_forward(sd2, x, cond, ts)).abs().max()) < TOL
    m.load_state_dict(sd)
    y = m({'x_t': x.to(cuda_device), 'cond': cond.to(cuda_device)}, ts.to(cuda_device)).cpu()
    assert float((y - posenet_oracle.posenet_forward(sd, x, cond, ts)).abs().max()) < TOL


def test_ddpm_step_bit_exact(cuda_device):
    """The fused posterior step equals the reference's chain of fp32 elementwise ops bit for bit."""
    tables, _ = do.create_diffusion('cosine', 1000, '')
    gen = torch.Generator().manual_seed(3)
    for shape in ([3, 294, 1, 143], [2, 144, 13], [1, 5]):
        x0, xt, nz, gr = (torch.randn(shape, generator=gen) for _ in range(4))
        d = _diff(1000, '', cuda_device)
        for i in (999, 500, 50, 1, 0):
            t = torch.full((shape[0],), i, dtype=torch.long, device=cuda_device)
            coef = d._coef_for(t)
            y = ops.ddpm_step(x0.to(cuda_device), xt.to(cuda_device), nz.to(cuda_device), coef).cpu()
            ref = do.p_sample_step(tables, i, xt, x0, nz)
            assert torch.equal(y, ref), (shape, i, float((y - ref).abs().max()))
            # guided variant: mean += (3e6 * var) * grad
            c2 = coef.clone()
            c2[:, 3] = 3e6 * coef[:, 3]
            y = ops.ddpm_step(x0.to(cuda_device), xt.to(cuda_device), nz.to(cuda_device), c2,
                              grads=(gr.to(cuda_device),)).cpu()
            ref = do.p_sample_step(tables, i, xt, x0, nz, [(3e6, gr)])
            assert torch.equal(y, ref), (shape, i)
    # per-clip coefficient rows (a batch of different timesteps)
    shape = [4, 294, 1, 16]
    x0, xt, nz = (torch.randn(shape, generator=gen) for _ in range(3))
    d = _diff(1000, '', cuda_device)
    t = torch.tensor([0, 7, 500, 999], device=cuda_device)
    y = ops.ddpm_step(x0.to(cuda_device), xt.to(cuda_device), nz.to(cuda_device), d._coef_for(t)).cpu()
    for b, i in enumerate([0, 7, 500, 999]):
        assert torch.equal(y[b], do.p_sample_step(tables, i, xt[b], x0[b], nz[b]))


def test_respaced_chain_matches_reference_golden(posenet, cuda_device):
    """20 respaced ancestral steps ('ddim20' of 1000), noise replayed from the fixture's seed: CUDA vs the reference."""
    m, sd = posenet
    g = golden("sampling.npz")
    B, T, bseed, nseed, steps = [int(v) for v in g["pose_ddim20_meta"]]
    d = _diff(1000, 'ddim20', cuda_device)
    assert d.num_timesteps == steps and d.timestep_map == list(range(0, 1000, 50))
    tape = NoiseTape(nseed, cuda_device)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    batch = {'cond': synthetic.posenet_batch(B, T, bseed)['cond'].to(cuda_device)}
    y = d.p_sample_loop(m, batch, [B, 294, 1, T], clip_denoised=False, cond_fn_with_grad=False).cpu()
    err = float((y - torch.from_numpy(g["pose_ddim20_out"])).abs().max())
    assert err < TOL, err
    assert batch['x_t'].shape == (B, 294, 1, T)  # side effect of the reference: batch['x_t'] is the last model input


def test_full_chain_properties_at_benchmark_size(posenet, cuda_device):
    """BASELINE configs[1] size (32 clips x 144 frames) on a 100-step respaced chain: seeded determinism, the last
    step returns pred_xstart exactly (coef1[0] = 1, coef2[0] = 0, no noise), trajectory channels == cond."""
    m, sd = posenet
    B, T = 32, 144
    d = _diff(1000, 'ddim100', cuda_device)
    batch = {'cond': synthetic.posenet_batch(B, T, 9)['cond'].to(cuda_device)}
    outs = []
    for _ in range(2):
        torch.manual_seed(4321)
        last = None
        for o in d.p_sample_loop_progressive(m, batch, [B, 294, 1, T], clip_denoised=False):
            last = o
        outs.append(last)
    assert torch.equal(outs[0]['sample'], outs[1]['sample'])
    assert torch.equal(outs[0]['sample'], outs[0]['pred_xstart'])
    assert torch.equal(outs[0]['sample'][:, :22], batch['cond'][:, :22])
    assert bool(torch.isfinite(outs[0]['sample']).all())
    # spot-check the final denoiser call against the oracle on 2 clips
    x_in = outs[0]['x_t'][:2].cpu()
    ref = posenet_oracle.posenet_forward(sd, x_in, batch['cond'][:2].cpu(), torch.zeros(2, dtype=torch.long))
    assert float((outs[0]['sample'][:2].cpu() - ref).abs().max()) < TOL


def test_eval_losses_api_and_early_stop(posenet, cuda_device):
    m, sd = posenet
    B, T = 2, 16
    d = _diff(1000, '', cuda_device)
    batch = {'cond': synthetic.posenet_batch(B, T, 2)['cond'].to(cuda_device)}
    torch.manual_seed(0)
    # early_stop keeps indices[0:980] and returns pred_xstart of the last executed step
    steps = []
    real = d.p_sample
    d.p_sample = lambda *a, **k: (steps.append(int(a[3][0])), real(*a, **k))[1]
    loss, out = d.eval_losses(model=m, batch=batch, shape=[B, 294, 1, T], progress=False, clip_denoised=False,
                              cond_fn_with_grad=False, early_stop=True, compute_loss=False, grad_type='amass')
    d.p_sample = real
    assert loss is None and out.shape == (B, 294, 1, T)
    assert steps[0] == 999 and steps[-1] == 20 and len(steps) == 980


def test_ddim_restated(posenet, cuda_device):
    """DDIM (eta=0) has no runnable reference (parity unpinned): CUDA path vs the oracle's restatement."""
    m, sd = posenet
    B, T = 2, 12
    d = _diff(1000, 'ddim10', cuda_device)
    tape = NoiseTape(5, cuda_device)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    cond = synthetic.posenet_batch(B, T, 4)['cond']
    _, y = d.eval_losses(model=m, batch={'cond': cond.to(cuda_device)}, shape=[B, 294, 1, T], progress=False,
                         clip_denoised=False, timestep_respacing='ddim10', compute_loss=False)
    tables, tmap = do.create_diffusion('cosine', 1000, 'ddim10')
    ctape = NoiseTape(5)
    x_T = ctape.randn(B, 294, 1, T)
    ref = do.ddim_sample_loop(tables, tmap,
                              lambda x, t: posenet_oracle.posenet_forward(sd, x, cond, torch.full((B,), t, dtype=torch.long)),
                              x_T, lambda i: ctape.randn_like(x_T))
    assert float((y.cpu() - ref).abs().max()) < TOL


def test_q_sample_matches_oracle(cuda_device):
    tables, _ = do.create_diffusion('cosine', 1000, '')
    d = _diff(1000, '', cuda_device)
    gen = torch.Generator().manual_seed(8)
    xs, nz = torch.randn(3, 294, 1, 20, generator=gen), torch.randn(3, 294, 1, 20, generator=gen)
    t = torch.tensor([0, 400, 999], device=cuda_device)
    y = d.q_sample(xs.to(cuda_device), t, nz.to(cuda_device)).cpu()
    for b, i in enumerate([0, 400, 999]):
        assert torch.equal(y[b], do.q_sample(tables, i, xs[b], nz[b]))


def test_recycled_condition_address_is_not_mistaken_for_the_cached_one(posenet, cuda_device):
    """Regression (round-1 advisor finding): the driver frees and rebuilds batch['cond'] per batch; the caching allocator
    hands the new tensor the old address with the same version count.  The step-invariant embedding must follow the tensor
    OBJECT, and every sampling loop must re-embed its condition."""
    m, sd = posenet
    B, T = 2, 16
    x = torch.randn(B, 294, 1, T, generator=torch.Generator().manual_seed(3)).to(cuda_device)
    ts = torch.tensor([10, 500], device=cuda_device)
    outs, ptrs = [], []
    for k in range(4):
        cond = synthetic.posenet_batch(B, T, 40 + k)['cond'].to(cuda_device)  # fresh tensor, previous one freed below
        cond[:, :, :, 0] = 0.0                                                # same number of in-place edits each time
        ptrs.append((cond.data_ptr(), cond._version))
        outs.append(m({'x_t': x, 'cond': cond}, ts).cpu())
        ref = posenet_oracle.posenet_forward(sd, x.cpu(), cond.cpu(), ts.cpu())
        assert float((outs[-1] - ref).abs().max()) < TOL, k
        del cond
    assert len(set(ptrs)) < 4, "allocator did not recycle the address: the scenario was not exercised"
    for k in range(1, 4):
        assert float((outs[k] - outs[k - 1]).abs().max()) > 1e-3
    # and through the sampler: two loops, same-shaped conditions rebuilt in between
    d = _diff(1000, 'ddim3', cuda_device)
    finals = []
    for k in range(2):
        cond = synthetic.posenet_batch(B, T, 60 + k)['cond'].to(cuda_device)
        tape = NoiseTape(5, cuda_device)
        d._randn, d._randn_like = tape.randn, tape.randn_like
        finals.append(d.p_sample_loop(m, {'cond': cond}, [B, 294, 1, T], clip_denoised=False).cpu())
        del cond
    assert float((finals[0] - finals[1]).abs().max()) > 1e-3


def test_out_of_range_timestep_poisons_the_output(posenet, cuda_device):
    """The reference raises on pe[t] with a bad t; the kernel cannot raise, so it must not return a plausible embedding."""
    m, sd = posenet
    B, T = 2, 8
    cond = synthetic.posenet_batch(B, T, 9)['cond'].to(cuda_device)
    x = torch.randn(B, 294, 1, T, device=cuda_device)
    y = m({'x_t': x, 'cond': cond}, torch.tensor([5, 5000], device=cuda_device))
    assert bool(torch.isnan(y[1, 22:]).all())
    # the poison stays in its clip: attention reads only the clip's own rows (the next clip lies inside clip 0's key tile)
    ref0 = posenet_oracle.posenet_forward(sd, x[:1].cpu(), cond[:1].cpu(), torch.tensor([5]))
    assert float((y[:1].cpu() - ref0).abs().max()) < TOL
    ok = m({'x_t': x, 'cond': cond}, torch.tensor([5, 4999], device=cuda_device))
    assert bool(torch.isfinite(ok).all())
    with pytest.raises(Exception):
        m({'x_t': x, 'cond': cond}, torch.tensor([5.0, 6.0], device=cuda_device))


def test_eval_losses_default_compute_loss_and_guards(posenet, cuda_device):
    """eval_losses with its default compute_loss=True (test_posenet.py:178) returns the reference's loss dictionary; DDIM
    respacing with guidance / early_stop is rejected BEFORE sampling."""
    m, _ = posenet
    B, T = 2, 16
    d = _diff(1000, 'ddim4', cuda_device)
    clean = synthetic.plausible_motion(B, T, 4, m.dataset).to(cuda_device)
    batch = {'cond': clean.clone(), 'motion_repr_clean': clean}
    loss, out = d.eval_losses(model=m, batch=batch, shape=[B, 294, 1, T], progress=False, clip_denoised=False,
                              cond_fn_with_grad=False)
    assert out.shape == (B, 294, 1, T) and 'loss' in loss and 'loss_foot_skating_from_smpl' in loss and len(loss) == 15
    calls = []
    real = m.forward
    m.forward = lambda *a, **k: (calls.append(1), real(*a, **k))[1]
    with pytest.raises(Exception):
        d.eval_losses(model=m, batch=batch, shape=[B, 294, 1, T], timestep_respacing='ddim4', cond_fn_with_grad=True,
                      grad_type='amass', compute_loss=False)
    with pytest.raises(Exception):
        d.eval_losses(model=m, batch=batch, shape=[B, 294, 1, T], timestep_respacing='ddim4', early_stop=True,
                      compute_loss=False)
    m.forward = real
    assert not calls, "the guard must fire before any denoiser step"


def test_prox_guidance_schedule_runs_both_terms(posenet, cuda_device):
    """grad_type='prox' (test_prox_egobody.py:316-323): 2-D reprojection guidance (3e5) then skating guidance (1e5) on
    step indices <= 100."""
    m, _ = posenet
    B, T = 2, 12
    dev = cuda_device
    ds = m.dataset
    ds.cam_R, ds.cam_t = torch.tensor([[1., 0, 0], [0, 0, 1], [0, -1, 0]], device=dev), torch.tensor([[0., -4, 1]], device=dev)
    d = _diff(1000, "3" + ",0" * 19, dev)
    init = synthetic.plausible_motion(B, T, 4, ds).to(dev)
    g = torch.Generator().manual_seed(1)
    batch = {'cond': init.clone(), 'transf_matrix': torch.eye(4, device=dev).repeat(B, 1, 1),
             'focal_length': torch.tensor([[1000., 1000.]], device=dev).repeat(B, 1),
             'camera_center': torch.tensor([[900., 500.]], device=dev).repeat(B, 1),
             'keypoints_2d': torch.cat([900 + 100 * torch.randn(B, T + 2, 22, 2, generator=g),
                                        torch.ones(B, T + 2, 22, 1)], dim=-1).to(dev)}
    used = []
    r2d, rsk = m.guide_2d_projection_with_smpl, m.guide_skating_with_smpl
    m.guide_2d_projection_with_smpl = lambda *a, **k: (used.append('2d'), r2d(*a, **k))[1]
    m.guide_skating_with_smpl = lambda *a, **k: (used.append('sk'), rsk(*a, **k))[1]
    torch.manual_seed(0)
    _, out = d.eval_losses(model=m, batch=batch, shape=[B, 294, 1, T], progress=False, clip_denoised=False,
                           cond_fn_with_grad=True, grad_type='prox', compute_loss=False)
    del m.guide_2d_projection_with_smpl, m.guide_skating_with_smpl
    assert used == ['2d', 'sk'] * 3 and bool(torch.isfinite(out).all())
    delattr(ds, 'cam_R'), delattr(ds, 'cam_t')


def test_in_kernel_noise_is_torchs_own_stream(cuda_device):
    """rohm_ddpm_step_philox draws what torch.randn_like would have drawn (same values, same generator advance), for sizes
    below / at / above one pass of torch's grid (SMs x 8 blocks x 256 threads x 4)."""
    dev = cuda_device
    gen = torch.cuda.default_generators[dev.index]
    for shape in [(1, 7, 1, 3), (2, 294, 1, 16), (32, 294, 1, 144), (128, 294, 1, 144), (64, 144, 13)]:
        torch.manual_seed(11)
        x0, x = torch.randn(shape, device=dev), torch.randn(shape, device=dev)
        coef = torch.rand(shape[0], 8, device=dev)
        g1 = torch.randn(shape, device=dev)
        off0 = gen.get_offset()
        ref = ops.ddpm_step(x0, x, torch.randn_like(x), coef, grads=(g1,))
        off_ref = gen.get_offset()
        gen.set_offset(off0)
        got = ops.ddpm_step_philox(x0, x, coef, grads=(g1,))
        assert gen.get_offset() == off_ref, shape
        assert torch.equal(got, ref), shape
        after_a = torch.randn(5, device=dev)
        gen.set_offset(off_ref)
        assert torch.equal(after_a, torch.randn(5, device=dev))


def test_fused_sample_step_equals_the_unfused_chain(posenet, cuda_device, monkeypatch):
    """One graph launch per step (forward + in-kernel-noise update) == forward, torch.randn_like, gather, update: bit for bit,
    for an un-respaced and a respaced schedule, and torch's generator ends in the same state."""
    m, _ = posenet
    B, T = 2, 16
    cond = synthetic.posenet_batch(B, T, 5)['cond'].to(cuda_device)
    gen = torch.cuda.default_generators[cuda_device.index]
    for steps, resp in ((1000, 'ddim6'), (6, '')):
        d = _diff(steps, resp, cuda_device)
        outs, offs = [], []
        for fused in (True, False):
            monkeypatch.setattr(diffusion, "_FUSED_STEP", fused)
            torch.manual_seed(123)
            outs.append(d.p_sample_loop(m, {'cond': cond}, [B, 294, 1, T], clip_denoised=False))
            offs.append(gen.get_offset())
        assert torch.equal(outs[0], outs[1]) and offs[0] == offs[1], (steps, resp)
    # guided tail (explicit forward + guidance + in-kernel noise) against the explicit-noise path
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    old = m.dataset
    m.dataset = ds
    try:
        d = _diff(1000, "4" + ",0" * 19, cuda_device)
        init = synthetic.plausible_motion(B, T, 4, ds).to(cuda_device)
        outs = []
        for fused in (True, False):
            monkeypatch.setattr(diffusion, "_FUSED_STEP", fused)
            torch.manual_seed(5)
            outs.append(d.p_sample_loop(m, {'cond': init}, [B, 294, 1, T], clip_denoised=False, cond_fn_with_grad=True,
                                        grad_type='amass'))
        assert torch.equal(outs[0], outs[1])
    finally:
        m.dataset = old
