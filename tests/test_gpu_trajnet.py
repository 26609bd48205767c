"""GPU parity tests for the TrajNet / TrajControl engine (conv-as-GEMM on wgmma) and its sampling loop."""
import argparse

import numpy as np
import pytest
import torch

from helpers import NoiseTape, TOL, golden
from oracle import diffusion_oracle as do
from oracle import trajnet_oracle
from rohm_b200 import diffusion, synthetic
from rohm_b200.trajnet import TrajNet

pytestmark = pytest.mark.gpu


def _build(control, dev, seed=2, mid_dim=512):
    ds = synthetic.make_dataset('traj')
    m = TrajNet(time_dim=32, mid_dim=mid_dim, cond_dim=13, traj_feat_dim=13, trajcontrol=control, device=dev, dataset=ds,
                repr_abs_only=True)
    sd = {k: v.cpu() for k, v in synthetic.synth_state_dict(m, seed).items()}
    m.load_state_dict(sd)
    m.to(dev).eval()
    return m, sd


@pytest.fixture(scope="module")
def nets(cuda_device):
    return {False: _build(False, cuda_device), True: _build(True, cuda_device)}


def test_forward_matches_reference_golden(nets, cuda_device):
    g = golden("trajnet_forward.npz")
    for c in range(int(g["n_cases"])):
        B, T, s, control = [int(v) for v in g[f"c{c}_meta"]]
        m, sd = nets[bool(control)]
        gen = torch.Generator().manual_seed(s)
        x = torch.randn(B, T, 13, generator=gen)
        batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, s + 100, control=bool(control)).items()}
        batch['x_t'] = x.to(cuda_device)
        ts = torch.from_numpy(g[f"c{c}_timesteps"]).to(cuda_device)
        y = m(batch, ts).cpu()
        err = float((y - torch.from_numpy(g[f"c{c}_out"])).abs().max())
        assert err < TOL, (c, err)


@pytest.mark.parametrize("prec", [2, 3])
def test_both_parity_precision_modes(nets, cuda_device, prec):
    """fp16 hi/lo pairs (2, default) and TF32 hi/lo pairs (3) are both fp32-grade."""
    m, sd = nets[True]
    B, T = 4, 144
    gen = torch.Generator().manual_seed(99)
    x = torch.randn(B, T, 13, generator=gen)
    batch = synthetic.trajnet_batch(B, T, 8, control=True)
    ts = torch.tensor([0, 17, 500, 999])
    ref = trajnet_oracle.trajnet_forward(sd, x, batch['cond'], ts, batch.get('control_cond'))
    gb = {k: v.to(cuda_device) for k, v in batch.items()}
    gb['x_t'] = x.to(cuda_device)
    m.precision = prec
    try:
        y = m(gb, ts.to(cuda_device)).cpu()
    finally:
        m.precision = None
    assert float((y - ref).abs().max()) < TOL


@pytest.mark.parametrize("control", [False, True])
@pytest.mark.parametrize("B,T", [(1, 16), (3, 48), (5, 144), (2, 160)])
def test_forward_matches_oracle(nets, cuda_device, control, B, T):
    m, sd = nets[control]
    gen = torch.Generator().manual_seed(7 * B + T)
    x = torch.randn(B, T, 13, generator=gen)
    batch = synthetic.trajnet_batch(B, T, 3, control=control)
    ts = torch.randint(0, 1000, (B,), generator=gen)
    ref = trajnet_oracle.trajnet_forward(sd, x, batch['cond'], ts, batch.get('control_cond'))
    gb = {k: v.to(cuda_device) for k, v in batch.items()}
    gb['x_t'] = x.to(cuda_device)
    y = m(gb, ts.to(cuda_device)).cpu()
    assert float((y - ref).abs().max()) < TOL


def test_cond_and_control_updates_are_picked_up(nets, cuda_device):
    m, sd = nets[True]
    B, T = 2, 32
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, 13, generator=gen)
    batch = synthetic.trajnet_batch(B, T, 9, control=True)
    ts = torch.tensor([5, 60])
    gb = {k: v.to(cuda_device) for k, v in batch.items()}
    gb['x_t'] = x.to(cuda_device)
    y1 = m(gb, ts.to(cuda_device)).cpu()
    gb['control_cond'][:, :, :5] += 0.5  # in-place edit (test_amass_full.py:256-258 rewrites control_cond per round)
    y2 = m(gb, ts.to(cuda_device)).cpu()
    ref2 = trajnet_oracle.trajnet_forward(sd, x, batch['cond'], ts, gb['control_cond'].cpu())
    assert float((y2 - ref2).abs().max()) < TOL and float((y2 - y1).abs().max()) > 1e-4
    gb['cond'] = gb['cond'] * 0.5  # new tensor
    y3 = m(gb, ts.to(cuda_device)).cpu()
    ref3 = trajnet_oracle.trajnet_forward(sd, x, gb['cond'].cpu(), ts, gb['control_cond'].cpu())
    assert float((y3 - ref3).abs().max()) < TOL


def test_rejects_bad_frame_count(nets, cuda_device):
    from rohm_b200 import RohmB200Error
    m, _ = nets[False]
    with pytest.raises(RohmB200Error):
        m({'x_t': torch.zeros(1, 20, 13, device=cuda_device), 'cond': torch.zeros(1, 20, 13, device=cuda_device)},
          torch.zeros(1, dtype=torch.long, device=cuda_device))


def test_rejects_mid_dim_that_is_not_a_multiple_of_256(cuda_device):
    """mid_dim = 128 makes the level-0 blocks 16 channels wide: GroupNorm(8) groups of 2 channels, which the GroupNorm kernel
    (float4 units) cannot take.  The engine refuses such a network when it is built and names the rule."""
    from rohm_b200 import RohmB200Error
    m, _ = _build(False, cuda_device, mid_dim=128)
    batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(1, 16, 3).items()}
    batch['x_t'] = torch.zeros(1, 16, 13, device=cuda_device)
    with pytest.raises(RohmB200Error, match=r"mid_dim \(128\) must be a positive multiple of 256"):
        m(batch, torch.zeros(1, dtype=torch.long, device=cuda_device))


def test_config1_trajnet_50_steps_matches_reference_golden(nets, cuda_device):
    """BASELINE configs[0]: TrajNet vanilla, 1 clip, 144 frames, 50 DDPM steps via eval_losses (noise replayed)."""
    m, sd = nets[False]
    g = golden("sampling.npz")
    B, T, bseed, nseed, steps = [int(v) for v in g["traj50_meta"]]
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    d = diffusion.create_gaussian_diffusion(args, diffusion, diffusion.SpacedDiffusionTrajNet, steps, '', cuda_device)
    tape = NoiseTape(nseed, cuda_device)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, bseed).items()}
    loss, y = d.eval_losses(model=m, batch=batch, shape=[B, T, 13], progress=False, clip_denoised=False,
                            timestep_respacing='', cond_fn_with_grad=True, compute_loss=False, smplx_model=None)
    assert loss is None
    err = float((y.cpu() - torch.from_numpy(g["traj50_out"])).abs().max())
    assert err < TOL, err


def test_control_chain_properties_at_config3_size(nets, cuda_device):
    """BASELINE configs[2] size (64 clips, TrajControl) on a 20-step respaced chain: determinism under a seed, final
    sample == pred_xstart, spot check of the last denoiser call against the oracle."""
    m, sd = nets[True]
    B, T = 64, 144
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    d = diffusion.create_gaussian_diffusion(args, diffusion, diffusion.SpacedDiffusionTrajNet, 1000, 'ddim20', cuda_device)
    batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, 5, control=True).items()}
    outs = []
    for _ in range(2):
        torch.manual_seed(99)
        last = None
        for o in d.p_sample_loop_progressive(m, batch, [B, T, 13], clip_denoised=False, cond_fn_with_grad=True):
            last = o
        outs.append(last)
    assert torch.equal(outs[0]['sample'], outs[1]['sample'])
    assert torch.equal(outs[0]['sample'], outs[0]['pred_xstart'])
    x_in = outs[0]['x_t'][:2].cpu()
    ref = trajnet_oracle.trajnet_forward(sd, x_in, batch['cond'][:2].cpu(), torch.zeros(2, dtype=torch.long),
                                         batch['control_cond'][:2].cpu())
    assert float((outs[0]['sample'][:2].cpu() - ref).abs().max()) < TOL


def test_recycled_condition_addresses_are_not_mistaken_for_the_cached_ones(nets, cuda_device):
    """Regression (round-1 advisor finding): cond / control_cond rebuilt per batch can reuse the freed tensors' addresses and
    version counts; the cached condition pyramid must follow the tensor objects."""
    m, sd = nets[True]
    B, T = 2, 32
    x = torch.randn(B, T, 13, generator=torch.Generator().manual_seed(1))
    ts = torch.tensor([3, 40])
    outs, ptrs = [], []
    for k in range(4):
        b = {kk: v.to(cuda_device) for kk, v in synthetic.trajnet_batch(B, T, 70 + k, control=True).items()}
        b['x_t'] = x.to(cuda_device)
        ptrs.append((b['cond'].data_ptr(), b['control_cond'].data_ptr()))
        y = m(b, ts.to(cuda_device)).cpu()
        ref = trajnet_oracle.trajnet_forward(sd, x, b['cond'].cpu(), ts, control_cond=b['control_cond'].cpu())
        assert float((y - ref).abs().max()) < TOL, k
        outs.append(y)
        del b
    assert len(set(ptrs)) < 4, "allocator did not recycle the addresses: the scenario was not exercised"
    for k in range(1, 4):
        assert float((outs[k] - outs[k - 1]).abs().max()) > 1e-3


def test_eval_losses_default_compute_loss(nets, cuda_device):
    """eval_losses with its default compute_loss=True (test_trajnet.py:154) returns the reference's loss dictionary."""
    from rohm_b200.body_model import BodyModel
    m, _ = nets[False]
    B, T = 2, 32
    a = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    d = diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionTrajNet, 5, '', cuda_device)
    b = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, 5).items()}
    m.device = cuda_device
    loss, out = d.eval_losses(model=m, batch=b, shape=[B, T, 13], progress=False, clip_denoised=False,
                              cond_fn_with_grad=True, smplx_model=BodyModel.create('', device=cuda_device))
    assert out.shape == (B, T, 13) and 'loss' in loss and float(loss['loss_root_pos_global_from_rel_traj']) == 0.0
    assert all(bool(torch.isfinite(v)) for v in loss.values())


def test_launch_switches_do_not_change_the_result(nets, cuda_device):
    """Programmatic dependent launch and CUDA-graph replay only change how the kernels are scheduled: the forward must be
    bit-identical with either switched off (rohm_trajnet_set_option 1 / 0)."""
    m, _ = nets[True]
    B, T = 5, 144
    gen = torch.Generator().manual_seed(31)
    batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, 3, control=True).items()}
    batch['x_t'] = torch.randn(B, T, 13, generator=gen).to(cuda_device)
    ts = torch.randint(0, 1000, (B,), generator=gen).to(cuda_device)
    ref = m(batch, ts).clone()
    eng = m._engine
    try:
        for option in (1, 0):
            assert eng.lib.rohm_trajnet_set_option(eng.handle, option, 0) == 0
            assert torch.equal(m(batch, ts), ref)
            assert eng.lib.rohm_trajnet_set_option(eng.handle, option, 1) == 0
            assert torch.equal(m(batch, ts), ref)
    finally:
        eng.lib.rohm_trajnet_set_option(eng.handle, 0, 1)
        eng.lib.rohm_trajnet_set_option(eng.handle, 1, 1)


@pytest.mark.parametrize("env", [{"ROHM_B200_TRAJ_SPLITK": "0"}, {"ROHM_B200_TRAJ_PARALLEL": "0"},
                                 {"ROHM_B200_TRAJ_SPLITK": "0", "ROHM_B200_TRAJ_PARALLEL": "0"}])
def test_split_k_and_in_kernel_statistics_agree_with_the_single_pass_paths(nets, cuda_device, monkeypatch, env):
    """The default engine cuts the deep-level convolutions into K ranges (fp32 partials added in split order by the GroupNorm
    kernel, which takes every GroupNorm's statistics itself) and runs its graph on several streams.  The engine built with
    ROHM_B200_TRAJ_SPLITK=0 (one K loop per tile, the GroupNorm kernel reading the one fp32 result) computes the same function
    with a different summation order: it must agree with the default and with the oracle far inside the parity tolerance.
    ROHM_B200_TRAJ_PARALLEL=0 (one serial chain) only changes the scheduling, so on its own it must be bit-identical.  Checked
    at a batch where the split path uses 3-6 ranges (64 clips) and at one where it uses 8 (2 clips)."""
    _, sd = nets[True]
    for B, seed in ((2, 51), (64, 52)):
        T = 144
        gen = torch.Generator().manual_seed(seed)
        b = synthetic.trajnet_batch(B, T, seed, control=True)
        x = torch.randn(B, T, 13, generator=gen)
        ts = torch.randint(0, 1000, (B,), generator=gen)
        batch = {k: v.to(cuda_device) for k, v in b.items()}
        batch['x_t'] = x.to(cuda_device)
        default_m, _ = _build(True, cuda_device)
        out_default = default_m(batch, ts.to(cuda_device)).cpu()
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        other_m, _ = _build(True, cuda_device)
        out_other = other_m(batch, ts.to(cuda_device)).cpu()
        for k in env:
            monkeypatch.delenv(k)
        if "ROHM_B200_TRAJ_SPLITK" not in env:
            assert torch.equal(out_default, out_other), "scheduling alone must not change the result"
        scale = float(out_default.abs().max())
        assert float((out_default - out_other).abs().max()) < 2e-5 * max(1.0, scale)
        if B == 2:
            with torch.no_grad():
                ref = trajnet_oracle.trajnet_forward(sd, x, b['cond'], ts, control_cond=b['control_cond'])
            assert float((out_default - ref).abs().max()) < TOL and float((out_other - ref).abs().max()) < TOL


def test_fused_sample_step_equals_the_unfused_chain(nets, cuda_device, monkeypatch):
    """One graph launch per step (TrajNet forward + in-kernel-noise update, rohm_trajnet_sample_step) == forward,
    torch.randn_like, update as separate launches: bit for bit, vanilla and TrajControl, for an un-respaced and a respaced
    schedule, through p_sample_loop and through eval_losses' cond_fn_with_grad route; torch's generator ends in the same state."""
    gen = torch.cuda.default_generators[cuda_device.index]
    a = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    for control in (False, True):
        m, _ = nets[control]
        B, T = 3, 144
        batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, 9, control=control).items()}
        for steps, resp in ((1000, 'ddim6'), (6, '')):
            d = diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionTrajNet, steps, resp, cuda_device)
            for with_grad in (False, True):
                outs, offs = [], []
                for fused in (True, False):
                    monkeypatch.setattr(diffusion, "_FUSED_STEP", fused)
                    torch.manual_seed(77)
                    outs.append(d.p_sample_loop(m, dict(batch), [B, T, 13], clip_denoised=False, cond_fn_with_grad=with_grad))
                    offs.append(gen.get_offset())
                assert torch.equal(outs[0], outs[1]) and offs[0] == offs[1], (control, steps, resp, with_grad)
                assert bool(torch.isfinite(outs[0]).all())
