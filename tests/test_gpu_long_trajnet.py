"""GPU: TrajNet, the inter-round glue and the round pipeline on clips longer than 1024 frames.

* The cluster GroupNorm + Mish kernel (gn_mish_split_kernel, rohm_b200/csrc/groupnorm.cu) through its test probe,
  against a float64 GroupNorm + Mish, for every cluster size.
* TrajNet / TrajNet+TrajControl forwards up to 4992 frames against oracle/trajnet_oracle, and the frame limit.
* traj_repr_from_joints / traj_to_full_repr (a cluster of ceil(T / 1024) CTAs per clip) up to 4992 frames with planted
  degenerate frames, against oracle/glue_oracle.
* pipeline.run_rounds at 1009 and 4993 raw frames (TrajNet at 1008 / 4992, PoseNet at 1007 / 4991)."""
import argparse

import numpy as np
import pytest
import torch

import group_norm_probe as gp
from helpers import NoiseTape, TOL
from oracle import diffusion_oracle as do
from oracle import glue_oracle as go
from oracle import pipeline_oracle, trajnet_oracle
from rohm_b200 import RohmB200Error, diffusion, glue, pipeline, synthetic
from rohm_b200.body_model import BodyModel
from rohm_b200.trajnet import TrajNet

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # fp32 unit roundoff
SENTINEL = 1234.0  # exact in fp16 too


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm + Mish kernel
# ---------------------------------------------------------------------------------------------------------------------
def _mish(x):
    return x * torch.tanh(torch.nn.functional.softplus(x))


def _gn_reference(part, bias, gamma, beta, tp, r1, r2, B, Tp, TL, C, groups=8):
    """float64 GroupNorm + Mish on the real rows, and the per-element error bound of the kernel's fp32 arithmetic.

    Derivation (u = 2^-24, s = splits):
      y      = bias + s partials added in fp32:            |dy| <= (s + 1) u S,  S = |bias| + sum |partial|
      mu, var: double sums of the fp32 y, so they see dy only; mu and rstd are rounded to fp32 (u each), and a mean
               error dmu = max |dy| shifts every element by at most that much
      z      = (y - mu) rstd gamma + beta in fp32 (3 roundings):
               |dz| <= rstd |gamma| (|dy| + max|dy| + 4 u (|y| + |mu|)) + |z - beta| max|dy| rstd + 2 u |z|
      mish   : |mish'| <= 1.1, and its fp32 evaluation (expf, log1pf, tanhf, 2 products) adds <= 8 u |mish| + 4 u
      + tp + r1 + r2: one rounding per add, <= 3 u |out|
    The bound is that sum, times 2 for the terms second order in u."""
    v = lambda t: t.view(B, Tp, C)[:, :TL].double()
    parts = [v(p) for p in part]
    y = v(bias.view(1, C).expand(B * Tp, C).contiguous()) + sum(parts)
    S = bias.double().abs().view(1, 1, C) + sum(p.abs() for p in parts)
    dy = (len(parts) + 1) * U * S
    gs = C // groups
    yg = y.view(B, TL, groups, gs)
    mu = yg.mean(dim=(1, 3), keepdim=True)
    var = ((yg - mu) ** 2).mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    ga, be = gamma.double().view(1, 1, groups, gs), beta.double().view(1, 1, groups, gs)
    z = (yg - mu) * rstd * ga + be
    dyg = dy.view(B, TL, groups, gs)
    dmax = dyg.amax(dim=(1, 3), keepdim=True)
    dz = rstd * ga.abs() * (dyg + dmax + 4 * U * (yg.abs() + mu.abs())) + (z - be).abs() * dmax * rstd + 2 * U * z.abs()
    m = _mish(z)
    out = m.clone()
    if tp is not None:
        out = out + tp[:, :C].double().view(B, 1, groups, gs)
    for r in (r1, r2):
        if r is not None:
            out = out + v(r).view(B, TL, groups, gs)
    bound = 2 * (1.1 * dz + 8 * U * m.abs() + 4 * U + 3 * U * out.abs())
    return out.view(B, TL, C), bound.view(B, TL, C)


def _gn_case(dev, T, C, div, splits, extras, f16, gen):
    B = 2
    L = div.bit_length() - 1
    TL, Tp = T // div, (T + 32) >> L
    rows = B * Tp
    rnd = lambda *s: torch.randn(*s, generator=gen).to(dev)
    part = rnd(splits, rows * C)
    bias, gamma, beta = rnd(C) * 0.5, 1.0 + 0.2 * rnd(C), 0.3 * rnd(C)
    tp = rnd(B, C + 4) if extras else None
    r1 = rnd(rows * C) if extras else None
    r2 = rnd(rows * C) if extras else None
    pair_dtype = torch.float16 if f16 else torch.float32
    return dict(B=B, TL=TL, Tp=Tp, rows=rows, part=part, bias=bias, gamma=gamma, beta=beta, tp=tp, r1=r1, r2=r2,
                pair_dtype=pair_dtype, splits=splits, f16=f16, C=C)


def _gn_run(case, n, reps=1):
    c = case
    extra = 64  # elements past the matrix: must keep the sentinel
    dev = c["part"].device
    out = torch.full((c["rows"] * c["C"] + extra,), SENTINEL, device=dev)
    hi = torch.full((c["rows"] * c["C"] + extra,), SENTINEL, device=dev, dtype=c["pair_dtype"])
    lo = torch.full_like(hi, SENTINEL)
    rc = gp.group_norm(c["part"], c["splits"], c["rows"] * c["C"], c["bias"], c["gamma"], c["beta"], c["tp"],
                       c["C"] + 4, c["r1"], c["r2"], out, hi, lo, c["C"], c["Tp"], c["TL"], c["B"], n, c["f16"], reps=reps)
    torch.cuda.synchronize()
    assert rc == 0, rc
    return out, hi, lo


@pytest.mark.parametrize("T", [16, 1520, 1536, 4992])
@pytest.mark.parametrize("C,div", [(64, 1), (32, 1), (128, 2), (512, 16)])
def test_cluster_group_norm_matches_float64(cuda_device, T, C, div):
    """Every option of the kernel (1 / 3 / 8 split-K partials, time projection and both residuals on or off, fp16 and
    tf32 operand pairs besides the fp32 output) at each cluster size n = 1, 2, 4, 8 against float64: real rows within
    the derived bound, pad rows exactly zero in every output, the sentinel past the matrix untouched, every n within the
    bound of n = 1, and a repeated launch bit-identical."""
    gen = torch.Generator().manual_seed(T * 31 + C)
    worst = 0.0
    for splits in (1, 3, 8):
        for extras in (False, True):
            for f16 in (1, 0):
                c = _gn_case(cuda_device, T, C, div, splits, extras, f16, gen)
                B, TL, Tp, rows = c["B"], c["TL"], c["Tp"], c["rows"]
                ref, bound = _gn_reference(c["part"], c["bias"], c["gamma"], c["beta"], c["tp"], c["r1"], c["r2"], B,
                                           Tp, TL, C)
                got = {}
                for n in (1, 2, 4, 8):
                    out, hi, lo = _gn_run(c, n)
                    m = rows * C
                    for buf in (out, hi, lo):
                        assert bool((buf[m:].float() == SENTINEL).all()), (n, "wrote past the matrix")
                        pad = buf[:m].view(B, Tp, C)[:, TL:]
                        assert bool((pad == 0).all()), (n, "pad rows must be zero")
                    o = out[:m].view(B, Tp, C)[:, :TL].double()
                    err = (o - ref).abs()
                    assert bool((err <= bound).all()), (splits, extras, f16, n, float(err.max()), float(bound.max()))
                    worst = max(worst, float((err / bound).max()))
                    pair = hi[:m].view(B, Tp, C)[:, :TL].double() + lo[:m].view(B, Tp, C)[:, :TL].double()
                    if f16:  # two fp16 halves carry 22 bits; below 2^-14 the halves are subnormal (2^-25 absolute)
                        assert bool(((pair - o).abs() <= 2.0 ** -21 * o.abs() + 2.0 ** -24).all()), n
                    else:  # tf32 hi + the exact fp32 remainder
                        assert torch.equal(pair, o), n
                    got[n] = o
                for n in (2, 4, 8):
                    assert bool(((got[n] - got[1]).abs() <= 2 * bound).all()), n
                again = _gn_run(c, 8)[0][:rows * C].view(B, Tp, C)[:, :TL].double()
                assert torch.equal(again, got[8])
    print(f"GroupNorm T={T} C={C} T_L={T // div}: worst error / bound = {worst:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# TrajNet forwards
# ---------------------------------------------------------------------------------------------------------------------
def _build(control, dev, seed=2):
    m = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=control, device=dev,
                dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
    sd = {k: v.cpu() for k, v in synthetic.synth_state_dict(m, seed).items()}
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


@pytest.fixture(scope="module")
def nets(cuda_device):
    return {False: _build(False, cuda_device), True: _build(True, cuda_device)}


def _inputs(B, T, control, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 13, generator=gen)
    batch = synthetic.trajnet_batch(B, T, seed, control=control)
    ts = torch.randint(0, 1000, (B,), generator=gen)
    return x, batch, ts


@pytest.mark.parametrize("control", [False, True])
@pytest.mark.parametrize("B,T", [(2, 1520), (2, 1536), (1, 2000), (1, 4992)])
def test_long_forward_matches_oracle(nets, cuda_device, control, B, T):
    """1536 frames is the first length whose level-0 GroupNorm groups exceed one CTA's default shared memory (clusters of
    2); 4992 uses clusters of 4.  At 4992 the forward is also held to a float64 oracle."""
    m, sd = nets[control]
    x, batch, ts = _inputs(B, T, control, 11 * T + B)
    gb = {k: v.to(cuda_device) for k, v in batch.items()}
    gb['x_t'] = x.to(cuda_device)
    y = m(gb, ts.to(cuda_device)).cpu()
    with torch.no_grad():
        ref = trajnet_oracle.trajnet_forward(sd, x, batch['cond'], ts, batch.get('control_cond'))
    err = float((y - ref).abs().max())
    print(f"TrajNet control={control} B={B} T={T}: max |cuda - oracle| = {err:.3e}")
    assert err < TOL, err
    if T == 4992:
        with torch.no_grad():
            ref64 = trajnet_oracle.trajnet_forward(sd, x.double(), batch['cond'].double(), ts,
                                                   None if not control else batch['control_cond'].double())
        err64 = float((y.double() - ref64).abs().max())
        print(f"TrajNet control={control} B={B} T={T}: max |cuda - float64 oracle| = {err64:.3e}")
        assert err64 < TOL, err64


def test_serial_graph_equals_multi_stream_graph_at_2000_frames(nets, cuda_device, monkeypatch):
    """Cluster launches capture into the multi-stream forward graph and the serial one (ROHM_B200_TRAJ_PARALLEL=0):
    only the scheduling differs, so the results are bit-identical."""
    B, T = 1, 2000
    x, batch, ts = _inputs(B, T, True, 5)
    gb = {k: v.to(cuda_device) for k, v in batch.items()}
    gb['x_t'] = x.to(cuda_device)
    m, _ = _build(True, cuda_device)
    y_par = m(gb, ts.to(cuda_device)).clone()
    monkeypatch.setenv("ROHM_B200_TRAJ_PARALLEL", "0")
    m_ser, _ = _build(True, cuda_device)
    y_ser = m_ser(gb, ts.to(cuda_device))
    assert torch.equal(y_par, y_ser)


def test_fused_sample_step_equals_the_unfused_chain_at_2000_frames(nets, cuda_device, monkeypatch):
    """rohm_trajnet_sample_step (forward + in-kernel-noise update as one graph) == forward, torch.randn_like, update:
    bit for bit, with torch's generator left at the same offset."""
    gen = torch.cuda.default_generators[cuda_device.index]
    a = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    B, T = 1, 2000
    for control in (False, True):
        m, _ = nets[control]
        batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, 9, control=control).items()}
        d = diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionTrajNet, 4, '', cuda_device)
        outs, offs = [], []
        for fused in (True, False):
            monkeypatch.setattr(diffusion, "_FUSED_STEP", fused)
            torch.manual_seed(77)
            outs.append(d.p_sample_loop(m, dict(batch), [B, T, 13], clip_denoised=False, cond_fn_with_grad=False))
            offs.append(gen.get_offset())
        assert torch.equal(outs[0], outs[1]) and offs[0] == offs[1], control
        assert bool(torch.isfinite(outs[0]).all())


def test_over_long_clip_is_refused_with_the_rule(cuda_device):
    """A clip whose GroupNorm group does not fit 8 CTAs' shared memory (about 58 000 frames at mid_dim 512) is refused by
    rohm_trajnet_create before it allocates, with the rule in the message, and no engine is left behind."""
    m, _ = _build(False, cuda_device)
    T = 60000
    batch = {'x_t': torch.zeros(1, T, 13, device=cuda_device), 'cond': torch.zeros(1, T, 13, device=cuda_device)}
    with pytest.raises(RohmB200Error, match=r"frames \(60000\) exceeds \d+ at mid_dim 512: a GroupNorm group"):
        m(batch, torch.zeros(1, dtype=torch.long, device=cuda_device))
    assert m._engine is None


# ---------------------------------------------------------------------------------------------------------------------
# Inter-round glue
# ---------------------------------------------------------------------------------------------------------------------
def _joints(B, T, seed):
    """Joint positions whose hip and shoulder axes stay well away from vertical, random global orientations and
    translations.  The forward directions stay within 135 degrees of +y: the root quaternion's w = 1 + cos(angle to +y)
    loses its precision in fp32 as that angle approaches 180 degrees, the degenerate direction the planted NaN frames hit
    exactly."""
    g = torch.Generator().manual_seed(seed)
    P = 0.5 * torch.randn(B, T, 22, 3, generator=g)
    th = 0.75 * np.pi * (2 * torch.rand(B, T, generator=g) - 1)
    axis = torch.stack([torch.cos(th), torch.sin(th), 0.1 * torch.randn(B, T, generator=g)], dim=-1)
    P[:, :, 1] = P[:, :, 2] + 0.3 * axis + 0.01 * torch.randn(B, T, 3, generator=g)
    P[:, :, 17] = P[:, :, 16] + 0.4 * axis + 0.01 * torch.randn(B, T, 3, generator=g)
    go_aa = 0.8 * torch.randn(B, T, 3, generator=g)
    tr = torch.randn(B, T, 3, generator=g)
    return P, go_aa, tr


def _plant_nan(P, b, t):
    """Frame t of clip b faces exactly -y: qbetween((0, -1, 0), (0, 1, 0)) is 0 / 0."""
    P[b, t, 2] = P[b, t, 1] + torch.tensor([0.3, 0.0, 0.0])
    P[b, t, 16] = P[b, t, 17] + torch.tensor([0.4, 0.0, 0.0])


@pytest.mark.parametrize("T", [1024, 1025, 2048, 4992])
def test_traj_repr_from_joints_long_clips_with_degenerate_frames(cuda_device, T):
    """Clip 0: a NaN frame past 1024 (mid-clip when T = 1024); clip 1: a NaN frame on a CTA boundary (its predecessor in
    the previous CTA); clip 2: two NaN frames, only the first repaired; clip 3: NaN at frame 0 (repaired from frame T - 1,
    in the last CTA, then pinned).  NaN positions must match the oracle exactly."""
    n = (T + 1023) // 1024
    rows = (T + n - 1) // n
    P, go_aa, tr = _joints(4, T, T)
    _plant_nan(P, 0, min(1500, T - 2) if T > 1025 else T // 2)
    _plant_nan(P, 1, rows if rows < T else T // 3)
    _plant_nan(P, 2, T // 4)
    _plant_nan(P, 2, T - 3)
    _plant_nan(P, 3, 0)
    dev = cuda_device
    m0, s1 = torch.zeros(294, device=dev), torch.ones(294, device=dev)
    out = glue.traj_repr_from_joints(P.to(dev), go_aa.to(dev), tr.to(dev), m0, s1).cpu().double()
    for b in range(4):
        ref = torch.from_numpy(go.traj_repr_from_joints(P[b].numpy(), go_aa[b].numpy(), tr[b].numpy()))
        assert torch.equal(torch.isnan(out[b]), torch.isnan(ref)), b
        fin = ~torch.isnan(ref)
        err = float((out[b][fin] - ref[fin]).abs().max())
        assert err < TOL, (b, err)
    assert bool(torch.isnan(out[2]).any()), "the second NaN frame stays NaN"


@pytest.fixture(scope="module")
def body(cuda_device):
    return BodyModel.create('', device=cuda_device, seed=0), synthetic.smplx_like_model(0)


@pytest.mark.parametrize("T", [1024, 1025, 2048, 4992])
def test_traj_to_full_repr_long_clips_matches_oracle(body, cuda_device, T):
    bm, model = body
    B = 1
    ds_p = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_t = synthetic.make_dataset('traj', seed=4, realistic_std=True)
    clean = synthetic.plausible_motion(B, T, T, ds_t)[:, :, 0].permute(0, 2, 1).contiguous()
    g = torch.Generator().manual_seed(T)
    sel = [0, 2, 3, 6] + list(range(7, 13)) + list(range(16, 19))
    traj = clean[..., sel] + 0.05 * torch.randn(B, T, 13, generator=g)
    comp, full = glue.traj_to_full_repr(bm, traj.to(cuda_device), clean.to(cuda_device), ds_t, ds_p)
    comp_o, full_o = go.traj_to_full_repr(traj, clean, ds_t.Mean, ds_t.Std, ds_p.Mean, ds_p.Std, model)
    assert torch.equal(comp.cpu(), comp_o)
    err = float((full.cpu() - full_o).abs().max())
    print(f"traj_to_full_repr T={T}: max |cuda - oracle| = {err:.3e}")
    assert err < TOL, err


def test_glue_refuses_clips_past_8192_frames(body, cuda_device):
    bm, _ = body
    dev = cuda_device
    T = 8193
    m0, s1 = torch.zeros(294, device=dev), torch.ones(294, device=dev)
    z = torch.zeros(1, T, 22, 3, device=dev)
    with pytest.raises(RohmB200Error, match=r"T=8193 frames exceeds 8192"):
        glue.traj_repr_from_joints(z, torch.zeros(1, T, 3, device=dev), torch.zeros(1, T, 3, device=dev), m0, s1)
    ds = synthetic.make_dataset('pose')
    with pytest.raises(RohmB200Error, match=r"T=8193 frames exceeds 8192"):
        glue.traj_to_full_repr(bm, torch.zeros(1, T, 13, device=dev), torch.zeros(1, T, 294, device=dev), ds, ds)


# ---------------------------------------------------------------------------------------------------------------------
# Round pipeline
# ---------------------------------------------------------------------------------------------------------------------
POSE_RESPACING = "3" + ",0" * 19  # PoseNet respaced to 3 steps of 1000
TRAJ_STEPS = 4


def _pipeline_models(dev):
    from test_gpu_pipeline import _diffusions, _models
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    mp, mt, mc, sd_p, sd_t, sd_c = _models(dev, ds_pose, ds_traj)
    dp, dt, dc = _diffusions(dev, TRAJ_STEPS, pose_steps=1000, pose_respacing=POSE_RESPACING)
    return ds_pose, ds_traj, (mp, mt, mc), (sd_p, sd_t, sd_c), (dp, dt, dc)


def _run_rounds(dev, models, diffs, ds_pose, ds_traj, body, B, frames, rounds, seeds, on_round=None):
    dp, dt, dc = diffs
    tape_p, tape_t = NoiseTape(seeds[0], dev), NoiseTape(seeds[1], dev)
    dp._randn, dp._randn_like = tape_p.randn, tape_p.randn_like
    for d in (dt, dc):
        d._randn, d._randn_like = tape_t.randn, tape_t.randn_like
    pose, traj = synthetic.pipeline_batches(B, seeds[2], ds_pose, frames=frames, device=dev)
    args = pipeline.make_args(sample_iter=rounds, mask_scheme='lower')
    return pipeline.run_rounds(args, *models, dp, dt, dc, ds_pose, ds_traj, body, pose, traj, on_round=on_round)


def test_run_rounds_at_1009_raw_frames_matches_oracle_stage_by_stage(cuda_device):
    """2 clips, 2 rounds (the second through TrajControl), TrajNet at 1008 frames, PoseNet at 1007 with the in-loop
    guidance.  Round k + 1 is conditioned on the oracle's round-k PoseNet output (the guided chain is chaotic, see
    test_full_pipeline_replays_reference_golden), so every stage is compared on the oracle's own inputs."""
    dev = cuda_device
    B, frames, rounds, seeds = 2, 1008, 2, (21, 22, 23)
    ds_pose, ds_traj, models, sds, diffs = _pipeline_models(dev)
    body_o = synthetic.smplx_like_model(0)
    pose_c, traj_c = synthetic.pipeline_batches(B, seeds[2], ds_pose, frames=frames)
    ref = pipeline_oracle.run_rounds(*sds, ds_pose, ds_traj, body_o, pose_c, traj_c, 1000, TRAJ_STEPS, rounds,
                                     NoiseTape(seeds[0]), NoiseTape(seeds[1]), pose_respacing=POSE_RESPACING)
    body = BodyModel.create('', device=dev, seed=0)
    seen = []

    def on_round(it, val_traj, traj_full, cond, val_pose):
        seen.append({"val_traj": val_traj.detach().cpu(), "cond": cond.detach().cpu()})
        return ref[it]["val_pose"].to(dev)

    _run_rounds(dev, models, diffs, ds_pose, ds_traj, body, B, frames, rounds, seeds, on_round)
    tp, mp_ = do.create_diffusion('cosine', 1000, POSE_RESPACING)
    dp = diffs[0]
    mean_p, std_p = torch.from_numpy(ds_pose.Mean), torch.from_numpy(ds_pose.Std)
    for it in range(rounds):
        e_traj = float((seen[it]["val_traj"] - ref[it]["val_traj"]).abs().max())
        _, tf_full = glue.traj_to_full_repr(body, ref[it]["val_traj"].to(dev), traj_c['motion_repr_clean'].to(dev),
                                            ds_traj, ds_pose)
        e_glue = float((tf_full.cpu() - ref[it]["traj_full"]).abs().max())
        # the final PoseNet step (t = 0, guided) from the oracle's round output as x_1, on the oracle's condition
        x1, cond = ref[it]["val_pose"], ref[it]["cond"]
        nz = NoiseTape(99).randn(*x1.shape)
        want, _ = pipeline_oracle.posenet_guided_step(tp, mp_, 0, x1, cond, sds[0], mean_p, std_p, body_o, nz)
        dp._randn_like = lambda x, _n=nz.to(dev): _n
        got = dp.p_sample_with_grad(models[0], {'cond': cond.to(dev)}, x1.to(dev), dp._t_rows(B, dev)[0],
                                    clip_denoised=False, grad_type='amass', _step_index=0)['sample'].cpu()
        e_pose = float((got - want).abs().max())
        print(f"run_rounds 2 x 1009 raw frames, round {it}: val_traj {e_traj:.3e}, glue (stage-wise) {e_glue:.3e}, "
              f"final PoseNet step {e_pose:.3e}")
        assert e_traj < TOL and e_glue < TOL and e_pose < TOL, (it, e_traj, e_glue, e_pose)


def test_run_rounds_at_4993_raw_frames(cuda_device):
    """1 clip at the longest clip PoseNet's positional table allows (TrajNet 4992 frames, PoseNet 4991), 2 rounds: round
    0's TrajNet chain and glue against the oracle, a finite PoseNet output, and two runs bit-identical."""
    dev = cuda_device
    B, frames, rounds, seeds = 1, 4992, 2, (31, 32, 33)
    ds_pose, ds_traj, models, sds, diffs = _pipeline_models(dev)
    body = BodyModel.create('', device=dev, seed=0)
    seen = []

    def on_round(it, val_traj, traj_full, cond, val_pose):
        seen.append({"val_traj": val_traj.detach().cpu(), "traj_full": traj_full.detach().cpu()})

    runs = [_run_rounds(dev, models, diffs, ds_pose, ds_traj, body, B, frames, rounds, seeds, on_round) for _ in range(2)]
    out_pose, out_traj, _ = runs[0]
    assert out_pose.shape == (B, 294, 1, frames - 1) and out_traj.shape == (B, frames, 13)
    assert bool(torch.isfinite(out_pose).all())
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    # round 0 through the oracle: the TrajNet chain on the same noise, then the glue stage on the oracle's own output
    _, traj_c = synthetic.pipeline_batches(B, seeds[2], ds_pose, frames=frames)
    tape = NoiseTape(seeds[1])
    tt, mt_ = do.create_diffusion('cosine', TRAJ_STEPS, '')
    x_T = tape.randn(B, frames, 13)
    fn = lambda x, t: trajnet_oracle.trajnet_forward(sds[1], x, traj_c['cond'], torch.full((B,), t, dtype=torch.long))
    with torch.no_grad():
        val_traj, _ = do.p_sample_loop(tt, mt_, fn, x_T, lambda i: tape.randn_like(x_T))
    _, full_o = go.traj_to_full_repr(val_traj, traj_c['motion_repr_clean'], ds_traj.Mean, ds_traj.Std, ds_pose.Mean,
                                     ds_pose.Std, synthetic.smplx_like_model(0))
    _, full_c = glue.traj_to_full_repr(body, val_traj.to(dev), traj_c['motion_repr_clean'].to(dev), ds_traj, ds_pose)
    e_traj = float((seen[0]["val_traj"] - val_traj).abs().max())
    e_glue = float((full_c.cpu() - full_o).abs().max())
    print(f"run_rounds 1 x 4993 raw frames, round 0: val_traj {e_traj:.3e}, glue (stage-wise) {e_glue:.3e}")
    assert e_traj < TOL and e_glue < TOL, (e_traj, e_glue)
