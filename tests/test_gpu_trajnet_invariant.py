"""Batch-invariant TrajNet and TrajNet + TrajControl (TrajNet.batch_invariant = True): each recording's real frames are the
same bits alone in a fresh engine at its own length, in ragged batches padded to other lengths, permuted, and in an engine
created for 64 clips, while the default mode differs between those engines; the benchmark shape keeps the default bits; the
clip-slice GroupNorm instance reproduces the default kernel on uniform clips; parity with the oracle and the golden file;
sampling with per-recording generators, shards, and two guided rounds against each recording alone; refusals."""
import argparse

import pytest
import torch

from helpers import TOL, golden
from oracle import trajnet_oracle
from rohm_b200 import diffusion, pipeline, synthetic
from rohm_b200._lib import PRECISION_F16X2, PRECISION_TF32, PRECISION_TF32X3, RohmB200Error
from rohm_b200.trajnet import TrajNet
from test_gpu_noise_streams import _clone, _gens

pytestmark = pytest.mark.gpu

LENGTHS = [16, 144, 400, 1536, 2000, 4992]  # 1536 and up: GroupNorm clusters of 2 to 4 CTAs at level 0 alone


def _build(control, dev, seed=2):
    m = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=control, device=dev,
                dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
    sd = {k: v.cpu() for k, v in synthetic.synth_state_dict(m, seed).items()}
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


@pytest.fixture(scope="module")
def nets(cuda_device):
    return {False: _build(False, cuda_device), True: _build(True, cuda_device)}


def _bits(t):
    return t.contiguous().view(torch.int32)


def _recordings(lengths, control, seed):
    """One input per recording at its own length: x_t, cond, control_cond and a timestep."""
    gen = torch.Generator().manual_seed(seed)
    recs = []
    for i, n in enumerate(lengths):
        b = synthetic.trajnet_batch(1, n, seed + i, control=control)
        r = {'x_t': torch.randn(1, n, 13, generator=gen), 'cond': b['cond']}
        if control:
            r['control_cond'] = b['control_cond']
        recs.append((r, int(torch.randint(0, 1000, (1,), generator=gen))))
    return recs


def _batch(recs, idx, T, dev, lengths=True):
    """Recordings `idx` padded to T frames (NaN past each recording: never read) with batch['lengths']."""
    out = {}
    for k in recs[0][0]:
        rows = []
        for i in idx:
            v = recs[i][0][k]
            pad = torch.full((1, T - v.shape[1], v.shape[2]), float('nan'))
            rows.append(torch.cat([v, pad], 1))
        out[k] = torch.cat(rows).to(dev)
    if lengths:
        out['lengths'] = torch.tensor([recs[i][0]['x_t'].shape[1] for i in idx], device=dev)
    return out, torch.tensor([recs[i][1] for i in idx], device=dev)


def _runs(m, recs, dev):
    """Each recording's real frames in every run (a)-(e), as a list per recording."""
    n_of = [r[0]['x_t'].shape[1] for r in recs]
    res = [[] for _ in recs]
    for i, (r, t) in enumerate(recs):  # (a) alone, fresh engine at its own T, B = 1, no lengths
        m.invalidate_engine()
        res[i].append(m({k: v.to(dev) for k, v in r.items()}, torch.tensor([t], device=dev))[0].clone())
        assert m._engine.max_batch == 1 and m._engine.frames == n_of[i]
    Tmax = max(n_of)
    everyone = list(range(len(recs)))
    m.invalidate_engine()
    b, ts = _batch(recs, everyone, Tmax, dev)  # (b) one ragged batch padded to the longest
    out = m(b, ts).clone()
    for i, n in enumerate(n_of):
        assert bool((out[i, n:] == 0).all()), f"recording {i}: padded frames are not zero"
        res[i].append(out[i, :n])
    perm = everyone[::-1][1:] + everyone[-1:]  # (c) permuted
    b, ts = _batch(recs, perm, Tmax, dev)
    out = m(b, ts)
    for j, i in enumerate(perm):
        res[i].append(out[j, :n_of[i]])
    short = [i for i in everyone if n_of[i] <= 2000]  # (d) the recordings of <= 2000 frames padded to 2000
    for fresh in (True, False):  # then (e): the same in an engine first created for 64 clips
        m.invalidate_engine()
        if not fresh:
            big, bts = _batch([recs[short[k % len(short)]] for k in range(64)], range(64), 2000, dev)
            m(big, bts)
            assert m._engine.max_batch == 64
        b, ts = _batch(recs, short, 2000, dev)
        out = m(b, ts)
        assert m._engine.max_batch == (len(short) if fresh else 64)
        for j, i in enumerate(short):
            res[i].append(out[j, :n_of[i]])
    return res


@pytest.mark.parametrize("control,prec,lengths", [
    (False, PRECISION_F16X2, LENGTHS), (True, PRECISION_F16X2, LENGTHS),
    (True, PRECISION_TF32X3, [144, 400, 2000]), (False, PRECISION_TF32, [16, 1536, 2000])])
def test_forward_same_bits_in_every_engine(nets, cuda_device, control, prec, lengths):
    m, sd = nets[control]
    recs = _recordings(lengths, control, 11)
    m.precision = prec
    try:
        m.batch_invariant = True
        inv = _runs(m, recs, cuda_device)
        m.batch_invariant = False
        default = _runs(m, recs, cuda_device)
    finally:
        m.precision, m.batch_invariant = None, False
        m.invalidate_engine()
    for i, runs in enumerate(inv):
        for k, r in enumerate(runs[1:]):
            assert torch.equal(_bits(r), _bits(runs[0])), f"recording {i} ({lengths[i]} frames), run {k + 1}"
    # the control: the default engines choose other plans for the same recordings
    assert any(not torch.equal(_bits(r), _bits(runs[0])) for runs in default for r in runs[1:])
    tol = TOL if prec != PRECISION_TF32 else 3e-3
    for i, runs in enumerate(inv):  # the same recordings in the default mode, up to summation order
        assert float((runs[0] - default[i][0]).abs().max()) < tol, i


@pytest.mark.parametrize("control", [False, True])
def test_benchmark_shape_keeps_the_default_bits(nets, cuda_device, control):
    """64 clips x 144 frames: the canonical plan is the default engine's plan there, so the two modes agree bit for bit."""
    m, _ = nets[control]
    B, T = 64, 144
    b = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, 5, control=control).items()
         if k != 'motion_repr_clean'}
    b['x_t'] = torch.randn(B, T, 13, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    ts = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(6)).to(cuda_device)
    try:
        ref = m(b, ts).clone()
        m.batch_invariant = True
        got = m(b, ts)
        assert m._engine.batch_invariant
    finally:
        m.batch_invariant = False
        m.invalidate_engine()
    assert torch.equal(_bits(got), _bits(ref))


def test_clip_slices_reproduce_the_default_kernel_on_uniform_clips(nets, cuda_device):
    """3 x 1536 frames (2-CTA GroupNorm clusters at levels 0-3): lengths = T for every clip runs the clip-slice instance
    with v = n, and gives the bits of the uniform layout's default cluster kernel in the same engine."""
    m, _ = nets[True]
    B, T = 3, 1536
    b = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, 7, control=True).items()
         if k != 'motion_repr_clean'}
    b['x_t'] = torch.randn(B, T, 13, generator=torch.Generator().manual_seed(7)).to(cuda_device)
    ts = torch.tensor([3, 400, 999], device=cuda_device)
    m.batch_invariant = True
    try:
        ref = m(b, ts).clone()
        e = m._engine
        got = m(dict(b, lengths=torch.full((B,), T, device=cuda_device)), ts)
        assert m._engine is e
    finally:
        m.batch_invariant = False
        m.invalidate_engine()
    assert torch.equal(_bits(got), _bits(ref))


def test_parity_with_the_oracle_and_the_golden_file(nets, cuda_device):
    g = golden("trajnet_forward.npz")
    try:
        for c in range(int(g["n_cases"])):
            B, T, s, control = [int(v) for v in g[f"c{c}_meta"]]
            m, _ = nets[bool(control)]
            m.batch_invariant = True
            x = torch.randn(B, T, 13, generator=torch.Generator().manual_seed(s))
            batch = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(B, T, s + 100, control=bool(control)).items()}
            batch['x_t'] = x.to(cuda_device)
            y = m(batch, torch.from_numpy(g[f"c{c}_timesteps"]).to(cuda_device)).cpu()
            assert float((y - torch.from_numpy(g[f"c{c}_out"])).abs().max()) < TOL, c
        m, sd = nets[True]
        m.batch_invariant = True
        recs = _recordings([400, 144, 16], True, 23)
        b, ts = _batch(recs, [0, 1, 2], 400, cuda_device)
        out = m(b, ts).cpu()
        for i, (r, t) in enumerate(recs):
            n = r['x_t'].shape[1]
            with torch.no_grad():
                ref = trajnet_oracle.trajnet_forward(sd, r['x_t'], r['cond'], torch.tensor([t]), r['control_cond'])
            assert float((out[i, :n] - ref[0]).abs().max()) < TOL, i
    finally:
        for m, _ in nets.values():
            m.batch_invariant = False
            m.invalidate_engine()


def _diff(dev, steps='10'):
    a = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionTrajNet, 1000, steps, dev)


def test_sampling_recording_alone_and_in_shards(nets, cuda_device):
    """A respaced p_sample_loop over a ragged TrajControl batch with one generator per recording: each recording equals
    its loop alone in a fresh engine at its own length; two shards run one after another, each in an engine made for its
    size, give the same bits."""
    m, _ = nets[True]
    dev = cuda_device
    lengths, T, seeds = [2000, 400, 144, 16], 2000, [91, 92, 93, 94]
    recs = _recordings(lengths, True, 31)
    m.batch_invariant = True
    try:
        m.invalidate_engine()
        b, _ = _batch(recs, range(4), T, dev)
        del b['x_t']
        b['generators'] = _gens(dev, seeds)
        full = _diff(dev).p_sample_loop(m, b, [4, T, 13], clip_denoised=False).clone()
        for i, n in enumerate(lengths):
            m.invalidate_engine()
            r = {k: v.to(dev) for k, v in recs[i][0].items() if k != 'x_t'}
            r['generators'] = _gens(dev, [seeds[i]])
            one = _diff(dev).p_sample_loop(m, r, [1, n, 13], clip_denoised=False)
            assert torch.equal(_bits(one[0]), _bits(full[i, :n])), f"recording {i} ({n} frames)"
            assert bool((full[i, n:] == 0).all())
        for shard in ([0, 1, 2], [3]):
            m.invalidate_engine()
            sb, _ = _batch(recs, shard, max(lengths[i] for i in shard), dev)
            del sb['x_t']
            sb['generators'] = _gens(dev, [seeds[i] for i in shard])
            part = _diff(dev).p_sample_loop(m, sb, [len(shard), sb['cond'].shape[1], 13], clip_denoised=False)
            assert m._engine.max_batch == len(shard)
            for j, i in enumerate(shard):
                assert torch.equal(_bits(part[j, :lengths[i]]), _bits(full[i, :lengths[i]])), f"shard recording {i}"
    finally:
        m.batch_invariant = False
        m.invalidate_engine()


# ---------------------------------------------------------------------------------------------------------- rounds
@pytest.fixture(scope="module")
def rounds_nets(cuda_device):
    import test_gpu_pipeline as tp
    from rohm_b200.body_model import BodyModel
    from test_gpu_pipeline_lengths import _datasets
    ds_p, ds_t = _datasets()
    mp, mt, mc, *_ = tp._models(cuda_device, ds_p, ds_t)
    return ds_p, ds_t, mp, mt, mc, BodyModel.create('', device=cuda_device, seed=0)


REC_KEYS = ('smpl_verts_rec', 'smpl_verts_clean', 'rec_ric_data_rec_from_smpl', 'rec_ric_data_rec_from_abs_traj',
            'rec_ric_data_clean', 'motion_repr_rec', 'smpl_verts_noisy', 'motion_repr_noisy')


def _rounds(nets, dev, lengths, T, gens, clip=None):
    """Two guided rounds; clip=b: recording b alone at its own length, without lengths, in fresh engines."""
    import test_gpu_pipeline as tp
    ds_p, ds_t, mp, mt, mc, bm = nets
    dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing="3" + ",0" * 19)
    pose, traj = synthetic.pipeline_batches(len(lengths), 5, ds_p, frames=T, device=dev)
    if clip is None:
        traj['lengths'] = torch.tensor(lengths, device=dev)
    else:
        n = lengths[clip]
        pose = {k: v[clip:clip + 1, :n].contiguous() for k, v in pose.items()}
        traj = {k: v[clip:clip + 1, :n].contiguous() for k, v in traj.items()}
        for net in (mt, mc):
            net.invalidate_engine()
    traj['generators'] = gens
    args = pipeline.make_args(sample_iter=2, mask_scheme='lower', cond_fn_with_grad=True)
    outs = pipeline.run_rounds(args, mp, mt, mc, dp, dt, dc, ds_p, ds_t, bm, pose, traj)
    rec = pipeline.reconstruct_outputs(args, ds_p, bm, pose, outs[0], outs[2], return_verts=True)
    return outs, rec


def test_guided_rounds_recording_alone_in_fresh_engines(rounds_nets, cuda_device):
    dev, lengths, T = cuda_device, [400, 144, 64, 16], 400
    mp, mt, mc = rounds_nets[2:5]
    gens = _gens(dev, [61, 62, 63, 64])
    clones = [_clone(g) for g in gens]
    mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'clip', True, True
    try:
        (vp, vt, tn), rec = _rounds(rounds_nets, dev, lengths, T, gens)
        for b, n in enumerate(lengths):
            (op, ot, on), r1 = _rounds(rounds_nets, dev, lengths, T, [clones[b]], clip=b)
            assert torch.equal(_bits(vp[b:b + 1, ..., :n - 1]), _bits(op)), f"recording {b}: val_output_pose"
            assert torch.equal(_bits(vt[b:b + 1, :n]), _bits(ot)), f"recording {b}: val_output_traj"
            assert torch.equal(_bits(tn[b:b + 1, :n]), _bits(on)), f"recording {b}: traj_noisy_full"
            for key in REC_KEYS:
                assert torch.equal(_bits(rec[key][b]), _bits(r1[key][0])), (b, key)
    finally:
        mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'batch', False, False
        mt.invalidate_engine()
        mc.invalidate_engine()
    assert all(bool(torch.isfinite(t).all()) for t in (vp, vt, tn))


# ---------------------------------------------------------------------------------------------------------- refusals
def test_attribute_and_refusals(nets, cuda_device):
    """A plain attribute (not in the state dict, kept by .to() and load_state_dict); a non-bool refused before any
    engine exists or any noise is drawn."""
    m, sd = nets[False]
    m.batch_invariant = True
    try:
        assert not any('batch_invariant' in k for k in m.state_dict())
        m.to(cuda_device)
        m.load_state_dict(sd)
        assert m.batch_invariant is True
    finally:
        m.batch_invariant = False
    b = {k: v.to(cuda_device) for k, v in synthetic.trajnet_batch(2, 32, 3, control=False).items()
         if k != 'motion_repr_clean'}
    b['x_t'] = torch.zeros(2, 32, 13, device=cuda_device)
    for bad in (1, 'yes', None, torch.tensor(True)):
        m.invalidate_engine()
        m.batch_invariant = bad
        try:
            with pytest.raises(RohmB200Error, match="batch_invariant"):
                m(b, torch.zeros(2, dtype=torch.long, device=cuda_device))
            d = _diff(cuda_device, '4')
            calls = []
            d._randn = lambda *s, **k: calls.append(s) or torch.randn(*s).to(cuda_device)
            d._randn_like = lambda x: calls.append(x.shape) or torch.randn(x.shape).to(cuda_device)
            with pytest.raises(RohmB200Error, match="batch_invariant"):
                d.p_sample_loop(m, {k: v for k, v in b.items() if k != 'x_t'}, [2, 32, 13], clip_denoised=False)
            assert not calls and m._engine is None
        finally:
            m.batch_invariant = False
