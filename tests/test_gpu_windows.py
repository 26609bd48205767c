"""Whole recordings through 145-frame windows on the device (rohm_b200.windows, rohm_window_encode / rohm_window_to_world):
the encoder against the reference's loaders (tests/golden/windows.npz, 24-frame windows to keep the fixture small) and
the float64 oracle (also on a 145-frame window in the round-trip test), each window the same bits in
any batch or order of recordings, nothing past a window read, the round trip back to the world frame, and two guided rounds
on the windows of three recordings against each recording run alone.

Bounds.  The encoder subtracts the window origin from world coordinates of magnitude up to S (the largest |coordinate| of
the window) and rotates the differences: each canonical coordinate carries at most a few ulps of S, and every channel is a
short chain of fp32 operations on those coordinates (at most ~32 roundings, each of relative size eps = 2^-24 on a value
of size <= 1 + S), so a de-normalised channel is within 32 eps (1 + S) of the float64 value, except where the heading
quaternion divides by |across| (hips + shoulders, at least a_min in these recordings): an error d of the joints turns the
heading by up to 2 d / a_min, which moves the channels that use the heading by that angle times their size.  The
z-scored channel (v - mean) / std then carries the de-normalised bound divided by std plus one rounding of its own size.
"""
import numpy as np
import pytest
import torch

import test_gpu_pipeline as tp
from helpers import golden
from oracle import windows_oracle as wo
from rohm_b200 import pipeline, windows
from rohm_b200.body_model import BodyModel
from test_gpu_noise_streams import _gens
from test_gpu_pipeline_lengths import _datasets
from test_windows_host import PARAM_NAMES, golden_case

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
HEADING = slice(0, 2)          # root angle and its velocity
USES_HEADING = np.r_[4:6, 22:154]  # root velocity, local positions, local velocities


def _bits(t):
    return t.contiguous().view(torch.int32)


def _dev(params, joints, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in params.items()}, \
        torch.from_numpy(np.ascontiguousarray(joints)).to(dev)


def _bound(joints_w, ref):
    """Per-channel bound of a window's de-normalised channels (module docstring)."""
    S = float(np.abs(joints_w).max())
    across = (joints_w[:, 1] - joints_w[:, 2]) + (joints_w[:, 17] - joints_w[:, 16])
    a = np.linalg.norm(across[:, 0:2], axis=-1)
    a_min = float(a[a > 0].min())
    e = 32 * EPS * (1 + S)
    turn = 2 * e / a_min
    b = np.full(ref.shape, e)
    b[..., HEADING] += 2 * turn
    b[..., USES_HEADING] += turn * (1 + np.abs(ref[..., USES_HEADING]))
    return b


def test_encoder_matches_golden_and_oracle(cuda_device):
    dev = cuda_device
    g = golden("windows.npz")
    ds_p, ds_t = _datasets()
    for c in range(int(g["n_cases"])):
        L, overlap, lengths, params, joints = golden_case(g, c)
        p, j = _dev(params, joints, dev)
        traj, pose, win = windows.encode_joints(p, j, lengths, ds_p, ds_t, L, overlap)
        table, transf, rep = wo.encode(params, joints, lengths, L, overlap)
        assert list(zip(win.recording.tolist(), win.start.tolist())) == [tuple(t) for t in table]
        assert np.abs(win.transf.cpu().numpy() - g[f"c{c}_transf"]).max() < 1e-5
        off = np.cumsum([0] + lengths)
        for name, out, ds in (("traj", traj['motion_repr_clean'], ds_t), ("pose", pose['motion_repr_clean'], ds_p)):
            z = out.cpu().numpy().astype(np.float64)
            mean, std = ds.Mean.astype(np.float64), ds.Std.astype(np.float64)
            for w, (r, s) in enumerate(table):
                jw = joints[off[r] + s:off[r] + s + L]
                for want, label in ((rep[w], "oracle"), (g[f"c{c}_repr"][w].astype(np.float64), "golden")):
                    b = _bound(jw, want) + (2e-5 * (1 + np.abs(want)) if label == "golden" else 0)
                    got = z[w] * std + mean
                    ratio = np.abs(got - want)[:, :290] / b[:, :290]
                    assert ratio.max() <= 1.0, (c, name, w, label, np.unravel_index(ratio.argmax(), ratio.shape))
                    zb = b / std + EPS * np.abs(z[w])
                    zr = np.abs(z[w] - (want - mean) / std)[:, :290] / zb[:, :290]
                    assert zr.max() <= 1.0, (c, name, w, label, np.unravel_index(zr.argmax(), zr.shape))
                # contact labels: exactly the reference's, z-scored by the same fp32 arithmetic
                lab = torch.from_numpy(g[f"c{c}_repr"][w][:, 290:].astype(np.float32))
                zc = (lab - torch.from_numpy(ds.Mean[290:])) / torch.from_numpy(ds.Std[290:])
                assert torch.equal(_bits(out[w, :, 290:].cpu()), _bits(zc)), (c, name, w)
        sel = list(windows.ABS_TRAJ_CHANNELS)
        assert torch.equal(traj['cond'], traj['motion_repr_clean'][..., sel])
        assert torch.equal(traj['control_cond'], traj['motion_repr_clean'][..., 22:])
        assert torch.equal(traj['motion_repr_noisy'], traj['motion_repr_clean'])
        assert torch.equal(pose['motion_repr_noisy'], pose['motion_repr_clean'])


def _windows_of(result):
    traj, pose, win = result
    return traj['motion_repr_clean'], pose['motion_repr_clean'], win.transf


def test_each_window_is_the_same_alone_among_others_and_in_any_order(cuda_device):
    dev = cuda_device
    g = golden("windows.npz")
    ds_p, ds_t = _datasets()
    lengths = [int(n) for n in g["lengths"]]
    off = np.cumsum([0] + lengths)
    params = {k: g[f"param_{k}"] for k in PARAM_NAMES}
    joints = g["joints"]
    L = int(g["clip_len"])

    def run(order):
        rows = np.concatenate([np.arange(off[r], off[r + 1]) for r in order])
        p, j = _dev({k: v[rows] for k, v in params.items()}, joints[rows], dev)
        return windows.encode_joints(p, j, [lengths[r] for r in order], ds_p, ds_t, L)

    every = run([0, 1, 2])
    per_rec = {0: [0, 1], 1: [2]}  # windows of each recording in that run
    for order in ([2, 0, 1], [1, 0], [0], [1], [2]):
        res = run(order)
        k = 0
        for r in order:
            for w in per_rec.get(r, []):
                for a, b in zip(_windows_of(res), _windows_of(every)):
                    assert torch.equal(_bits(a[k]), _bits(b[w])), (order, r, w)
                k += 1
        assert len(res[2]) == k


def test_poison_past_the_windows_never_reaches_a_window(cuda_device):
    """Frames no window covers (the tail after a recording's last window, a recording shorter than a window) hold NaN and
    +-Inf in every input: the windows keep their bits."""
    dev = cuda_device
    g = golden("windows.npz")
    ds_p, ds_t = _datasets()
    lengths = [int(n) for n in g["lengths"]]
    params = {k: g[f"param_{k}"].copy() for k in PARAM_NAMES}
    joints = g["joints"].copy()
    L = int(g["clip_len"])
    clean = windows.encode_joints(*_dev(params, joints, dev), lengths, ds_p, ds_t, L)
    off = np.cumsum([0] + lengths)
    read = np.zeros(off[-1], dtype=bool)
    for r, s in windows.window_table(lengths, L):
        read[off[r] + s:off[r] + s + L] = True
    assert (~read).sum() > 10
    bad = np.where(~read)[0]
    for i, f in enumerate(bad):
        v = (np.nan, np.inf, -np.inf)[i % 3]
        joints[f] = v
        for k in PARAM_NAMES:
            params[k][f] = v
    dirty = windows.encode_joints(*_dev(params, joints, dev), lengths, ds_p, ds_t, L)
    for a, b in zip(_windows_of(dirty), _windows_of(clean)):
        assert torch.equal(_bits(a), _bits(b))


def _recording_params(n, seed):
    """A walking-like recording: heading turning through +-180 deg, smooth translation, small body poses."""
    g = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    yaw = np.pi * np.sin(t / 300.0 + seed) + 0.3 * np.sin(t / 23.0)
    go = np.stack([0.05 * np.sin(t / 11.0), 0.04 * np.cos(t / 17.0), yaw], -1)
    transl = np.stack([2.0 * np.sin(t / 250.0), 2.0 * np.cos(t / 310.0) + seed % 3, 0.9 + 0.03 * np.sin(t / 9.0)], -1)
    betas = np.repeat(0.5 * g.standard_normal((1, 10)), n, axis=0)
    body_pose = 0.15 * g.standard_normal((1, 63)) + 0.1 * np.sin(t[:, None] / 15.0 + np.arange(63))
    return {k: v.astype(np.float32) for k, v in (("global_orient", go), ("transl", transl), ("betas", betas),
                                                   ("body_pose", body_pose))}


@pytest.mark.parametrize("overlap", [2, 0])
def test_round_trip_to_world_frame(cuda_device, overlap):
    """Encoded clean windows -> reconstruct_outputs -> to_recordings equals FK of the input parameters in world coordinates
    on covered frames; the other frames are zero and uncovered.  Bound: the reconstruction's rot6d -> axis-angle ->
    Rodrigues route (the reference's, in fp32: ~1e-6 per rotation) along kinematic chains of up to 8 rotations with lever
    arms below 1 m, plus the z-score round trip and the two rigid transforms (a few ulps of S, the largest |world
    coordinate|): 3e-5 (1 + S)."""
    dev = cuda_device
    ds_p, ds_t = _datasets()
    bm = BodyModel.create('', device=dev, seed=0)
    lengths = [145, 1000, 3000, 100]
    recs = [_recording_params(n, 7 + i) for i, n in enumerate(lengths)]
    params = {k: torch.from_numpy(np.concatenate([r[k] for r in recs])).to(dev) for k in PARAM_NAMES}
    traj, pose, win = windows.encode(bm, params, lengths, ds_p, ds_t, overlap=overlap)
    clean = pose['motion_repr_clean'][:, 0:-1].permute(0, 2, 1).unsqueeze(-2).contiguous()
    args = pipeline.make_args(input_noise=False)
    rec = pipeline.reconstruct_outputs(args, ds_p, bm, {'motion_repr_clean': clean}, clean, None, return_verts=False)
    world, covered = windows.to_recordings(win, rec['rec_ric_data_clean'])
    fk = bm(**{k: v for k, v in params.items()}, return_verts=False).joints[:, 0:22]
    fk = torch.split(fk, lengths)
    table = windows.window_table(lengths, 145, overlap)
    # the 145-frame recording's window against the float64 oracle, within the module's bound (the contact labels of these
    # recordings have no margin to their thresholds, so only channels [0, 290))
    jw = fk[0].cpu().numpy()
    host = {k: v[0:145].cpu().numpy() for k, v in params.items()}
    tf0 = wo.canonical_frame(jw)
    rep0 = wo.encode_window(jw, host['global_orient'], host['transl'], host['betas'], host['body_pose'], tf0)
    got = traj['motion_repr_clean'][0].cpu().numpy().astype(np.float64) * ds_t.Std + ds_t.Mean
    assert np.abs(win.transf[0].cpu().numpy() - tf0).max() < 1e-5
    ratio = (np.abs(got - rep0) / _bound(jw, rep0))[:, :290]
    assert ratio.max() <= 1.0, np.unravel_index(ratio.argmax(), ratio.shape)
    for r, n in enumerate(lengths):
        want = torch.zeros(n, dtype=torch.bool)
        for rr, s in table:
            if rr == r:
                want[s:s + 143] = True
        assert torch.equal(covered[r].cpu(), want), r
        assert world[r].shape == (n, 22, 3)
        assert bool((world[r][~want.to(dev)] == 0).all())
        if want.any():
            S = float(fk[r].abs().max())
            err = float((world[r][want.to(dev)] - fk[r][want.to(dev)]).abs().max())
            assert err <= 3e-5 * (1 + S), (r, err, S)
    assert sum(int(c.sum()) for c in covered) == len(table) * 143


def test_two_guided_rounds_per_recording_equal_the_recording_alone(cuda_device):
    """Three recordings' windows in one batch through two respaced, guided rounds (one generator per window, per-clip
    guidance normalisers, batch-invariant TrajNets): each recording's world-frame joints are bit-identical to the same
    recording encoded and run alone."""
    dev = cuda_device
    ds_p, ds_t = _datasets()
    mp, mt, mc, *_ = tp._models(dev, ds_p, ds_t)
    bm = BodyModel.create('', device=dev, seed=0)
    lengths = [300, 145, 433]
    recs = [_recording_params(n, 21 + i) for i, n in enumerate(lengths)]

    def run(idx):
        params = {k: torch.from_numpy(np.concatenate([recs[i][k] for i in idx])).to(dev) for k in PARAM_NAMES}
        traj, pose, win = windows.encode(bm, params, [lengths[i] for i in idx], ds_p, ds_t)
        seeds = [1000 * idx[r] + s for r, s in zip(win.recording.tolist(), win.start.tolist())]
        traj['generators'] = _gens(dev, seeds)
        dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing="3" + ",0" * 19)
        args = pipeline.make_args(sample_iter=2, mask_scheme='lower', cond_fn_with_grad=True)
        outs = pipeline.run_rounds(args, mp, mt, mc, dp, dt, dc, ds_p, ds_t, bm, pose, traj)
        rec = pipeline.reconstruct_outputs(args, ds_p, bm, pose, outs[0], outs[2], return_verts=False)
        return windows.to_recordings(win, rec['rec_ric_data_rec_from_smpl'])

    mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'clip', True, True
    try:
        world, covered = run([0, 1, 2])
        for i in range(3):
            mt.invalidate_engine()
            mc.invalidate_engine()
            w1, c1 = run([i])
            assert torch.equal(covered[i], c1[0]), i
            assert torch.equal(_bits(world[i]), _bits(w1[0])), i
            assert bool(torch.isfinite(world[i]).all())
    finally:
        mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'batch', False, False
        mt.invalidate_engine()
        mc.invalidate_engine()


def test_refusals(cuda_device):
    dev = cuda_device
    ds_p, ds_t = _datasets()
    p = {k: torch.zeros(150, w, device=dev) for k, w in windows.PARAMS}
    with pytest.raises(windows.RohmB200Error, match="params"):
        windows.encode_joints(p, torch.zeros(150, 22, 3, device=dev), [149], ds_p, ds_t)
    with pytest.raises(windows.RohmB200Error, match="joints"):
        windows.encode_joints(p, torch.zeros(149, 22, 3, device=dev), [150], ds_p, ds_t)
    traj, pose, win = windows.encode_joints(p, torch.zeros(150, 22, 3, device=dev), [100, 50], ds_p, ds_t)
    assert len(win) == 0 and traj['motion_repr_clean'].shape == (0, 144, 294)
    world, covered = windows.to_recordings(win, torch.zeros(0, 143, 22, 3, device=dev))
    assert [tuple(w.shape) for w in world] == [(100, 22, 3), (50, 22, 3)] and not any(bool(c.any()) for c in covered)
    with pytest.raises(windows.RohmB200Error, match="joints"):
        windows.to_recordings(win, torch.zeros(1, 143, 22, 3, device=dev))
