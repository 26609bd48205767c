"""Input noise on whole recordings' windows on the device (rohm_b200.windows.InputNoise, rohm_window_param_noise and
rohm_window_encode_canonical): the noisy windows against the reference's AMASS loader with preset noise
(tests/golden/windows_noise.npz, 24-frame windows) and the float64 oracle (also on a 145-frame window), zero noise against
the clean rows, device draws against torch's own draws bit for bit, the drawn noise's standard deviations, each window the
same bits in any batch or order and with poison outside the windows, and two guided rounds with input_noise on the noisy
windows of three recordings against each recording run alone.

Bounds.  The rotations' Euler round trip runs in float64, so a noisy parameter carries the float32 rounding of its
inputs and of its output: the canonical global orientation is a float32 rotvec -> matrix -> canonical rotation (a few
roundings of size <= 1 each), the body pose a float32 rotvec, and the output one more rounding; at most 64 roundings of a
value of size <= 1 + |v| give e_p = 64 eps (1 + max |v|).  The noisy joints are float32 FK of those parameters: each
joint is a chain of at most 8 rigid transforms of the window's coordinates (size <= S), 64 eps (1 + S), plus each of the
8 rotations' parameter error e_p times a lever arm below 1 m: e_j = 64 eps (1 + S) + 8 e_p.  A channel of the
representation is a difference of two joints or a parameter, computed as the encoder's module bound (test_gpu_windows)
says, so its error is that bound on the window plus 4 e_j + 2 e_p, and the channels that use the heading turn by
2 (4 e_j) / a_min more.  A contact label is exact where the oracle's foot height is more than e_j from its threshold and
its squared speed v2 more than 4 sqrt(v2) e_j + 4 e_j^2 from 5e-5.
"""
import numpy as np
import pytest
import torch

import test_gpu_pipeline as tp
from helpers import golden
from oracle import windows_noise_oracle as wno
from oracle import windows_oracle as wo
from rohm_b200 import pipeline, synthetic, windows
from rohm_b200.body_model import BodyModel
from test_gpu_noise_streams import _clone, _gens
from test_gpu_pipeline_lengths import _datasets
from test_gpu_windows import EPS, HEADING, USES_HEADING, _bits, _recording_params
from test_gpu_windows import _bound as _clean_bound
from test_windows_noise_host import PARAM_NAMES, noise_case

pytestmark = pytest.mark.gpu

LEVEL3 = {'transl': 0.03, 'betas': 0.1, 'global_orient': 3.0, 'body_pose': 3.0}
SHAPES = {'transl': (3,), 'betas': (10,), 'global_orient': (3,), 'body_pose': (21, 3)}
FEET, FOOT_THR = [7, 10, 8, 11], np.array([0.18, 0.15, 0.18, 0.15])


@pytest.fixture(scope="module")
def bm(cuda_device):
    return BodyModel.create('', device=cuda_device, seed=0)


def _to(d, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in d.items()}


def _given(noise, dev):
    t = _to({k: np.asarray(v, np.float32) for k, v in noise.items()}, dev)
    return windows.InputNoise.given(t['transl'], t['betas'], t['global_orient'], t['body_pose'])


def _cpu_noise(W, L, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return {k: (scale * LEVEL3[k] * torch.randn((W, L) + SHAPES[k], generator=g)).numpy() for k in PARAM_NAMES}


def _bounds(jw, ref, params):
    """(e_p, e_j, per-channel bound of the noisy rows) for one window: module docstring."""
    S = float(np.abs(jw).max())
    e_p = 64 * EPS * (1 + max(float(np.abs(v).max()) for v in params.values()))
    e_j = 64 * EPS * (1 + S) + 8 * e_p
    across = (jw[:, 1] - jw[:, 2]) + (jw[:, 17] - jw[:, 16])
    a = np.linalg.norm(across[:, 0:2], axis=-1)
    a_min = float(a[a > 0].min())
    e = 32 * EPS * (1 + S) + 4 * e_j + 2 * e_p
    turn = 2 * e / a_min
    b = np.full(ref.shape, e)
    b[..., HEADING] += 2 * turn
    b[..., USES_HEADING] += turn * (1 + np.abs(ref[..., USES_HEADING]))
    return e_p, e_j, b


def _sure_contacts(jw, e_j):
    """[T-1, 4] mask of the contact decisions the bound settles (module docstring)."""
    v2 = ((jw[1:, FEET] - jw[:-1, FEET]) ** 2).sum(-1)
    z = jw[:-1, FEET, 2]
    return (np.abs(z - FOOT_THR) > e_j) & (np.abs(v2 - 5e-5) > 4 * np.sqrt(v2) * e_j + 4 * e_j ** 2)


def _check_against(traj, pose, win, want_params, want_joints, want_rep, clean_rep, ds_p, ds_t, extra=None, label=""):
    """The device's noisy windows against float64 (or float32 golden) noisy params, joints and un-normalised rows."""
    W, L = want_joints.shape[0], want_joints.shape[1]
    got_p = win.noisy_params.cpu().numpy().astype(np.float64)
    got_j = traj['noisy_joints'].cpu().numpy().astype(np.float64)
    assert torch.equal(traj['noisy_joints'], pose['noisy_joints'])
    inside = 0
    for w in range(W):
        pw = {k: want_params[k][w] for k in PARAM_NAMES}
        e_p, e_j, b = _bounds(want_joints[w], want_rep[w], pw)
        for k in PARAM_NAMES:
            err = np.abs(got_p[w][:, windows.NOISY_ROW[k]] - pw[k].reshape(L, -1)).max()
            tol = e_p if k != 'transl' else 64 * EPS * (1 + float(np.abs(want_joints[w]).max())) + e_p
            assert err <= tol + (extra or 0) * (1 + np.abs(pw[k]).max()), (label, w, k, err, tol)
        err = np.abs(got_j[w] - want_joints[w]).max()
        assert err <= e_j + (extra or 0) * (1 + np.abs(want_joints[w]).max()), (label, w, err, e_j)
        if extra:
            b = b + extra * (1 + np.abs(want_rep[w]))
        for name, z, ds in (("traj", traj['motion_repr_noisy'][w], ds_t), ("pose", pose['motion_repr_noisy'][w], ds_p)):
            got = z.cpu().numpy().astype(np.float64) * ds.Std + ds.Mean
            want = want_rep[w].copy()
            if name == "pose":
                want[:, 0:ds_p.traj_feat_dim] = clean_rep[w][:, 0:ds_p.traj_feat_dim]
            ratio = np.abs(got - want)[:, :290] / b[:, :290]
            assert ratio.max() <= 1.0, (label, name, w, np.unravel_index(ratio.argmax(), ratio.shape))
            sure = _sure_contacts(want_joints[w], e_j)
            assert np.array_equal((got[:, 290:] > 0.5)[sure], (want[:, 290:] > 0.5)[sure]), (label, name, w)
            inside += int((~sure).sum())
    print(f"{label}: {inside} foot decisions inside the margin (of {2 * W * (L - 1) * 4})")
    sel = list(windows.ABS_TRAJ_CHANNELS)
    assert torch.equal(traj['cond'], traj['motion_repr_noisy'][..., sel])
    assert torch.equal(traj['control_cond'], traj['motion_repr_clean'][..., 22:])
    assert torch.equal(_bits(pose['motion_repr_noisy'][..., 0:22]), _bits(pose['motion_repr_clean'][..., 0:22]))


def test_given_noise_matches_golden_and_oracle(cuda_device, bm):
    dev = cuda_device
    g = golden("windows_noise.npz")
    ds_p, ds_t = _datasets()
    L, overlap, lengths, params, joints, noise = noise_case(g)
    model = synthetic.smplx_like_model(0)
    traj, pose, win = windows.encode_joints(_to(params, dev), _to({'j': joints}, dev)['j'], lengths, ds_p, ds_t, L,
                                            overlap, noise=_given(noise, dev), body_model=bm)
    o_params, o_joints, o_rep = wno.encode_noisy(params, joints, lengths, noise, model, L, overlap)
    _, _, clean = wo.encode(params, joints, lengths, L, overlap)
    _check_against(traj, pose, win, o_params, o_joints, o_rep, clean, ds_p, ds_t, label="oracle")
    # the reference's float32 pipeline, as stored
    gp = {k: g[f"noisy_param_{k}"].astype(np.float64) for k in PARAM_NAMES}
    gj = g["noisy_joints"].astype(np.float64)
    grep = np.asarray(g["traj_motion_repr_noisy"], np.float64) * ds_t.Std + ds_t.Mean
    gclean = clean.copy()
    _check_against(traj, pose, win, gp, gj, grep, gclean, ds_p, ds_t, extra=2e-5, label="golden")
    # the other entries of the reference's dicts, de-normalised: the pose rows (noisy local channels, clean trajectory
    # channels), the TrajNet condition (noisy) and control signal (clean).  Noisy channels: this module's bound; clean
    # channels: the encoder's (test_gpu_windows._bound, on the window's world joints); both plus the float32 rounding of
    # the stored reference, 2e-5 (1 + |v|) as in test_gpu_windows.
    sel = list(windows.ABS_TRAJ_CHANNELS)
    off = np.cumsum([0] + lengths)
    for w, (r, s) in enumerate(g["table"]):
        gpw = {k: gp[k][w] for k in PARAM_NAMES}
        b_noisy = _bounds(gj[w], grep[w], gpw)[2] + 2e-5 * (1 + np.abs(grep[w]))
        b_clean = _clean_bound(joints[off[r] + s:off[r] + s + L], clean[w]) + 2e-5 * (1 + np.abs(clean[w]))
        b_pose = np.concatenate([b_clean[:, :ds_p.traj_feat_dim], b_noisy[:, ds_p.traj_feat_dim:]], axis=-1)
        for name, got, mean, std, bound in (
                ("pose_motion_repr_noisy", pose['motion_repr_noisy'], ds_p.Mean, ds_p.Std, b_pose),
                ("traj_cond", traj['cond'], ds_t.Mean[sel], ds_t.Std[sel], b_noisy[:, sel]),
                ("traj_control_cond", traj['control_cond'], ds_t.Mean[22:], ds_t.Std[22:], b_clean[:, 22:])):
            want = np.asarray(g[name][w], np.float64) * std + mean
            err = np.abs(got[w].cpu().numpy().astype(np.float64) * std + mean - want)
            n = min(want.shape[-1], bound.shape[-1] - (4 if name != "traj_cond" else 0))  # contacts: checked above
            ratio = err[:, :n] / bound[:, :n]
            assert ratio.max() <= 1.0, (name, w, np.unravel_index(ratio.argmax(), ratio.shape))


def test_given_noise_on_a_145_frame_window(cuda_device, bm):
    dev = cuda_device
    ds_p, ds_t = _datasets()
    params = _recording_params(145, 5)
    noise = _cpu_noise(1, 145, 17)
    traj, pose, win = windows.encode(bm, _to(params, dev), [145], ds_p, ds_t, noise=_given(noise, dev))
    fk = bm(**_to(params, dev), return_verts=False).joints[:, 0:22].cpu().numpy()
    model = synthetic.smplx_like_model(0)
    o_params, o_joints, o_rep = wno.encode_noisy(params, fk, [145], noise, model)
    _, _, clean = wo.encode(params, fk, [145])
    _check_against(traj, pose, win, o_params, o_joints, o_rep, clean, ds_p, ds_t, label="145 frames")


def test_zero_noise_gives_the_clean_rows(cuda_device, bm):
    """Zero noise: the noisy windows are the clean ones through a different route (fp64 Euler round trip, FK of the
    canonical parameters instead of canonicalised FK joints): within the module's bounds, not bit-identical -- except
    the channels of the translation and the betas, which the noise kernel takes from the encoder's own functions."""
    dev = cuda_device
    ds_p, ds_t = _datasets()
    lengths = [300, 145]
    recs = [_recording_params(n, 31 + i) for i, n in enumerate(lengths)]
    params = {k: np.concatenate([r[k] for r in recs]) for k in PARAM_NAMES}
    W = len(windows.window_table(lengths))
    zero = {k: np.zeros((W, 145) + SHAPES[k], np.float32) for k in PARAM_NAMES}
    traj, pose, win = windows.encode(bm, _to(params, dev), lengths, ds_p, ds_t, noise=_given(zero, dev))
    fk = bm(**_to(params, dev), return_verts=False).joints[:, 0:22].cpu().numpy()
    table, transf, clean = wo.encode(params, fk, lengths)
    off = np.cumsum([0] + lengths)
    for w, (r, s) in enumerate(table):
        rows = slice(off[r] + s, off[r] + s + 145)
        cano = wno.canonical_params({k: v[rows] for k, v in params.items()}, fk[rows], transf[w])
        cj = fk[rows].astype(np.float64) @ transf[w][:3, :3].T + transf[w][:3, 3]
        e_p, e_j, b = _bounds(cj, clean[w], cano)
        got_j = traj['noisy_joints'][w].cpu().numpy()
        assert np.abs(got_j - cj).max() <= 2 * e_j, w  # FK of the canonical parameters vs the canonicalised FK joints
        got_go = win.noisy_params[w, :, 0:3].cpu().numpy()
        assert np.abs(wo.rotvec_to_matrix(got_go) - wo.rotvec_to_matrix(cano['global_orient'])).max() <= e_p, w
        got = traj['motion_repr_noisy'][w].cpu().numpy().astype(np.float64) * ds_t.Std + ds_t.Mean
        ref = traj['motion_repr_clean'][w].cpu().numpy().astype(np.float64) * ds_t.Std + ds_t.Mean
        assert (np.abs(got - ref)[:, :290] / (2 * b[:, :290])).max() <= 1.0, w
    # the canonical translation and the betas under the noise are the bits the clean rows were encoded from (the noise
    # kernel rebuilds the encoder's CanoFrame from transf and the frame-0 root, and calls the same cano_transl): with zero
    # noise the channels built from them alone -- translation, its velocity, betas -- are bit-identical
    for ch in (slice(16, 22), slice(280, 290)):
        assert torch.equal(_bits(traj['motion_repr_noisy'][..., ch]), _bits(traj['motion_repr_clean'][..., ch])), ch


def test_drawn_equals_given_bit_for_bit_beyond_256_windows(cuda_device, bm):
    """InputNoise.drawn(gens) equals InputNoise.given fed with std * torch.randn(shape, generator=clone) drawn in the
    reference's order, bit for bit, over 310 windows (two launches of at most 256 per draw); the generators' offsets end
    where torch leaves the clones'."""
    dev = cuda_device
    ds_p, ds_t = _datasets()
    lengths = [143 * 150 + 2, 143 * 160 + 2]
    recs = [_recording_params(n, 41 + i) for i, n in enumerate(lengths)]
    params = _to({k: np.concatenate([r[k] for r in recs]) for k in PARAM_NAMES}, dev)
    W = len(windows.window_table(lengths))
    assert W == 310
    gens = _gens(dev, [900 + w for w in range(W)], offsets=[4 * (w % 3) for w in range(W)])
    clones = [_clone(x) for x in gens]
    draws = {k: [] for k in PARAM_NAMES}
    for c in clones:  # dataloader_amass.py:159: transl, body_pose, betas, global_orient
        draws['transl'].append(0.03 * torch.randn([145, 3], generator=c, device=dev))
        draws['body_pose'].append(3.0 * torch.randn([145 * 21, 3], generator=c, device=dev).reshape(145, 21, 3))
        draws['betas'].append(0.1 * torch.randn([145, 10], generator=c, device=dev))
        draws['global_orient'].append(3.0 * torch.randn([145, 3], generator=c, device=dev))
    given = windows.InputNoise.given(*(torch.stack(draws[k]) for k in ('transl', 'betas', 'global_orient', 'body_pose')))
    a = windows.encode(bm, params, lengths, ds_p, ds_t, noise=windows.InputNoise.drawn(gens))
    b = windows.encode(bm, params, lengths, ds_p, ds_t, noise=given)
    assert torch.equal(_bits(a[2].noisy_params), _bits(b[2].noisy_params))
    for key in ('motion_repr_noisy', 'noisy_joints'):
        for d in (0, 1):
            assert torch.equal(_bits(a[d][key]), _bits(b[d][key])), (d, key)
    assert [g.get_offset() for g in gens] == [c.get_offset() for c in clones]


def test_drawn_noise_has_the_requested_deviations(cuda_device, bm):
    """About 400 windows of drawn noise at non-default deviations: the noisy - clean differences of the translation, the
    betas and (away from the lock, where the Euler decomposition is unique) the 'zxy' angles have the requested standard
    deviations.  Sampling bound: the sample deviation of n normal draws has relative standard error 1/sqrt(2n); the test
    allows 6 of them."""
    dev = cuda_device
    ds_p, ds_t = _datasets()
    lengths = [143 * 200 + 2, 143 * 200 + 2]
    recs = [_recording_params(n, 51 + i) for i, n in enumerate(lengths)]
    params = _to({k: np.concatenate([r[k] for r in recs]) for k in PARAM_NAMES}, dev)
    W = len(windows.window_table(lengths))
    std = {'global_orient': 2.0, 'body_pose': 4.0, 'transl': 0.05, 'betas': 0.2}
    noise = windows.InputNoise.drawn(_gens(dev, [3000 + w for w in range(W)]), std_global_rot=2.0, std_body_rot=4.0,
                                     std_transl=0.05, std_betas=0.2)
    zero = {k: torch.zeros((W, 145) + SHAPES[k], device=dev) for k in PARAM_NAMES}
    zero = windows.InputNoise.given(zero['transl'], zero['betas'], zero['global_orient'], zero['body_pose'])
    noisy = windows.encode(bm, params, lengths, ds_p, ds_t, noise=noise)[2].noisy_params.cpu().numpy().astype(np.float64)
    clean = windows.encode(bm, params, lengths, ds_p, ds_t, noise=zero)[2].noisy_params.cpu().numpy().astype(np.float64)
    for k in ('transl', 'betas'):
        d = (noisy[..., windows.NOISY_ROW[k]] - clean[..., windows.NOISY_ROW[k]]).ravel()
        r = d.std() / std[k]
        assert abs(r - 1) < 6 / np.sqrt(2 * d.size), (k, r, d.size)
    for k in ('global_orient', 'body_pose'):
        qn = wno.quat_from_rotvec(noisy[..., windows.NOISY_ROW[k]].reshape(-1, 3))
        qc = wno.quat_from_rotvec(clean[..., windows.NOISY_ROW[k]].reshape(-1, 3))
        far = (wno.lock_distance(qc) > 0.2) & (wno.lock_distance(qn) > 0.2)
        d = np.degrees(wno.euler_zxy(qn[far]) - wno.euler_zxy(qc[far]))
        d = (d + 180.0) % 360.0 - 180.0
        r = d.std() / std[k]
        assert abs(r - 1) < 6 / np.sqrt(2 * d.size), (k, r, d.size)
        assert abs(d.mean()) < 6 * std[k] / np.sqrt(d.size), k


def _window_noise(lengths, idx, dev, drawn):
    """Per-window noise keyed by (recording id, start): the same noise for a window in any batch."""
    table = windows.window_table([lengths[i] for i in idx])
    if drawn:
        return windows.InputNoise.drawn(_gens(dev, [7000 + 1000 * idx[r] + s for r, s in table]))
    per = [_cpu_noise(1, 145, 10_000 * idx[r] + s) for r, s in table]
    return _given({k: np.concatenate([p[k] for p in per]) for k in PARAM_NAMES}, dev)


@pytest.mark.parametrize("drawn", [False, True])
def test_each_noisy_window_is_the_same_alone_among_others_and_in_any_order(cuda_device, bm, drawn):
    dev = cuda_device
    ds_p, ds_t = _datasets()
    lengths = [300, 145, 433]
    recs = [_recording_params(n, 61 + i) for i, n in enumerate(lengths)]

    def run(idx, poison=False):
        p = {k: np.concatenate([recs[i][k] for i in idx]) for k in PARAM_NAMES}
        if poison:  # every frame no window reads holds NaN or +-Inf
            off = np.cumsum([0] + [lengths[i] for i in idx])
            read = np.zeros(off[-1], dtype=bool)
            for r, s in windows.window_table([lengths[i] for i in idx]):
                read[off[r] + s:off[r] + s + 145] = True
            assert (~read).sum() > 10
            for n_, f in enumerate(np.where(~read)[0]):
                for k in PARAM_NAMES:
                    p[k][f] = (np.nan, np.inf, -np.inf)[n_ % 3]
        traj, pose, win = windows.encode(bm, _to(p, dev), [lengths[i] for i in idx], ds_p, ds_t,
                                         noise=_window_noise(lengths, idx, dev, drawn))
        out = {}
        k = 0
        for r, s in zip(win.recording.tolist(), win.start.tolist()):
            out[(idx[r], s)] = (win.noisy_params[k], traj['noisy_joints'][k], traj['motion_repr_noisy'][k],
                                pose['motion_repr_noisy'][k])
            k += 1
        return out

    every = run([0, 1, 2])
    assert len(every) == 2 + 1 + 3
    for idx, poison in (([2, 0, 1], False), ([1], False), ([0], False), ([2], False), ([0, 1, 2], True)):
        res = run(idx, poison)
        for key, vals in res.items():
            for a, b in zip(vals, every[key]):
                assert torch.equal(_bits(a), _bits(b)), (idx, poison, key)


def test_two_guided_noisy_rounds_per_recording_equal_the_recording_alone(cuda_device, bm):
    """Three recordings' noisy windows in one batch through two respaced, guided rounds with input_noise (one sampling
    generator and one noise generator per window, per-clip guidance normalisers, batch-invariant TrajNets): each
    recording's world-frame joints and its rec_ric_data_noisy are bit-identical to the same recording encoded with the
    same noise and run alone, and the noisy reconstruction differs from the clean one by the noise."""
    dev = cuda_device
    ds_p, ds_t = _datasets()
    mp, mt, mc, *_ = tp._models(dev, ds_p, ds_t)
    lengths = [300, 145, 433]
    recs = [_recording_params(n, 21 + i) for i, n in enumerate(lengths)]

    def run(idx):
        params = _to({k: np.concatenate([recs[i][k] for i in idx]) for k in PARAM_NAMES}, dev)
        traj, pose, win = windows.encode(bm, params, [lengths[i] for i in idx], ds_p, ds_t,
                                         noise=_window_noise(lengths, idx, dev, True))
        seeds = [1000 * idx[r] + s for r, s in zip(win.recording.tolist(), win.start.tolist())]
        traj['generators'] = _gens(dev, seeds)
        dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing="3" + ",0" * 19)
        args = pipeline.make_args(sample_iter=2, mask_scheme='lower', cond_fn_with_grad=True, input_noise=True)
        outs = pipeline.run_rounds(args, mp, mt, mc, dp, dt, dc, ds_p, ds_t, bm, pose, traj)
        rec = pipeline.reconstruct_outputs(args, ds_p, bm, pose, outs[0], outs[2], return_verts=False)
        world, covered = windows.to_recordings(win, rec['rec_ric_data_rec_from_smpl'])
        noisy = rec['rec_ric_data_noisy'].reshape(len(win), -1, 22, 3)
        clean = rec['rec_ric_data_clean'].reshape(len(win), -1, 22, 3)
        return world, covered, win.recording, noisy, clean

    mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'clip', True, True
    try:
        world, covered, recording, noisy, clean = run([0, 1, 2])
        assert float((noisy - clean).norm(dim=-1).mean()) > 1e-3  # the rounds saw noisy inputs
        for i in range(3):
            mt.invalidate_engine()
            mc.invalidate_engine()
            w1, c1, _, n1, _ = run([i])
            assert torch.equal(covered[i], c1[0]), i
            assert torch.equal(_bits(world[i]), _bits(w1[0])), i
            assert torch.equal(_bits(noisy[recording == i]), _bits(n1)), i
            assert bool(torch.isfinite(world[i]).all()) and bool(torch.isfinite(n1).all())
    finally:
        mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'batch', False, False
        mt.invalidate_engine()
        mc.invalidate_engine()


def test_noise_refusals(cuda_device, bm):
    dev = cuda_device
    ds_p, ds_t = _datasets()
    p = {k: torch.zeros(300, w, device=dev) for k, w in windows.PARAMS}
    j = torch.zeros(300, 22, 3, device=dev)
    ok = {k: torch.zeros((2, 145) + SHAPES[k], device=dev) for k in PARAM_NAMES}
    mk = lambda d: windows.InputNoise.given(d['transl'], d['betas'], d['global_orient'], d['body_pose'])
    with pytest.raises(windows.RohmB200Error, match="float32"):
        mk(dict(ok, betas=ok['betas'].double()))
    with pytest.raises(windows.RohmB200Error, match="body_pose must be"):
        mk(dict(ok, body_pose=torch.zeros(2, 145, 63, device=dev)))
    with pytest.raises(windows.RohmB200Error, match="covers"):
        mk(dict(ok, global_orient=torch.zeros(3, 145, 3, device=dev)))
    with pytest.raises(windows.RohmB200Error, match="cut 2 windows"):  # 3 windows' noise for 2
        windows.encode_joints(p, j, [300], ds_p, ds_t, noise=mk({k: torch.zeros((3, 145) + SHAPES[k], device=dev)
                                                                 for k in PARAM_NAMES}), body_model=bm)
    with pytest.raises(windows.RohmB200Error, match="cut 2 windows of 145"):  # clip_len 24 noise
        windows.encode_joints(p, j, [300], ds_p, ds_t, noise=mk({k: torch.zeros((2, 24) + SHAPES[k], device=dev)
                                                                 for k in PARAM_NAMES}), body_model=bm)
    with pytest.raises(windows.RohmB200Error, match="no window"):
        windows.encode_joints(p, j, [100, 100, 100], ds_p, ds_t, noise=windows.InputNoise.drawn([]), body_model=bm)
    with pytest.raises(windows.RohmB200Error, match="generators"):
        windows.encode(bm, p, [300], ds_p, ds_t, noise=windows.InputNoise.drawn(_gens(dev, [1])))
    g = _gens(dev, [1])[0]
    with pytest.raises(windows.RohmB200Error, match="twice"):
        windows.encode(bm, p, [300], ds_p, ds_t, noise=windows.InputNoise.drawn([g, g]))
    with pytest.raises(windows.RohmB200Error, match="cpu generator"):
        windows.encode(bm, p, [300], ds_p, ds_t, noise=windows.InputNoise.drawn([g, torch.Generator()]))
    # a refused call leaves the generators where they were
    assert g.get_offset() == 0
    # without noise: no new keys
    traj, pose, win = windows.encode(bm, p, [300], ds_p, ds_t)
    assert set(traj) == {'motion_repr_clean', 'motion_repr_noisy', 'cond', 'control_cond'}
    assert set(pose) == {'motion_repr_clean', 'motion_repr_noisy'} and win.noisy_params is None
