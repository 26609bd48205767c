"""The video loader's windows on the device (rohm_b200.windows.encode_video: rohm_window_encode_video,
rohm_window_keypoints, rohm_window_scene_joints) against the reference's DataloaderVideo (tests/golden/windows_video.npz)
and the float64 oracle, and per-window cameras in PoseNet's projection guidance."""
import types

import numpy as np
import pytest
import torch

from helpers import golden
from oracle import windows_video_oracle as wvo
from rohm_b200 import synthetic, windows
from rohm_b200.body_model import BodyModel
from test_gpu_windows import _bound, _recording_params
from test_windows_video_host import PARAMS, fk, oracle_case, video_case

pytestmark = pytest.mark.gpu

# float32 bounds, derived as in test_gpu_windows.py: joints and transforms of O(3 m) carry a few ulp(4) = 4.8e-7 each
# through two rigid maps and the FK (float32 on both sides); the z-scored rows add the statistics' division
EPS = 2.0 ** -23
JOINT_TOL = 64 * 4 * EPS       # 3.1e-5 m
ROW_TOL = 2e-4                 # relative, as windows.npz's rows (the reference's own float32 quaternion helpers)
KP_F64 = 1e-9                  # the float64 undistortion against the float64 reference (cv2 / the oracle), pixels


def _kp_bound(ref):
    """Per element: the float32 rounding of the float64 result (half a float32 spacing, doubled to cover a result that
    rounds across a binade edge) plus KP_F64."""
    return np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + KP_F64


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.fixture(scope="module")
def body(cuda_device):
    return BodyModel.create('', device=cuda_device, seed=0)


def _datasets():
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    tr = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    # the golden's loaders share the pose model's statistics (tools/gen_golden.py gen_windows_video)
    traj = types.SimpleNamespace(Mean=ds.Mean, Std=ds.Std, traj_feat_dim=tr.traj_feat_dim, pose_feat_dim=tr.pose_feat_dim)
    return ds, traj


def _inputs(g, cases, dev):
    """Packed inputs of golden cases (all of one dataset)."""
    ys = {video_case(g, c)[0] for c in cases}
    assert len(ys) == 1
    y_up = ys.pop()
    key = "egobody" if y_up else "prox"
    lengths, params, kp, dm, c2w, m2w, fl, wide, gt = [], {k: [] for k in PARAMS}, [], [], [], [], [], [], {k: [] for k in PARAMS}
    for c in cases:
        _, n, p, cam, master, floor, _ = video_case(g, c)
        lengths.append(n)
        for k in PARAMS:
            params[k].append(p[k])
            if y_up:
                gt[k].append(g[f"c{c}_gt_{k}"])
        kp.append(g[f"c{c}_keypoints25"])
        dm.append(g[f"c{c}_depth_mask"].astype(np.float32))
        c2w.append(cam), m2w.append(master), fl.append(floor), wide.append(bool(g[f"c{c}_kp_float64"]))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.concatenate(a))).to(dev)
    R = len(cases)
    kw = dict(cam2world=np.asarray(c2w), focal_length=np.repeat(g[f"{key}_f"][None], R, 0),
              camera_center=np.repeat(g[f"{key}_c"][None], R, 0), camera_mtx=np.repeat(g[f"{key}_camera_mtx"][None], R, 0),
              dist=np.repeat(g[f"{key}_k"][None], R, 0), keypoints=t(kp), depth_mask=t(dm), floor=fl,
              keypoints_float64=wide)
    if y_up:
        kw.update(gt_params={k: t(v) for k, v in gt.items()}, master2world=np.asarray(m2w))
    return key, {k: t(v) for k, v in params.items()}, lengths, kw


def _encode(g, cases, dev, body, **over):
    key, params, lengths, kw = _inputs(g, cases, dev)
    kw.update(over)
    if 'gt_params' in kw:
        kw['gt_body_model'] = body
    ds, traj = _datasets()
    return windows.encode_video(body, params, lengths, key, pose_dataset=ds, traj_dataset=traj,
                                clip_len=int(g["clip_len"]), overlap=int(g["overlap"]), **kw)


def test_every_key_matches_the_reference_loader(cuda_device, body):
    g = golden("windows_video.npz")
    ds, traj = _datasets()
    near = 0
    for cases in ((0, 1), (2, 3)):
        bt, bp, win = _encode(g, cases, cuda_device, body)
        w0 = 0
        for c in cases:
            table, wins = oracle_case(g, c)
            for w in range(len(wins)):
                W = w0 + w
                tag = (c, w)
                rel = lambda got, want: float((np.abs(got.cpu().double().numpy() - want) / (1 + np.abs(want))).max())
                assert rel(bp['transf_matrix'][W], g[f"c{c}_transf_matrix"][w]) < JOINT_TOL, tag
                assert rel(bp['noisy_joints_scene_coord'][W], g[f"c{c}_noisy_joints_scene_coord"][w]) < JOINT_TOL, tag
                assert rel(bp['noisy_joints'][W], g[f"c{c}_noisy_joints"][w]) < JOINT_TOL, tag
                for k in PARAMS:
                    assert rel(bp['cano_smplx_params_dict'][k][W], g[f"c{c}_cano_{k}"][w]) < 1e-4, (tag, k)
                    assert rel(bp['cano_smplx_params_dict'][k][W], wins[w]['cano_params'][k]) < 1e-4, (tag, k)
                ref = g[f"c{c}_motion_repr_noisy"][w].astype(np.float64)
                for rows in (bp['motion_repr_noisy'][W], bt['motion_repr_noisy'][W]):
                    got = rows.cpu().double().numpy()
                    err = np.abs(got - ref) / (1 + np.abs(ref))
                    assert err[:, :290].max() < ROW_TOL, (tag, np.unravel_index(err[:, :290].argmax(), (23, 290)))
                    # contacts: exact wherever the oracle's foot is farther from a threshold than the joint bound
                    cj = wins[w]['cano_joints']
                    for s, j in enumerate((7, 10, 8, 11)):
                        v2 = ((cj[1:, j] - cj[:-1, j]) ** 2).sum(-1)
                        h = cj[:-1, j, 2] - (0.18 if s % 2 == 0 else 0.15)
                        clear = (np.abs(v2 - 5e-5) > 4 * JOINT_TOL * 0.1) & (np.abs(h) > 4 * JOINT_TOL)
                        near += int((~clear).sum())
                        assert np.array_equal(got[clear, 290 + s], ref[clear, 290 + s]), (tag, s)
                assert torch.equal(bt['cond'][W], bt['motion_repr_noisy'][W][:, list(windows.ABS_TRAJ_CHANNELS)])
                for k in ('mask_joint_vis', 'mask_vec_vis', 'focal_length', 'camera_center'):
                    assert np.array_equal(bp[k][W].cpu().numpy(), g[f"c{c}_{k}"][w].astype(np.float32)), (tag, k)
                    assert torch.equal(bp[k][W], bt[k][W])
                kp = bp['keypoints_2d'][W].cpu().double().numpy()
                ref_kp = g[f"c{c}_keypoints_2d"][w]
                assert (np.abs(kp - ref_kp) <= _kp_bound(ref_kp)).all(), (tag, float(np.abs(kp - ref_kp).max()))
                if 'gt_joints_scene_coord' in bp:
                    assert rel(bp['gt_joints_scene_coord'][W], g[f"c{c}_gt_joints_scene_coord"][w]) < JOINT_TOL, tag
                assert torch.equal(bp['cam2world'][W].cpu(), torch.from_numpy(g[f"c{c}_cam2world"]).float())
            w0 += len(wins)
    print(f"contact decisions within the bound of a threshold: {near}")


def test_identity_camera_gives_encode_joints_rows(cuda_device, body):
    g = golden("windows_video.npz")
    key, params, lengths, kw = _inputs(g, (0, 1), cuda_device)
    R = len(lengths)
    ds, traj = _datasets()
    kw.update(cam2world=np.repeat(np.eye(4)[None], R, 0), floor=None)
    bt, bp, win = windows.encode_video(body, params, lengths, 'prox', pose_dataset=ds, traj_dataset=traj, clip_len=24,
                                       **kw)
    joints = body(**params, return_verts=False).joints[:, 0:22].contiguous()
    t2, p2, w2 = windows.encode_joints(params, joints, lengths, ds, traj, clip_len=24)
    assert torch.equal(_bits(bp['noisy_joints_scene_coord'].reshape(-1, 66)),
                       _bits(torch.cat([joints[s:s + 24].reshape(24, 66) for s in (0, 22, 46)])))
    assert torch.equal(_bits(win.transf), _bits(w2.transf))
    assert torch.equal(_bits(bp['motion_repr_noisy']), _bits(p2['motion_repr_clean']))
    assert torch.equal(_bits(bt['motion_repr_noisy']), _bits(t2['motion_repr_clean']))


def test_identity_camera_gives_encode_joints_rows_145(cuda_device, body):
    """The same at 145 frames (five warps per CTA), on recordings of 145 and 300 frames."""
    dev, lengths = cuda_device, [145, 300]
    recs = [_recording_params(n, 31 + i) for i, n in enumerate(lengths)]
    params = {k: torch.from_numpy(np.concatenate([r[k] for r in recs])).to(dev) for k in PARAMS}
    N, R = sum(lengths), len(lengths)
    ds, traj = _datasets()
    bt, bp, win = windows.encode_video(
        body, params, lengths, 'prox', cam2world=np.repeat(np.eye(4)[None], R, 0), focal_length=np.ones((R, 2)),
        camera_center=np.ones((R, 2)), camera_mtx=np.repeat(np.eye(3)[None], R, 0), dist=np.zeros((R, 4)),
        keypoints=torch.zeros(N, 25, 3, device=dev), depth_mask=torch.ones(N, 25, device=dev), pose_dataset=ds,
        traj_dataset=traj)
    joints = body(**params, return_verts=False).joints[:, 0:22].contiguous()
    t2, p2, w2 = windows.encode_joints(params, joints, lengths, ds, traj)
    assert len(win) == 3
    assert torch.equal(_bits(win.transf), _bits(w2.transf))
    assert torch.equal(_bits(bp['motion_repr_noisy']), _bits(p2['motion_repr_clean']))
    assert torch.equal(_bits(bt['motion_repr_noisy']), _bits(t2['motion_repr_clean']))


def test_each_window_alone_permuted_and_poisoned(cuda_device, body):
    g = golden("windows_video.npz")
    full = _encode(g, (2, 3), cuda_device, body)
    alone = [_encode(g, (c,), cuda_device, body) for c in (2, 3)]
    swapped = _encode(g, (3, 2), cuda_device, body)
    n2 = len(alone[0][2])
    order = list(range(n2, len(full[2]))) + list(range(n2))
    for d in (0, 1):
        for k, v in full[d].items():
            if isinstance(v, dict):
                continue
            assert torch.equal(_bits(v), _bits(torch.cat([alone[0][d][k], alone[1][d][k]]))), k
            assert torch.equal(_bits(v[order]), _bits(swapped[d][k])), k
    # NaN / +-Inf in frames no window covers (case 3 has 46 frames: its last window ends at frame 45, frame 45 is in)
    key, params, lengths, kw = _inputs(g, (2, 3), cuda_device)
    ext = {k: torch.cat([v[:lengths[0]], v[lengths[0]:], torch.full((3,) + v.shape[1:], float('nan'), device=v.device)])
           for k, v in params.items()}
    ext['transl'][-2] = float('inf')
    kw['keypoints'] = torch.cat([kw['keypoints'], torch.full((3, 25, 3), float('-inf'), device=cuda_device)])
    kw['depth_mask'] = torch.cat([kw['depth_mask'], torch.full((3, 25), float('nan'), device=cuda_device)])
    kw['gt_params'] = {k: torch.cat([v, torch.full((3,) + v.shape[1:], float('nan'), device=v.device)])
                       for k, v in kw['gt_params'].items()}
    ds, traj = _datasets()
    bt, bp, win = windows.encode_video(body, ext, [lengths[0], lengths[1] + 3], key, pose_dataset=ds, traj_dataset=traj,
                                       clip_len=24, gt_body_model=body, **kw)
    assert len(win) == len(full[2])
    for k, v in full[1].items():
        if not isinstance(v, dict):
            assert torch.equal(_bits(v), _bits(bp[k])), k


def test_to_recordings_gives_back_the_scene_joints(cuda_device, body):
    g = golden("windows_video.npz")
    for cases in ((0, 1), (2, 3)):
        bt, bp, win = _encode(g, cases, cuda_device, body)
        P = win.clip_len - 2
        world, covered = windows.to_recordings(win, bp['noisy_joints'][:, :P])
        scene = bp['noisy_joints_scene_coord'][:, :P]
        off = 0
        for r, n in enumerate(win.lengths):
            for w in range(len(win)):
                if int(win.recording[w]) != r:
                    continue
                s = int(win.start[w])
                assert bool(covered[r][s:s + P].all())
                assert float((world[r][s:s + P] - scene[w]).abs().max()) < 8 * JOINT_TOL
        if cases == (2, 3):  # y up: the scene's vertical is y, as the loader's scene joints
            assert float(world[0][covered[0]][..., 1].std()) > 0.1


def test_projection_guidance_with_per_window_cameras(cuda_device, body):
    from test_gpu_clip_guidance import _camera
    from test_gpu_posenet_lengths import _guidance_setup
    dev, B, T = cuda_device, 4, 23
    ds, x, m, mean, std, k = _guidance_setup(dev, B, T, 4)
    cam = _camera(ds, B, T, 9, dev)
    xg = x.to(dev)
    m.guidance_normaliser = 'clip'
    try:
        old = m.guide_2d_projection_with_smpl(cam, {'pred_xstart': xg}, None, compute_grad='x_0')
        c2w = torch.eye(4, device=dev).repeat(B, 1, 1)
        c2w[:, 0:3, 0:3], c2w[:, 0:3, 3] = ds.cam_R, ds.cam_t.reshape(3)
        new = m.guide_2d_projection_with_smpl(dict(cam, cam2world=c2w), {'pred_xstart': xg}, None, compute_grad='x_0')
        assert torch.equal(_bits(old), _bits(new))
        # two cameras: each clip gets the bits of the clip alone with its camera as the dataset's
        other = torch.eye(4, device=dev)
        other[0:3, 0:3] = torch.tensor([[0., 0, 1], [1, 0, 0], [0, 1, 0]], device=dev)
        other[0:3, 3] = torch.tensor([4.0, 0.3, 1.1], device=dev)
        c2w[1], c2w[3] = other, other
        got = m.guide_2d_projection_with_smpl(dict(cam, cam2world=c2w), {'pred_xstart': xg}, None, compute_grad='x_0')
        saved = ds.cam_R, ds.cam_t
        for b in range(B):
            ds.cam_R, ds.cam_t = c2w[b, 0:3, 0:3].clone(), c2w[b, 0:3, 3].reshape(1, 3).clone()
            one = {key: v[b:b + 1] for key, v in cam.items()}
            alone = m.guide_2d_projection_with_smpl(one, {'pred_xstart': xg[b:b + 1].contiguous()}, None,
                                                    compute_grad='x_0')
            assert torch.equal(_bits(got[b:b + 1]), _bits(alone)), b
        ds.cam_R, ds.cam_t = saved
        assert not torch.equal(_bits(got[1]), _bits(old[1]))
    finally:
        m.guidance_normaliser = 'batch'


def _rz(a, tilt=0.0):
    ca, sa, ct, st = np.cos(a), np.sin(a), np.cos(tilt), np.sin(tilt)
    return np.array([[ca, -sa, 0], [sa, ca, 0], [0, 0, 1.0]]) @ np.array([[1.0, 0, 0], [0, ct, -st], [0, st, ct]])


@pytest.mark.parametrize("dataset", ["prox", "egobody"])
def test_145_frame_windows_match_the_oracle(cuda_device, body, dataset):
    """Windows of 145 frames (five warps per CTA) against the float64 oracle, every key.  Recordings of 145 and 300 frames
    (three windows); the oracle takes the device's FK joints, so the comparison is of the window path alone.  Bounds:
    the rows and joints by test_gpu_windows._bound on the z-up scene joints, doubled for the camera map's extra roundings
    of size S; the canonical parameters by the same joint bound; keypoints per element (_kp_bound); masks, cameras exact;
    contacts exact wherever the oracle's foot is clear of both thresholds by the joint bound."""
    dev = cuda_device
    y_up = dataset == 'egobody'
    lengths = [145, 300]
    R, N = len(lengths), sum(lengths)
    recs = [_recording_params(n, 21 + i) for i, n in enumerate(lengths)]
    host = {k: np.concatenate([r[k] for r in recs]) for k in PARAMS}
    params = {k: torch.from_numpy(v).to(dev) for k, v in host.items()}
    c2w = np.repeat(np.eye(4)[None], R, 0)
    for r in range(R):
        A = _rz(0.7 + r, 0.05)
        c2w[r, :3, :3] = wvo.Q.T @ A if y_up else A
        c2w[r, :3, 3] = [0.3 * r, -1.2, 2.0 + 0.5 * r]
    gk = np.random.default_rng(4)
    kp = np.concatenate([gk.uniform(-200, 2100, (N, 25, 1)), gk.uniform(-100, 1200, (N, 25, 1)), gk.uniform(0, 1, (N, 25, 1))],
                        -1).astype(np.float32)
    kp[gk.uniform(0, 1, (N, 25)) < 0.05, 2] = np.float32(0.2)
    kp[[10, 200]] = 0  # no person: recording 0 and recording 1 become float64 in the loader
    depth = (gk.uniform(0, 1, (N, 25)) > 0.1).astype(np.float32)
    K = np.array([[1060.53, 0.0, 951.3], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]])
    k = [0.0548, -0.0489, 0.0009, -0.0012, 0.0102]
    floors = [-0.8, 0.0]
    ds, traj = _datasets()
    kw = dict(cam2world=c2w, focal_length=np.repeat([[1060.53, 1060.38]], R, 0),
              camera_center=np.repeat([[951.3, 536.77]], R, 0), camera_mtx=np.repeat(K[None], R, 0),
              dist=np.repeat([k], R, 0), keypoints=torch.from_numpy(kp).to(dev), depth_mask=torch.from_numpy(depth).to(dev),
              floor=floors)
    if y_up:
        kw.update(gt_params=params, gt_body_model=body, master2world=c2w)
    bt, bp, win = windows.encode_video(body, params, lengths, dataset, pose_dataset=ds, traj_dataset=traj, **kw)
    assert len(win) == 3 and win.clip_len == 145
    joints = body(**params, return_verts=False).joints[:, 0:22].cpu().numpy().astype(np.float64)
    off = np.concatenate([[0], np.cumsum(lengths)])
    clear_total = near = 0
    for w, (r, s) in enumerate(windows.window_table(lengths)):
        rows = slice(off[r] + s, off[r] + s + 145)
        c32 = c2w[r].astype(np.float32).astype(np.float64)
        o = wvo.encode_window_video(joints[rows], {key: v[rows] for key, v in host.items()}, c32, y_up, floors[r])
        zj = o['scene_joints'] @ wvo.Q.T if y_up else o['scene_joints']
        S = float(np.abs(zj).max())
        jb = 2 * 32 * EPS * (1 + S)
        got = lambda key: bp[key][w].cpu().double().numpy()
        assert np.abs(got('noisy_joints_scene_coord') - o['scene_joints']).max() <= jb, w
        assert np.abs(got('noisy_joints') - o['cano_joints']).max() <= jb, w
        assert np.abs(got('transf_matrix') - o['transf']).max() <= jb, w
        for key in ('transl', 'betas', 'body_pose'):
            assert np.abs(bp['cano_smplx_params_dict'][key][w].cpu().double().numpy() - o['cano_params'][key]).max() <= jb, key
        from scipy.spatial.transform import Rotation
        Rg = Rotation.from_rotvec(bp['cano_smplx_params_dict']['global_orient'][w].cpu().double().numpy()).as_matrix()
        assert np.abs(Rg - Rotation.from_rotvec(o['cano_params']['global_orient']).as_matrix()).max() <= jb, w
        rep = o['repr']
        b = 2 * _bound(zj, rep)
        for rows_, stats in ((bp['motion_repr_noisy'][w], ds), (bt['motion_repr_noisy'][w], traj)):
            de = rows_.cpu().double().numpy() * stats.Std + stats.Mean
            ratio = (np.abs(de - rep) / (b + EPS * np.abs(stats.Mean)))[:, :290]
            assert ratio.max() <= 1.0, (w, np.unravel_index(ratio.argmax(), ratio.shape))
            cj = o['cano_joints']
            for c, j in enumerate((7, 10, 8, 11)):
                v2 = ((cj[1:, j] - cj[:-1, j]) ** 2).sum(-1)
                h = cj[:-1, j, 2] - (0.18 if c % 2 == 0 else 0.15)
                dv = 4 * jb * np.sqrt(v2) + 4 * jb * jb
                clear = (np.abs(v2 - 5e-5) > dv) & (np.abs(h) > jb)
                clear_total += int(clear.sum())
                near += int((~clear).sum())
                assert np.array_equal(de[clear, 290 + c], rep[clear, 290 + c]), (w, c)
        wide = bool((kp[off[r]:off[r + 1]] == 0).all(axis=(1, 2)).any())
        kpo, vis, vec = wvo.keypoints_window(kp[rows], depth[rows], not y_up, K, k, wide)
        assert (np.abs(got('keypoints_2d') - kpo) <= _kp_bound(kpo)).all(), w
        assert np.array_equal(got('mask_joint_vis'), vis) and np.array_equal(got('mask_vec_vis'), vec), w
        assert np.array_equal(got('focal_length'), np.float32([1060.53, 1060.38]).astype(np.float64))
        assert np.array_equal(got('camera_center'), np.float32([951.3, 536.77]).astype(np.float64))
        assert np.array_equal(got('cam2world'), c2w[r].astype(np.float32).astype(np.float64))
        if y_up:
            assert np.abs(got('gt_joints_scene_coord') - o['scene_joints']).max() <= jb, w
        for key in bt:  # the traj dict shares every key but its rows and TrajNet inputs
            if key not in ('motion_repr_noisy', 'cond', 'control_cond', 'cano_smplx_params_dict'):
                assert torch.equal(bt[key][w], bp[key][w]), key
    assert clear_total > 0
    print(f"{dataset}: {near} contact decisions within the bound of a threshold, {clear_total} clear")


def test_guided_prox_loop_with_per_window_cameras(cuda_device):
    """A guided grad_type='prox' PoseNet loop with the 'clip' normaliser and one generator per window, on six windows of
    three cameras (groups of 3, 2 and 1 windows): each window gets the bits of its loop alone with its camera as
    dataset.cam_R / cam_t."""
    from test_gpu_clip_guidance import _guided_diff, _loop_batch
    from test_gpu_noise_streams import _gens
    from test_gpu_posenet_lengths import _model
    dev, B, T = cuda_device, 6, 64
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    m = _model(dev, ds)
    batch = _loop_batch(m, dev, 'prox', lengths=[T] * B, T=T)
    del batch['lengths']
    cams = []
    for i in range(3):
        c = torch.eye(4)
        c[:3, :3] = torch.from_numpy(_rz(0.9 * i, 0.1 * i) @ np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]])).float()
        c[:3, 3] = torch.tensor([0.2 + i, -5.0 + 0.5 * i, 1.0])
        cams.append(c)
    which = [0, 1, 0, 2, 1, 0]
    batch['cam2world'] = torch.stack([cams[i] for i in which]).to(dev)
    seeds = [51, 52, 53, 54, 55, 56]
    m.guidance_normaliser = 'clip'
    saved = ds.cam_R, ds.cam_t
    try:
        out = _guided_diff(dev).p_sample_loop(m, dict(batch, generators=_gens(dev, seeds)), [B, 294, 1, T],
                                              clip_denoised=False, cond_fn_with_grad=True, grad_type='prox')
        finite = 0
        for b in range(B):
            c = batch['cam2world'][b]
            ds.cam_R, ds.cam_t = c[:3, :3].clone(), c[:3, 3].reshape(1, 3).clone()
            one = {k: v[b:b + 1] for k, v in batch.items() if k != 'cam2world'}
            alone = _guided_diff(dev).p_sample_loop(m, dict(one, generators=_gens(dev, [seeds[b]])), [1, 294, 1, T],
                                                    clip_denoised=False, cond_fn_with_grad=True, grad_type='prox')
            assert torch.equal(_bits(out[b:b + 1]), _bits(alone)), b
            finite += int(bool(torch.isfinite(alone).all()))
        print(f"prox loop with per-window cameras: {finite} of {B} windows finite")
    finally:
        ds.cam_R, ds.cam_t = saved
        m.guidance_normaliser = 'batch'
