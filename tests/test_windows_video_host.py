"""CPU: the float64 video-window oracle (oracle/windows_video_oracle.py) against the reference's DataloaderVideo, pinned by
tests/golden/windows_video.npz (tools/gen_golden.py gen_windows_video), its undistortion against cv2, the EgoBody
canonical frame as cano_seq_smplx after Q, and encode_video's refusals before any device work."""
import numpy as np
import pytest
import torch

from helpers import golden
from oracle import kinematics_oracle as ko
from oracle import windows_video_oracle as wvo
from rohm_b200 import synthetic, windows
from rohm_b200._lib import RohmB200Error

PARAMS = ("global_orient", "transl", "betas", "body_pose")


def video_case(g, c):
    """Inputs of golden case c: (y_up, frames, params, cam2world, master2world, floor, camera dict)."""
    y_up, n, _ = (int(v) for v in g[f"c{c}_meta"])
    key = "egobody" if y_up else "prox"
    cam = {k: g[f"{key}_{k}"] for k in ("f", "c", "camera_mtx", "k")}
    params = {k: g[f"c{c}_param_{k}"] for k in PARAMS}
    return bool(y_up), n, params, g[f"c{c}_cam2world"], g[f"c{c}_master2world"], float(g[f"c{c}_floor"]), cam


def fk(params):
    t = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in params.items()}
    j, _ = ko.smplx_forward(synthetic.smplx_like_model(0), t['global_orient'], t['body_pose'], t['betas'], t['transl'],
                            return_verts=False)
    return j[:, 0:22].numpy()


def oracle_case(g, c):
    y_up, n, params, cam2world, master, floor, cam = video_case(g, c)
    L = int(g["clip_len"])
    cam32 = cam2world.astype(np.float32).astype(np.float64)  # the loader applies cam2world.float()
    table, wins = wvo.encode_video(params, fk(params), [n], cam32[None], y_up, [floor], L, int(g["overlap"]))
    return table, wins


def test_oracle_matches_the_reference_video_loader():
    g = golden("windows_video.npz")
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    for c in range(int(g["n_cases"])):
        y_up, n, params, cam2world, master, floor, cam = video_case(g, c)
        table, wins = oracle_case(g, c)
        assert len(wins) == g[f"c{c}_transf_matrix"].shape[0]
        for w, win in enumerate(wins):
            tag = (c, w)
            # float32 loader arrays (joints, the quaternion helpers) against float64: relative 2e-5 as windows.npz
            rel = lambda a, b: float((np.abs(a - b) / (1.0 + np.abs(b))).max())
            assert rel(win['transf'], g[f"c{c}_transf_matrix"][w]) < 1e-6, tag
            assert rel(win['scene_joints'], g[f"c{c}_noisy_joints_scene_coord"][w]) < 1e-6, tag
            assert rel(win['cano_joints'], g[f"c{c}_noisy_joints"][w]) < 1e-5, tag
            for k in PARAMS:
                assert rel(win['cano_params'][k], g[f"c{c}_cano_{k}"][w]) < 1e-5, (tag, k)
            rep = (win['repr'] - ds.Mean) / ds.Std
            ref = g[f"c{c}_motion_repr_noisy"][w]
            err = np.abs(rep - ref) / (1.0 + np.abs(ref))
            assert err[:, :290].max() < 2e-4, (tag, np.unravel_index(err[:, :290].argmax(), err[:, :290].shape))
            assert np.array_equal(rep[:, 290:], ref[:, 290:]), tag
            r, s = table[w]
            rows = slice(s, s + int(g["clip_len"]))
            kp, vis, vec = wvo.keypoints_window(g[f"c{c}_keypoints25"][rows], g[f"c{c}_depth_mask"][rows], not y_up,
                                                cam['camera_mtx'], cam['k'], bool(g[f"c{c}_kp_float64"]))
            assert np.abs(kp - g[f"c{c}_keypoints_2d"][w]).max() < 1e-9, tag
            assert np.array_equal(vis, g[f"c{c}_mask_joint_vis"][w]), tag
            assert np.array_equal(vec, g[f"c{c}_mask_vec_vis"][w]), tag
            assert np.array_equal(g[f"c{c}_focal_length"][w], cam['f'].astype(np.float32))
            assert np.array_equal(g[f"c{c}_camera_center"][w], cam['c'].astype(np.float32))
            if y_up:
                gt = {k: g[f"c{c}_gt_{k}"] for k in PARAMS}
                m = master.astype(np.float32).astype(np.float64)
                want = fk(gt)[rows].astype(np.float64) @ m[:3, :3].T + m[:3, 3]
                assert rel(want, g[f"c{c}_gt_joints_scene_coord"][w]) < 1e-6, tag


def test_golden_covers_the_cases_the_issue_names():
    g = golden("windows_video.npz")
    ups = [int(g[f"c{c}_meta"][0]) for c in range(int(g["n_cases"]))]
    assert sorted(set(ups)) == [0, 1]
    assert any(int(g[f"c{c}_meta"][2]) for c in range(4))  # an EgoBody sub view
    floors = [float(g[f"c{c}_floor"]) for c in range(4)]
    assert any(f != 0 for f in floors) and any(f == 0 for f in floors)
    kp64 = [bool(g[f"c{c}_kp_float64"]) for c in range(4)]
    assert any(kp64) and not all(kp64)
    # confidence exactly 0.2f: True in float64, False in float32
    for c in range(4):
        conf = g[f"c{c}_keypoints25"][..., 2]
        assert (conf == np.float32(0.2)).any()
    # contact masks both ways, and a depth zero on each foot joint
    vec = np.concatenate([g[f"c{c}_mask_vec_vis"].reshape(-1, 294) for c in range(4)])
    assert vec[:, 290].min() == 0 and vec[:, 290].max() == 1 and vec[:, 292].max() == 1
    dm = np.concatenate([g[f"c{c}_depth_mask"] for c in range(4)])
    assert all((~dm[:, j]).any() for j in (7, 8, 10, 11))
    # global rotations near pi in the canonical frame of some window
    ang = np.concatenate([np.linalg.norm(g[f"c{c}_cano_global_orient"], axis=-1).ravel() for c in range(4)])
    assert np.abs(ang - np.pi).min() < 0.2


def test_floor_zero_takes_the_window_minimum():
    g = golden("windows_video.npz")
    c = 1  # preset floor 0.0
    assert float(g[f"c{c}_floor"]) == 0.0
    z = g[f"c{c}_noisy_joints"][..., 2]
    assert abs(float(z.min(axis=(1, 2)).max())) < 1e-6  # the window's lowest joint sits on the floor
    table, wins = oracle_case(g, c)
    assert np.abs(wins[0]['transf'] - g[f"c{c}_transf_matrix"][0]).max() < 1e-6


def test_undistortion_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    g = np.random.default_rng(5)
    K = np.array([[1060.53, 0.0, 951.3], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]])
    pts = np.concatenate([np.stack([g.uniform(0, 1920, 200), g.uniform(0, 1080, 200)], -1),
                          [[0, 0], [1919, 1079], [0, 1079], [1919, 0], [-6000, 9000], [12000, -7000], [1e5, 1e5]]])
    for k in ([0.0548, -0.0489, 0.0009, -0.0012], [0.0548, -0.0489, 0.0009, -0.0012, 0.0102],
              [0.4761, -2.7413, 0.0004, -0.0002, 1.5812, 0.3563, -2.5628, 1.5138], [-0.9, 0.0, 0.0, 0.0]):
        want = cv2.undistortPoints(pts.reshape(-1, 1, 2), K, np.asarray(k), P=K).reshape(-1, 2)
        got = wvo.undistort_points(pts, K, k)
        assert np.abs(got - want).max() < 1e-9, k
    # a far point under k1 = -0.9 comes back unchanged (negative icdist)
    far = np.array([[-6000.0, 9000.0]])
    assert np.abs(wvo.undistort_points(far, K, [-0.9, 0, 0, 0]) - far).max() < 1e-9


def test_egobody_frame_is_cano_seq_smplx_after_q():
    """T_z Q equals the reference's cano_seq_smplx_egobody transf_matrix, and cano_seq_smplx of Q p its canonical joints
    and parameters (float64, random joints and parameters, both floor modes; the reference's outputs are the golden's
    q* arrays)."""
    from scipy.spatial.transform import Rotation
    from oracle.windows_noise_oracle import canonical_params
    g = golden("windows_video.npz")
    floors = []
    for t in range(int(g["q_trials"])):
        j, floor = g[f"q{t}_joints"], float(g[f"q{t}_floor"])
        floors.append(floor)
        tz = wvo.canonical_frame(j @ wvo.Q.T, floor)
        qq = np.eye(4)
        qq[:3, :3] = wvo.Q
        assert np.abs(tz @ qq - g[f"q{t}_transf"]).max() < 1e-12, t
        assert np.abs((j @ wvo.Q.T) @ tz[:3, :3].T + tz[:3, 3] - g[f"q{t}_cano_joints"]).max() < 1e-12, t
        # the parameters through Q: the pelvis moves, delta_T = pelvis - transl does not
        go, tr = g[f"q{t}_global_orient"], g[f"q{t}_transl"]
        delta = j[:, 0] - tr
        zp = {'global_orient': Rotation.from_matrix(wvo.Q @ Rotation.from_rotvec(go).as_matrix()).as_rotvec(),
              'transl': j[:, 0] @ wvo.Q.T - delta}
        cp = canonical_params(zp, j @ wvo.Q.T, tz)
        ref_R = Rotation.from_rotvec(g[f"q{t}_cano_global_orient"]).as_matrix()
        assert np.abs(Rotation.from_rotvec(cp['global_orient']).as_matrix() - ref_R).max() < 1e-12, t
        assert np.abs(cp['transl'] - g[f"q{t}_cano_transl"]).max() < 1e-12, t
    assert any(f == 0 for f in floors) and any(f != 0 for f in floors)


def test_refusals_before_any_device_work():
    N, R = 30, 1
    p = {k: torch.zeros(N, w) for k, w in windows.PARAMS}
    good = dict(cam2world=np.eye(4)[None], focal_length=np.ones((R, 2)), camera_center=np.ones((R, 2)),
                camera_mtx=np.eye(3)[None], dist=np.zeros((R, 5)), keypoints=torch.zeros(N, 25, 3),
                depth_mask=torch.zeros(N, 25), pose_dataset=None, traj_dataset=None)

    def call(**kw):
        a = dict(good, **kw)
        return windows.encode_video(None, p, [N], a.pop('dataset', 'prox'), clip_len=a.pop('clip_len', 24),
                                    overlap=a.pop('overlap', 2), **a)

    with pytest.raises(RohmB200Error, match="noise"):
        call(noise=object())
    with pytest.raises(RohmB200Error, match="dataset"):
        call(dataset='amass')
    for clip_len, overlap in ((24, 3), (2, 0), (161, 0), (24, -1)):
        with pytest.raises(RohmB200Error, match="clip_len"):
            call(clip_len=clip_len, overlap=overlap)
    with pytest.raises(RohmB200Error, match="dist"):
        call(dist=np.zeros((R, 6)))
    with pytest.raises(RohmB200Error, match="cam2world"):
        call(cam2world=np.eye(4))
    bad = np.eye(4)[None].copy()
    bad[0, 0, 3] = np.inf
    with pytest.raises(RohmB200Error, match="non-finite"):
        call(cam2world=bad)
    with pytest.raises(RohmB200Error, match="non-finite"):
        call(focal_length=np.array([[np.nan, 1.0]]))
    with pytest.raises(RohmB200Error, match="keypoints"):
        call(keypoints=torch.zeros(N, 22, 3))
    with pytest.raises(RohmB200Error, match="depth_mask"):
        call(depth_mask=torch.zeros(N - 1, 25))
    with pytest.raises(RohmB200Error, match="ground truth"):
        call(dataset='egobody', master2world=np.eye(4)[None])
    with pytest.raises(RohmB200Error, match="CUDA"):
        call()
