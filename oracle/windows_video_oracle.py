"""Oracle (test infrastructure only): the video loader's windows (DataloaderVideo, PROX and EgoBody), restated in float64.

* camera frame -> scene   data_loaders/dataloader_video.py:127-142 / :287-301 (joints by cam2world, update_globalRT_for_smplx
                          with delta_T = pelvis - transl)
* canonical frame         PROX: motion_representation.py:47-110 cano_seq_smplx; EgoBody: cano_seq_smplx of Q p with
                          Q = Rx(+90 deg), (x, y, z) -> (x, -z, y), and transf_matrix = T_z Q, which is what
                          cano_seq_smplx_egobody (:113-184) computes (DESIGN §4.14)
* keypoints and masks     dataloader_video.py:441-484 (BODY_25 -> SMPL, PROX flip + cv2.undistortPoints + flip back,
                          mask_joint_vis, mask_vec_vis); undistort_points restates OpenCV 4.13's cvUndistortPointsInternal
                          (5 fixed iterations, a negative icdist keeps the input point)

numpy float64 throughout; the 294-channel encoding is oracle/windows_oracle.py's encode_window and the canonical
parameters windows_noise_oracle.canonical_params.  Pinned by tests/golden/windows_video.npz, produced by the reference's own
DataloaderVideo (tools/gen_golden.py gen_windows_video).
"""
import numpy as np
from scipy.spatial.transform import Rotation

from .glue_oracle import rotvec_to_matrix
from .windows_noise_oracle import canonical_params
from .windows_oracle import encode_window, window_table

Q = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])  # y-up scene -> z-up
BODY25_TO_SMPL = [8, 12, 9, 8, 13, 10, 8, 14, 11, 1, 20, 23, 1, 5, 2, 0, 5, 2, 6, 3, 7, 4]
FLIP_X = 1919.0
UNDISTORT_ITERS = 5


def undistort_points(pts, K, k):
    """cv2.undistortPoints(pts, K, k, P=K) in float64, OpenCV's order of operations: pts [n,2] -> [n,2]."""
    kk = np.zeros(14)
    kk[:len(k)] = k
    K = np.asarray(K, np.float64)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    ifx, ify = 1.0 / fx, 1.0 / fy
    out = np.empty((len(pts), 2))
    for i, (u, v) in enumerate(np.asarray(pts, np.float64)):
        x, y = (u - cx) * ifx, (v - cy) * ify
        x0, y0 = x, y
        for _ in range(UNDISTORT_ITERS):
            r2 = x * x + y * y
            icdist = (1 + ((kk[7] * r2 + kk[6]) * r2 + kk[5]) * r2) / (1 + ((kk[4] * r2 + kk[1]) * r2 + kk[0]) * r2)
            if icdist < 0:
                x, y = (u - cx) * ifx, (v - cy) * ify
                break
            dx = 2 * kk[2] * x * y + kk[3] * (r2 + 2 * x * x) + kk[8] * r2 + kk[9] * r2 * r2
            dy = kk[2] * (r2 + 2 * y * y) + 2 * kk[3] * x * y + kk[10] * r2 + kk[11] * r2 * r2
            x, y = (x0 - dx) * icdist, (y0 - dy) * icdist
        xx = K[0, 0] * x + K[0, 1] * y + K[0, 2]
        yy = K[1, 0] * x + K[1, 1] * y + K[1, 2]
        ww = 1.0 / (K[2, 0] * x + K[2, 1] * y + K[2, 2])
        out[i] = xx * ww, yy * ww
    return out


def keypoints_window(kp25, depth, prox, K, k, wide):
    """One window's 2-D inputs: kp25 [T,25,3] (float32 values), depth [T,25], wide: the loader's array is float64 ->
    (keypoints_2d [T,22,3], mask_joint_vis [T,22], mask_vec_vis [T,294]), float64."""
    kp = np.asarray(kp25)[:, BODY25_TO_SMPL]
    kp = kp.astype(np.float64 if wide else np.float32)
    conf = kp[..., 2] > (0.2 if wide else np.float32(0.2))
    out = kp.astype(np.float64)
    if prox:
        x = (FLIP_X - kp[..., 0]).astype(np.float64)  # float32 arithmetic for a float32 array
        pts = undistort_points(np.stack([x, out[..., 1]], -1).reshape(-1, 2), K, k).reshape(kp.shape[0], 22, 2)
        out[..., 0] = FLIP_X - pts[..., 0]
        out[..., 1] = pts[..., 1]
    vis = conf * np.asarray(depth, np.float64)[:, 0:22]
    T = vis.shape[0]
    left = (vis[:, 7] == 1) & (vis[:, 10] == 1)
    right = (vis[:, 8] == 1) & (vis[:, 11] == 1)
    feet = np.zeros((T, 4))
    feet[left, 0:2] = 1.0
    feet[right, 2:4] = 1.0
    vec = np.concatenate([np.ones((T, 22)), vis.repeat(3, axis=1), vis.repeat(3, axis=1), vis[:, 1:].repeat(6, axis=1),
                          np.ones((T, 10)), feet], axis=-1)
    return out, vis, vec


def canonical_frame(joints_z, floor=None):
    """cano_seq_smplx's transf_matrix for z-up joints [T,22,3]; floor: a preset height (falsy: the window minimum)."""
    j = np.asarray(joints_z, np.float64)
    fl = floor if floor else j[..., 2].min()
    o = np.array([j[0, 0, 0], j[0, 0, 1], fl])
    x = (j[0, 2] - j[0, 1]) + (j[0, 17] - j[0, 16])
    x[2] = 0
    x = x / np.linalg.norm(x)
    y = np.cross([0.0, 0.0, 1.0], x)
    y = y / np.linalg.norm(y)
    rt = np.stack([x, y, [0.0, 0.0, 1.0]])
    m = np.eye(4)
    m[:3, :3], m[:3, 3] = rt, -rt @ o
    return m


def scene_window(joints_cam, params_cam, cam2world):
    """The loader's scene-frame joints and SMPL-X parameters of one window from camera-frame ones (float64)."""
    c = np.asarray(cam2world, np.float64)
    j = np.asarray(joints_cam, np.float64)
    p = {k: np.asarray(v, np.float64) for k, v in params_cam.items()}
    delta = j[:, 0] - p['transl']
    scene = dict(p)
    scene['global_orient'] = Rotation.from_matrix(c[:3, :3] @ rotvec_to_matrix(p['global_orient'])).as_rotvec()
    scene['transl'] = (p['transl'] + delta) @ c[:3, :3].T + c[:3, 3] - delta
    return j @ c[:3, :3].T + c[:3, 3], scene


def encode_window_video(joints_cam, params_cam, cam2world, y_up, floor=None):
    """One window -> dict of scene joints, transf (scene -> canonical), canonical joints, canonical parameters and the
    un-normalised representation [T-1,294]."""
    scene_j, scene_p = scene_window(joints_cam, params_cam, cam2world)
    z_j, z_p = scene_j, scene_p
    if y_up:
        # update_globalRT_for_smplx with the fixed rotation Q: the pelvis moves, delta_T = pelvis - transl does not
        delta = scene_j[:, 0] - scene_p['transl']
        z_j = scene_j @ Q.T
        z_p = dict(scene_p, global_orient=Rotation.from_matrix(Q @ rotvec_to_matrix(scene_p['global_orient'])).as_rotvec(),
                   transl=z_j[:, 0] - delta)
    tz = canonical_frame(z_j, floor)
    cano_p = canonical_params(z_p, z_j, tz)
    cano_j = z_j @ tz[:3, :3].T + tz[:3, 3]
    rep = encode_window(z_j, z_p['global_orient'], z_p['transl'], z_p['betas'], z_p['body_pose'], tz)
    transf = tz.copy()
    if y_up:
        qq = np.eye(4)
        qq[:3, :3] = Q
        transf = tz @ qq
    return {'scene_joints': scene_j, 'transf': transf, 'cano_joints': cano_j, 'cano_params': cano_p, 'repr': rep}


def encode_video(params_cam, joints_cam, lengths, cam2world, y_up, floors=None, clip_len=145, overlap=2):
    """Every window of R recordings packed frame after frame -> (table, list of encode_window_video dicts)."""
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    out = []
    table = window_table(lengths, clip_len, overlap)
    for r, s in table:
        rows = slice(off[r] + s, off[r] + s + clip_len)
        out.append(encode_window_video(joints_cam[rows], {k: v[rows] for k, v in params_cam.items()}, cam2world[r], y_up,
                                       None if floors is None else floors[r]))
    return table, out
