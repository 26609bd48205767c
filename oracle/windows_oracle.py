"""Oracle (test infrastructure only): sliding-window batching of whole recordings, restated in float64.

* window rule            data_loaders/dataloader_video.py:160-183 (overlap 2), dataloader_amass.py:105-131 (overlap 0)
* canonical frame        data_loaders/motion_representation.py:47-110 cano_seq_smplx, utils/other_utils.py:189-240
                         update_globalRT_for_smplx (delta_T = pelvis - transl)
* 294-channel encoding   data_loaders/motion_representation.py:187-282 get_repr_smplx, :23-44 foot_detect
* back to the world      eval_prox_egobody.py:177-182 (points_coord_trans with the inverse of transf_matrix)

numpy float64 throughout.  Pinned by tests/golden/windows.npz, produced by the unmodified reference functions
(tools/gen_golden.py gen_windows).
"""
import numpy as np

from .glue_oracle import rotvec_to_matrix

FEET = ((7, 10), (8, 11))     # foot_detect fid_l, fid_r
FOOT_HEIGHTS = (0.18, 0.15)   # heightfactor, per index into a foot pair
FOOT_VEL = 5e-5               # get_repr_smplx feet_vel_thre


def window_table(lengths, clip_len, overlap):
    """The reference loop: start = k * (clip_len - overlap) while start + clip_len <= frames -> [(recording, start)]."""
    out = []
    for r, n in enumerate(lengths):
        k = 0
        while True:
            start = k * (clip_len - overlap)
            if start + clip_len > n:
                break
            out.append((r, start))
            k += 1
    return out


def canonical_frame(joints):
    """transf_matrix of cano_seq_smplx for one window's joints [T,22,3]: floor at the lowest joint, frame-0 root XY at the
    origin, frame 0 facing +y."""
    j = np.asarray(joints, np.float64)
    floor = j[..., 2].min()
    o = np.array([j[0, 0, 0], j[0, 0, 1], floor])
    x = (j[0, 2] - j[0, 1]) + (j[0, 17] - j[0, 16])
    x[2] = 0
    x = x / np.linalg.norm(x)
    y = np.cross([0.0, 0.0, 1.0], x)
    y = y / np.linalg.norm(y)
    rt = np.stack([x, y, [0.0, 0.0, 1.0]])  # rows: the canonical axes in world coordinates
    m = np.eye(4)
    m[:3, :3], m[:3, 3] = rt, -rt @ o
    return m


def _qmul(q, r):
    w = q[..., 0] * r[..., 0] - q[..., 1] * r[..., 1] - q[..., 2] * r[..., 2] - q[..., 3] * r[..., 3]
    x = q[..., 0] * r[..., 1] + q[..., 1] * r[..., 0] + q[..., 2] * r[..., 3] - q[..., 3] * r[..., 2]
    y = q[..., 0] * r[..., 2] - q[..., 1] * r[..., 3] + q[..., 2] * r[..., 0] + q[..., 3] * r[..., 1]
    z = q[..., 0] * r[..., 3] + q[..., 1] * r[..., 2] - q[..., 2] * r[..., 1] + q[..., 3] * r[..., 0]
    return np.stack([w, x, y, z], axis=-1)


def _qrot(q, v):
    uv = np.cross(q[..., 1:], v)
    uuv = np.cross(q[..., 1:], uv)
    return v + 2 * (q[..., :1] * uv + uuv)


def encode_window(joints, global_orient, transl, betas, body_pose, transf):
    """get_repr_smplx of one window after cano_seq_smplx -> [T-1, 294] (REPR_LIST order, un-normalised)."""
    j = np.asarray(joints, np.float64)
    T = j.shape[0]
    rt, tv = transf[:3, :3], transf[:3, 3]
    c = j @ rt.T + tv
    R = rt @ rotvec_to_matrix(global_orient)
    delta = j[:, 0] - transl
    tr = (transl + delta) @ rt.T + tv - delta
    across = (c[:, 1] - c[:, 2]) + (c[:, 17] - c[:, 16])
    with np.errstate(invalid='ignore', divide='ignore'):
        across = across / np.linalg.norm(across, axis=-1, keepdims=True)
        fwd = np.cross([0.0, 0.0, 1.0], across)
        fwd = fwd / np.linalg.norm(fwd, axis=-1, keepdims=True)
        q = np.concatenate([np.linalg.norm(fwd, axis=-1, keepdims=True) + fwd[:, 1:2],
                            np.cross(fwd, [0.0, 1.0, 0.0])], axis=-1)
        q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    bad = np.where(np.isnan(q).any(axis=-1))[0]
    if len(bad):
        q[bad[0]] = q[bad[0] - 1]
    q[0] = [1.0, 0.0, 0.0, 0.0]
    qv = _qmul(q[1:], q[:-1] * [1.0, -1.0, -1.0, -1.0])
    local = c.copy()
    local[..., 0:2] -= c[:, 0:1, 0:2]
    local = _qrot(np.repeat(q[:, None], 22, axis=1), local)
    lvel = _qrot(np.repeat(q[:-1, None], 22, axis=1), c[1:] - c[:-1])
    w = np.matmul(R[1:] - R[:-1], np.transpose(R[:-1], (0, 2, 1)))
    rot_vel = np.stack([(-w[:, 1, 2] + w[:, 2, 1]) / 2, (w[:, 0, 2] - w[:, 2, 0]) / 2, (-w[:, 0, 1] + w[:, 1, 0]) / 2], -1)
    pose6 = rotvec_to_matrix(np.asarray(body_pose, np.float64).reshape(T, 21, 3))[..., :2].reshape(T, 126)
    feet = []
    for pair in FEET:
        for k, jj in enumerate(pair):
            v2 = ((c[1:, jj] - c[:-1, jj]) ** 2).sum(-1)
            feet.append(((v2 < FOOT_VEL) & (c[:-1, jj, 2] < FOOT_HEIGHTS[k])).astype(np.float64))
    return np.concatenate([
        np.arctan2(q[:-1, 3:4], q[:-1, 0:1]), np.arctan2(qv[:, 3:4], qv[:, 0:1]), c[:-1, 0, 0:2],
        _qrot(q[1:], c[1:, 0] - c[:-1, 0])[:, 0:2], c[:-1, 0, 2:3], R[:-1, :, 0:2].reshape(T - 1, 6), rot_vel, tr[:-1],
        tr[1:] - tr[:-1], local[:-1].reshape(T - 1, 66), lvel.reshape(T - 1, 66), pose6[:-1],
        np.asarray(betas, np.float64)[:-1], np.stack(feet, -1)], axis=-1)


def encode(params, joints, lengths, clip_len=145, overlap=2):
    """params: dict of packed float arrays (global_orient [N,3], transl [N,3], betas [N,10], body_pose [N,63]), joints
    [N,22,3] world positions, lengths per recording -> (table [(recording, start)], transf [W,4,4], repr [W,clip_len-1,294])."""
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    table = window_table(lengths, clip_len, overlap)
    tf, rep = [], []
    for r, s in table:
        rows = slice(off[r] + s, off[r] + s + clip_len)
        m = canonical_frame(joints[rows])
        p = {k: np.asarray(v[rows], np.float64) for k, v in params.items()}
        tf.append(m)
        rep.append(encode_window(joints[rows], p['global_orient'], p['transl'], p['betas'], p['body_pose'], m))
    return (table, np.asarray(tf).reshape(-1, 4, 4),
            np.asarray(rep).reshape(-1, clip_len - 1, 294))


def to_world(cano_joints, table, transf, lengths, clip_len=145):
    """cano_joints [W, clip_len-2, 22, 3] -> (world [N,22,3] packed by recording, covered bool [N])."""
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    world = np.zeros((int(off[-1]), 22, 3))
    covered = np.zeros(int(off[-1]), dtype=bool)
    for w, (r, s) in enumerate(table):
        inv = np.linalg.inv(transf[w])
        rows = slice(off[r] + s, off[r] + s + clip_len - 2)
        world[rows] = np.asarray(cano_joints[w], np.float64) @ inv[:3, :3].T + inv[:3, 3]
        covered[rows] = True
    return world, covered
