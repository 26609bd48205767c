"""Oracle (test infrastructure only): input noise on the windows of whole recordings, restated in float64.

* input noise            data_loaders/dataloader_amass.py:156-215 (sep_noise False): noise on the canonical SMPL-X
                         parameters, scipy 'zxy' Euler angles for the rotations, FK of the noisy parameters, get_repr_smplx
                         of the noisy window without re-canonicalisation
* canonical R/T          utils/other_utils.py:189-240 update_globalRT_for_smplx (delta_T = pelvis - transl)

numpy float64 throughout (scipy Rotation for from_euler / as_rotvec, the noisy FK in float64 through the oracle body);
the window rule, canonical frame and encoding are oracle/windows_oracle.py's.  Pinned by tests/golden/windows_noise.npz,
produced by the reference's own DataloaderAMASS (tools/gen_golden.py gen_windows_noise).
"""
import numpy as np
import torch
from scipy.spatial.transform import Rotation

from . import kinematics_oracle as ko
from .glue_oracle import rotvec_to_matrix
from .windows_oracle import canonical_frame, encode_window, window_table

EULER_LOCK = 1e-7  # scipy's gimbal-lock threshold on the (unshifted) middle angle, radians


def quat_from_rotvec(rv):
    """Rotation.from_rotvec(rv).as_quat() (scalar last), float64."""
    rv = np.asarray(rv, np.float64)
    a = np.linalg.norm(rv, axis=-1, keepdims=True)
    a2 = a * a
    sc = np.where(a <= 1e-3, 0.5 - a2 / 48 + a2 * a2 / 3840, np.sin(a / 2) / np.where(a <= 1e-3, 1.0, a))
    return np.concatenate([sc * rv, np.cos(a / 2)], axis=-1)


def euler_zxy(quat):
    """Rotation.from_quat(quat).as_euler('zxy') in radians, restated: scipy 1.18's quaternion method (Bernardes & Viollet
    2022) for the extrinsic sequence z, x, y.  Middle angle in [-pi/2, pi/2]; within EULER_LOCK of the gimbal lock
    (middle angle +-pi/2) the third angle is 0 and the first takes the whole rotation about the vertical; every angle
    brought into [-pi, pi] by one turn where it lies outside (scipy's rule: an exact +-pi stays as computed)."""
    q = np.asarray(quat, np.float64)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    a, b, c, d = w - x, z + y, x + w, y - z
    hs, hd = np.arctan2(b, a), np.arctan2(d, c)
    th = 2 * np.arctan2(np.hypot(c, d), np.hypot(a, b))
    lock0, lock1 = np.abs(th) <= EULER_LOCK, np.abs(th - np.pi) <= EULER_LOCK
    lock = lock0 | lock1
    e0 = np.where(lock, np.where(lock0, 2 * hs, -2 * hd), hs - hd)
    e2 = np.where(lock, 0.0, hs + hd)
    e = np.stack([e0, th - np.pi / 2, e2], axis=-1)
    return np.where(e < -np.pi, e + 2 * np.pi, np.where(e > np.pi, e - 2 * np.pi, e))


def lock_distance(quat):
    """Distance of the unshifted middle angle from scipy's lock points (0 and pi), radians."""
    q = np.asarray(quat, np.float64)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    th = 2 * np.arctan2(np.hypot(x + w, y - z), np.hypot(w - x, z + y))
    return np.minimum(np.abs(th), np.abs(th - np.pi))


def _rot_noise(quat, noise_deg):
    """angles (degrees) + noise -> from_euler('zxy', degrees=True).as_rotvec(), float64."""
    e = np.degrees(euler_zxy(quat)) + np.asarray(noise_deg, np.float64)
    return Rotation.from_euler('zxy', e.reshape(-1, 3), degrees=True).as_rotvec().reshape(e.shape)


def canonical_params(params, joints, transf):
    """update_globalRT_for_smplx of one window (delta_T = pelvis - transl): canonical global_orient (rotvec), transl, and
    the unchanged betas and body_pose, float64."""
    p = {k: np.asarray(v, np.float64) for k, v in params.items()}
    j = np.asarray(joints, np.float64)
    rt, tv = transf[:3, :3], transf[:3, 3]
    delta = j[:, 0] - p['transl']
    out = dict(p)
    out['global_orient'] = Rotation.from_matrix(rt @ rotvec_to_matrix(p['global_orient'])).as_rotvec()
    out['transl'] = (p['transl'] + delta) @ rt.T + tv - delta
    return out


def noisy_params(cano, noise):
    """dataloader_amass.py:159-192 on one window's canonical parameters: noise dict of transl [T,3], betas [T,10],
    global_orient [T,3] and body_pose [T,21,3] (degrees for the rotations) -> noisy parameters (body_pose [T,63])."""
    T = cano['transl'].shape[0]
    go = Rotation.from_rotvec(cano['global_orient']).as_quat()
    bp = Rotation.from_rotvec(np.asarray(cano['body_pose']).reshape(-1, 3)).as_quat()
    return {'transl': cano['transl'] + noise['transl'], 'betas': cano['betas'] + noise['betas'],
            'global_orient': _rot_noise(go, noise['global_orient']),
            'body_pose': _rot_noise(bp, np.asarray(noise['body_pose']).reshape(-1, 3)).reshape(T, 63)}


def encode_noisy(params, joints, lengths, noise, model, clip_len=145, overlap=2):
    """The noisy windows: params / joints / lengths as ``encode``, noise a dict of window-major arrays (transl [W,T,3],
    betas [W,T,10], global_orient [W,T,3], body_pose [W,T,21,3]), model the body of kinematics_oracle.smplx_forward ->
    (noisy params dict of [W,T,.], noisy canonical joints [W,T,22,3], repr [W,T-1,294] of the noisy windows,
    un-normalised)."""
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    out_p, out_j, out_r = [], [], []
    for w, (r, s) in enumerate(window_table(lengths, clip_len, overlap)):
        rows = slice(off[r] + s, off[r] + s + clip_len)
        m = canonical_frame(joints[rows])
        cano = canonical_params({k: v[rows] for k, v in params.items()}, joints[rows], m)
        p = noisy_params(cano, {k: np.asarray(v[w], np.float64) for k, v in noise.items()})
        t = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in p.items()}
        j, _ = ko.smplx_forward(model, t['global_orient'], t['body_pose'], t['betas'], t['transl'], return_verts=False,
                                dtype=torch.float64)
        j = j[:, 0:22].numpy()
        out_p.append(p)
        out_j.append(j)
        out_r.append(encode_window(j, p['global_orient'], p['transl'], p['betas'], p['body_pose'], np.eye(4)))
    stack = lambda k, width: np.asarray([p[k] for p in out_p]).reshape(-1, clip_len, width)
    return ({k: stack(k, wd) for k, wd in (('global_orient', 3), ('transl', 3), ('betas', 10), ('body_pose', 63))},
            np.asarray(out_j).reshape(-1, clip_len, 22, 3), np.asarray(out_r).reshape(-1, clip_len - 1, 294))
