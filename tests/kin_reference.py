"""Float64 references of the device helpers in rohm_b200/csrc/kin.cuh and repr.cuh, and the edge inputs they are tested at
(not collected by pytest).

Each reference is the reference code's formula evaluated in float64 on the exact float32 values a kernel receives:
  rot6d_to_mat / rot6d_vjp   oracle.kinematics_oracle.rot6d_to_rotmat (and torch.autograd through it)
  mat_to_aa                  oracle.kinematics_oracle.rotmat_to_aa (kornia's quaternion route, eps 1e-6)
  rodrigues                  smplx batch_rodrigues, restated here because the reference adds its 1e-8 to a float32
                             tensor: the offset is float32(1e-8), which makes r = -float32(1e-8) in every component
                             an exact zero vector (NaN), where kinematics_oracle.batch_rodrigues in float64 adds the
                             double 1e-8 and stays finite
  rotvec_to_mat              oracle.glue_oracle.rotvec_to_matrix (scipy's rotvec -> quaternion -> matrix)
  heading_quat / qrot_z /    the qbetween, qmul, qinv, qrot and estimate_angular_velocity_np lines of get_repr_smplx
  traj_channels              (glue_oracle.traj_repr_from_joints), restated in float64; glue_oracle's copies are float32
                             because the reference's are.
"""
import math

import numpy as np
import torch

from oracle import glue_oracle as go
from oracle import kinematics_oracle as ko

U = 2.0 ** -24  # float32 unit roundoff
EPS_RODRIGUES = float(np.float32(1e-8))


def f32(x):
    """float64 array -> the float32 values a kernel receives, as float64 (exact)."""
    return torch.as_tensor(np.asarray(x, dtype=np.float64)).float().double()


# ------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------
def rot6d_to_mat(x):
    """[n, 6] -> (R [n, 3, 3], (l1, l2, s) [n, 3]) in float64, the clamped norms rot6d_to_mat reports."""
    x = x.double()
    R = ko.rot6d_to_rotmat(x)
    a1, a2 = x[:, 0::2], x[:, 1::2]
    l1 = a1.norm(dim=1).clamp_min(1e-12)
    s = ((a1 / l1[:, None]) * a2).sum(1)
    l2 = (a2 - s[:, None] * a1 / l1[:, None]).norm(dim=1).clamp_min(1e-12)
    return R, torch.stack([l1, l2, s], dim=1)


def rot6d_vjp(x, G):
    """d<G, rot6d_to_rotmat(x)>/dx in float64 through torch.autograd."""
    x = x.double().clone().requires_grad_()
    R = ko.rot6d_to_rotmat(x)
    return torch.autograd.grad((R * G.double()).sum(), x)[0]


def round_trip(x):
    """The reference's 6-D -> R -> axis-angle -> R in float64 (differentiable)."""
    return rodrigues(ko.rotmat_to_aa(ko.rot6d_to_rotmat(x)))


def round_trip_vjp(x, G):
    """d<G, round_trip(x)>/dx in float64 through torch.autograd (the gradient the reference's guidance takes)."""
    x = x.double().clone().requires_grad_()
    return torch.autograd.grad((round_trip(x) * G.double()).sum(), x)[0]


def mat_to_aa(R):
    return ko.rotmat_to_aa(R.double())


def rodrigues(r, eps=EPS_RODRIGUES):
    """smplx batch_rodrigues with the float32 offset (see the module docstring)."""
    n = r.shape[0]
    angle = torch.norm(r + eps, dim=1, keepdim=True)
    d = r / angle
    cos, sin = torch.cos(angle)[:, None], torch.sin(angle)[:, None]
    rx, ry, rz = torch.split(d, 1, dim=1)
    zeros = torch.zeros((n, 1), dtype=r.dtype)
    K = torch.cat([zeros, -rz, ry, rz, zeros, -rx, -ry, rx, zeros], dim=1).view(n, 3, 3)
    return torch.eye(3, dtype=r.dtype)[None] + sin * K + (1 - cos) * torch.bmm(K, K)


def rotvec_to_mat(r):
    return torch.from_numpy(go.rotvec_to_matrix(np.asarray(r, dtype=np.float64)))


def _qmul(q, r):
    w = r[:, 0] * q[:, 0] - r[:, 1] * q[:, 1] - r[:, 2] * q[:, 2] - r[:, 3] * q[:, 3]
    x = r[:, 0] * q[:, 1] + r[:, 1] * q[:, 0] - r[:, 2] * q[:, 3] + r[:, 3] * q[:, 2]
    y = r[:, 0] * q[:, 2] + r[:, 1] * q[:, 3] + r[:, 2] * q[:, 0] - r[:, 3] * q[:, 1]
    z = r[:, 0] * q[:, 3] - r[:, 1] * q[:, 2] + r[:, 2] * q[:, 1] + r[:, 3] * q[:, 0]
    return np.stack([w, x, y, z], axis=1)


def _qrot(q, v):
    qv = q[:, 1:]
    uv = np.cross(qv, v)
    uuv = np.cross(qv, uv)
    return v + 2 * (q[:, :1] * uv + uuv)


def heading_quat(j1, j2, j17, j16):
    """qbetween(forward, +y) of get_repr_smplx in float64: joints [n, 3] each -> (q0, q1, q3) [n, 3] (NaN where the
    reference's is)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        across = (j1 - j2) + (j17 - j16)
        across = across / np.sqrt((across ** 2).sum(axis=-1))[:, None]
        forward = np.cross(np.array([[0.0, 0.0, 1.0]]), across, axis=-1)
        forward = forward / np.sqrt((forward ** 2).sum(axis=-1))[:, None]
        target = np.array([[0.0, 1.0, 0.0]]).repeat(len(forward), axis=0)
        v = np.cross(forward, target, axis=-1)
        w = np.sqrt((forward ** 2).sum(-1, keepdims=True) * (target ** 2).sum(-1, keepdims=True)) + \
            (forward * target).sum(-1, keepdims=True)
        q = np.concatenate([w, v], axis=-1)
        q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    return q[:, [0, 1, 3]]


def qrot_z(wz, v):
    q = np.zeros((len(wz), 4))
    q[:, 0], q[:, 3] = wz[:, 0], wz[:, 1]
    return _qrot(q, v)


def traj_channels(q, roots, rots, trs):
    """Channels [0, 22) of frame 0 of a two-frame pair: q [n, 4] = (w0, z0, w1, z1) repaired heading quaternions, roots /
    trs [n, 2, 3], rots [n, 2, 3, 3] -> [n, 22] float64."""
    n = len(q)
    q0, q1 = np.zeros((n, 4)), np.zeros((n, 4))
    q0[:, 0], q0[:, 3], q1[:, 0], q1[:, 3] = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    q_vel = _qmul(q1, q0 * np.array([1.0, -1.0, -1.0, -1.0]))
    ang = np.arctan2(q0[:, 3:4], q0[:, 0:1])
    ang_vel = np.arctan2(q_vel[:, 3:4], q_vel[:, 0:1])
    root_vel = _qrot(q1, roots[:, 1] - roots[:, 0])
    R0, R1 = rots[:, 0], rots[:, 1]
    w = np.matmul(R1 - R0, np.transpose(R0, (0, 2, 1)))
    rot_vel = np.stack([(-w[:, 1, 2] + w[:, 2, 1]) / 2.0, (w[:, 0, 2] - w[:, 2, 0]) / 2.0,
                        (-w[:, 0, 1] + w[:, 1, 0]) / 2.0], axis=-1)
    return np.concatenate([ang, ang_vel, roots[:, 0, 0:2], root_vel[:, 0:2], roots[:, 0, 2:3], R0[:, :, :2].reshape(n, 6),
                           rot_vel, trs[:, 0], trs[:, 1] - trs[:, 0]], axis=-1)


# ------------------------------------------------------------------------------------------------------------
# edge inputs
# ------------------------------------------------------------------------------------------------------------
def unit(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def axis_angle_mat(axes, angles):
    """Exact float64 rotations about unit axes [n, 3] by angles [n] (Rodrigues' formula)."""
    axes, angles = unit(axes), np.asarray(angles, dtype=np.float64)
    K = np.zeros((len(axes), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -axes[:, 2], axes[:, 1], -axes[:, 0]
    K[:, 1, 0], K[:, 2, 0], K[:, 2, 1] = axes[:, 2], -axes[:, 1], axes[:, 0]
    s, c = np.sin(angles)[:, None, None], np.cos(angles)[:, None, None]
    return np.eye(3)[None] + s * K + (1 - c) * (K @ K)


def rot6d_of(R):
    """R [n, 3, 3] -> the 6-D channels (row-major 3 x 2: a1 = column 0, a2 = column 1)."""
    return np.asarray(R)[:, :, :2].reshape(-1, 6)


def random_axes(n, rng):
    return unit(rng.standard_normal((n, 3)))


def rotation_families(n, rng):
    """{name: float64 rotations [n, 3, 3]}: the rotation regimes where the reference's clamps or branches act."""
    ax = random_axes(n, rng)
    return {
        "identity": np.repeat(np.eye(3)[None], n, axis=0),
        "1e-3 rad": axis_angle_mat(ax, np.full(n, 1e-3)),
        "2pi/3": axis_angle_mat(ax, np.full(n, 2 * math.pi / 3)),
        "pi - 1e-4": axis_angle_mat(ax, np.full(n, math.pi - 1e-4)),
    }


def nonorthonormal_families(n, rng):
    """{name: (float64 6-D [n, 6])}: 6-D inputs like a denoiser's pred_xstart, built from random rotations."""
    R = axis_angle_mat(random_axes(n, rng), rng.uniform(0.1, 3.0, n))
    a1, a2 = R[:, :, 0], R[:, :, 1]
    out = {}
    x = np.empty((n, 6))
    x[:, 0::2], x[:, 1::2] = 0.3 * a1, 3.0 * a2
    out["columns x0.3, x3"] = x.copy()
    x[:, 0::2], x[:, 1::2] = 3.0 * a1, 0.3 * a2
    out["columns x3, x0.3"] = x.copy()
    c = rng.uniform(0.2, 0.9, n)[:, None]
    x[:, 0::2], x[:, 1::2] = a1, a2 + c * a1
    out["a2 along a1 0.2-0.9"] = x.copy()
    # near-collinear: a2 at angle 1/kappa from a1 (kappa = |a2| / l2 up to 1e3)
    kap = np.exp(rng.uniform(np.log(10.0), np.log(1e3), n))[:, None]
    x[:, 0::2], x[:, 1::2] = a1, np.cos(1 / kap) * a1 + np.sin(1 / kap) * a2
    out["near-collinear kappa<=1e3"] = x.copy()
    return out


def kappa(x):
    """Conditioning of the Gram-Schmidt columns of 6-D inputs x [n, 6] (float64): |a2| / l2."""
    x = np.asarray(x, dtype=np.float64)
    a1, a2 = x[:, 0::2], x[:, 1::2]
    b1 = unit(a1)
    u2 = a2 - (b1 * a2).sum(1, keepdims=True) * b1
    return np.linalg.norm(a2, axis=1) / np.linalg.norm(u2, axis=1)
