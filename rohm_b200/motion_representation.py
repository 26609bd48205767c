"""``recover_from_repr_smpl`` on the CUDA kernels: drop-in for the one function of
data_loaders/motion_representation.py (:332-398) that the inference drivers call between and after the sampling loops
(test_amass_full.py:292, 406, 416-418, 428; test_posenet.py / test_trajnet.py through compute_losses_with_smpl).

Same signature, same dict-of-tensors input (de-normalised [..., T, d] slices of the 294-channel row, keyed by REPR_LIST),
same outputs; the arithmetic runs in librohm_b200.so (rohm_joints_from_traj, rohm_body_from_repr).
"""
import torch

from . import glue
from ._lib import RohmB200Error

# utils/other_utils.py:17-37
REPR_LIST = ['root_rot_angle', 'root_rot_angle_vel', 'root_l_pos', 'root_l_vel', 'root_height',
             'smplx_rot_6d', 'smplx_rot_vel', 'smplx_trans', 'smplx_trans_vel',
             'local_positions', 'local_vel',
             'smplx_body_pose_6d', 'smplx_betas',
             'foot_contact']
REPR_DIM_DICT = {'root_rot_angle': 1, 'root_rot_angle_vel': 1, 'root_l_pos': 2, 'root_l_vel': 2, 'root_height': 1,
                 'smplx_rot_6d': 6, 'smplx_rot_vel': 3, 'smplx_trans': 3, 'smplx_trans_vel': 3,
                 'local_positions': 22 * 3, 'local_vel': 22 * 3,
                 'smplx_body_pose_6d': 21 * 6, 'smplx_betas': 10,
                 'foot_contact': 4}


def split_repr(full_repr):
    """[..., 294] -> dict keyed by REPR_LIST (views)."""
    out, cur = {}, 0
    for name in REPR_LIST:
        out[name] = full_repr[..., cur:cur + REPR_DIM_DICT[name]]
        cur += REPR_DIM_DICT[name]
    return out


def _row_from_dict(data_dict):
    """Re-assembles the [B, T, 294] row from the dict (missing entries, which the chosen mode does not read, are zero)."""
    ref = next(iter(data_dict.values()))
    lead = tuple(ref.shape[:-1])
    if len(lead) == 1:  # [T, d] -> one clip
        lead = (1,) + lead
    parts = []
    for name in REPR_LIST:
        v = data_dict.get(name)
        if v is None:
            v = torch.zeros(lead + (REPR_DIM_DICT[name],), device=ref.device, dtype=torch.float32)
        parts.append(v.reshape(lead + (REPR_DIM_DICT[name],)).to(torch.float32))
    row = torch.cat(parts, dim=-1)
    return row.reshape(-1, lead[-1], row.shape[-1]).contiguous(), lead


_unit_stats = {}


def _unit(device):
    key = str(device)
    if key not in _unit_stats:
        _unit_stats[key] = (torch.zeros(294, device=device), torch.ones(294, device=device))
    return _unit_stats[key]


def recover_from_repr_smpl(data_dict, recover_mode='joint_abs_traj', smplx_model=None, return_verts=False,
                           return_full_joints=False, lengths=None):
    """joints [bs, T, 22, 3] (and vertices [bs, T, V, 3] with return_verts) from the motion representation:
    'joint_abs_traj' / 'joint_rel_traj' (joint-based, quaternion path) or 'smplx_params' (6-D -> axis-angle -> SMPL-X).
    lengths (int32 device [bs], see glue.device_lengths): clip b has lengths[b] <= T frames; only those are computed and
    the results are packed: joints [sum of lengths, 22, 3], vertices [sum of lengths, V, 3]."""
    if recover_mode not in ('joint_abs_traj', 'joint_rel_traj', 'smplx_params'):
        raise RohmB200Error(f"recover_from_repr_smpl: recover_mode {recover_mode!r} is not one of 'joint_abs_traj', "
                            "'joint_rel_traj', 'smplx_params'")
    row, lead = _row_from_dict(data_dict)
    if row.device.type != "cuda":
        raise RohmB200Error("recover_from_repr_smpl: tensors must live on a CUDA device (no CPU path)")
    mean, std = _unit(row.device)
    B, T = row.shape[0], row.shape[1]
    if lengths is not None and len(lead) != 2:
        raise RohmB200Error("recover_from_repr_smpl: lengths go with [bs, T, d] entries")
    if recover_mode != 'smplx_params':
        j = glue.joints_from_traj_repr(row, mean, std, relative=(recover_mode == 'joint_rel_traj'), channels_last=True,
                                       lengths=lengths)
        return j if lengths is not None else j.reshape(lead + (22, 3))
    if return_full_joints:
        raise RohmB200Error("recover_from_repr_smpl(return_full_joints=True): the 72 landmark joints beyond the 55 "
                            "kinematic ones are not evaluated by the CUDA body kernels (no inference driver asks for them)")
    if smplx_model is None:
        raise RohmB200Error("recover_from_repr_smpl('smplx_params') needs smplx_model")
    from .body_model import kernels_for
    if lengths is not None:
        _, total = glue.clip_layout(lengths, B, T, "recover_from_repr_smpl")
        k = kernels_for(smplx_model, row.device, total, with_vertices=bool(return_verts))
        return k.from_repr(row, mean, std, want_vertices=bool(return_verts), num_joints=22, channels_last=True,
                           lengths=lengths)
    k = kernels_for(smplx_model, row.device, B * T, with_vertices=bool(return_verts))
    res = k.from_repr(row, mean, std, want_vertices=bool(return_verts), num_joints=22, channels_last=True)
    if return_verts:
        joints, verts = res
        return joints.reshape(lead + (22, 3)), verts.reshape(lead + (verts.shape[-2], 3))
    return res.reshape(lead + (22, 3))
