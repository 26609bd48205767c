"""Evaluation loss dictionaries returned by ``eval_losses(compute_loss=True)`` -- the default the single-model drivers use
(reference test_posenet.py:178, test_trajnet.py:154).  Restates ``compute_losses_with_smpl`` of model/posenet.py:99-193 and
model/trajnet.py:278-400 key for key.

This runs ONCE after a sampling loop, on [B, T, .] tensors of a few hundred KB: it is not part of the denoising hot path
(SURVEY.md 8a), so the reductions are plain device-side torch ops; every joint / rotation recovery inside goes through the
CUDA entry points (rohm_joints_from_traj, rohm_body_from_repr, rohm_rot6d_to_aa).
"""
import torch

from . import glue
from .motion_representation import recover_from_repr_smpl, split_repr


def _mse(a, b):
    return (a - b) ** 2  # nn.MSELoss(reduction='none')


def _skating(joints, contact_gt, foot_idx, fps, thres):
    vel = (joints[:, 1:, foot_idx] - joints[:, 0:-1, foot_idx]) * fps
    vel = torch.norm(vel, dim=-1)
    mask = (vel - thres).gt(0) * contact_gt[:, 0:-1]
    return (vel * mask).sum() / mask.sum()


def posenet_losses(model, batch, model_output, smplx_model=None, epoch=0):
    """model/posenet.py:99-193.  model_output, batch['motion_repr_clean']: [bs, 294, 1, T]."""
    dev = model_output.device
    mean, std = glue.stats_on(model.dataset, dev)
    body = smplx_model if smplx_model is not None else model.smplx_model
    clean_n = batch['motion_repr_clean'].to(dev)
    d = {}
    rec_all = _mse(clean_n, model_output)[:, :, 0].permute(0, 2, 1)
    d['loss_repr_full_body'] = rec_all[:, :, model.traj_feat_dim:-4].mean()

    full_clean = clean_n[:, :, 0].permute(0, 2, 1) * std + mean
    full_rec = model_output[:, :, 0].permute(0, 2, 1) * std + mean
    rd_clean, rd_rec = split_repr(full_clean), split_repr(full_rec)
    j_clean = recover_from_repr_smpl(rd_clean, 'joint_abs_traj', body)
    j_abs = recover_from_repr_smpl(rd_rec, 'joint_abs_traj', body)
    j_rel = recover_from_repr_smpl(rd_rec, 'joint_rel_traj', body)
    j_smpl = recover_from_repr_smpl(rd_rec, 'smplx_params', body)
    for name, j in (('abs_traj', j_abs), ('rel_traj', j_rel), ('smpl', j_smpl)):
        d[f'loss_joint_pos_global_from_{name}'] = _mse(j, j_clean).mean()
    v_clean = j_clean[:, 1:] - j_clean[:, 0:-1]
    vels = {}
    for name, j in (('abs_traj', j_abs), ('rel_traj', j_rel), ('smpl', j_smpl)):
        vels[name] = j[:, 1:] - j[:, 0:-1]
        d[f'loss_joint_vel_global_from_{name}'] = _mse(vels[name], v_clean).mean()
    for name in ('abs_traj', 'rel_traj', 'smpl'):
        acc = vels[name][:, 1:] - vels[name][:, 0:-1]
        d[f'loss_joint_smooth_from_{name}'] = torch.mean(acc ** 2)
    d['loss_repr_foot_contact_mse'] = _mse(clean_n[:, -4:, :, :], model_output[:, -4:, :, :]).mean()
    contact_gt = full_clean[:, :, -4:]
    for name, j in (('abs_traj', j_abs), ('rel_traj', j_rel), ('smpl', j_smpl)):
        d[f'loss_foot_skating_from_{name}'] = _skating(j, contact_gt, model.foot_joint_index_list, model.fps,
                                                       model.foot_skating_vel_thres)
    w_skate = model.weight_loss_foot_skating if epoch >= model.start_skating_loss_epoch else 0.0
    tri = lambda stem: d[f'{stem}_from_abs_traj'] + d[f'{stem}_from_rel_traj'] + d[f'{stem}_from_smpl']
    d["loss"] = (model.weight_loss_rec_repr_full_body * d['loss_repr_full_body'] +
                 model.weight_loss_repr_foot_contact_mse * d['loss_repr_foot_contact_mse'] +
                 model.weight_loss_joint_pos_global * tri('loss_joint_pos_global') +
                 model.weight_loss_joint_vel_global * tri('loss_joint_vel_global') +
                 model.weight_loss_joint_smooth * tri('loss_joint_smooth') +
                 w_skate * tri('loss_foot_skating'))
    return d


def _angular_velocity(R, dRdt):
    """utils/other_utils.py:243-261."""
    w = torch.matmul(dRdt, R.transpose(-1, -2))
    return torch.stack([(-w[..., 1, 2] + w[..., 2, 1]) / 2.0, (w[..., 0, 2] - w[..., 2, 0]) / 2.0,
                        (-w[..., 0, 1] + w[..., 1, 0]) / 2.0], dim=-1)


def trajnet_losses(model, batch, model_output, smplx_model=None):
    """model/trajnet.py:278-400.  model_output: [bs, T, traj_feat_dim]; batch['motion_repr_clean']: [bs, T, 294]."""
    dev = model_output.device
    mean, std = glue.stats_on(model.dataset, dev)
    body = smplx_model
    clean_n = batch['motion_repr_clean'].to(dev)
    d = {}
    if not model.repr_abs_only:
        full_rec = torch.cat([model_output, clean_n[:, :, model.traj_feat_dim:]], dim=-1)
    else:
        full_rec = clean_n.clone()
        full_rec[..., 0] = model_output[..., 0]
        full_rec[..., 2:4] = model_output[..., 1:3]
        full_rec[..., 6] = model_output[..., 3]
        full_rec[..., 7:13] = model_output[..., 4:10]
        full_rec[..., 16:19] = model_output[..., 10:13]
    la = _mse(clean_n, full_rec)
    d['loss_repr_traj_root_rot_angle'] = la[:, :, 0].mean()
    d['loss_repr_traj_root_l_pos'] = la[:, :, 2:4].mean()
    d['loss_repr_traj_root_height'] = la[:, :, 6].mean()
    d['loss_repr_traj_smplx_rot_6d'] = la[:, :, 7:13].mean()
    d['loss_repr_traj_smplx_trans'] = la[:, :, 16:19].mean()
    if not model.repr_abs_only:
        d['loss_repr_traj_root_rot_angle_vel'] = la[:, :, 1].mean()
        d['loss_repr_traj_root_l_vel'] = la[:, :, 4:6].mean()
        d['loss_repr_traj_smplx_rot_vel'] = la[:, :, 13:16].mean()
        d['loss_repr_traj_smplx_trans_vel'] = la[:, :, 19:22].mean()
        d['loss_repr_traj'] = la[..., 0:model.traj_feat_dim].mean()
    else:
        d['loss_repr_traj'] = torch.cat([la[..., 0:1], la[..., 2:4], la[..., 6:7], la[..., 7:13], la[..., 16:19]],
                                        dim=-1).mean()
    full_clean = clean_n * std + mean
    full_rec = full_rec * std + mean
    rd_clean, rd_rec = split_repr(full_clean), split_repr(full_rec)
    root_clean = recover_from_repr_smpl(rd_clean, 'joint_abs_traj', body)[:, :, 0]
    roots = {'abs_traj': recover_from_repr_smpl(rd_rec, 'joint_abs_traj', body)[:, :, 0],
             'rel_traj': recover_from_repr_smpl(rd_rec, 'joint_rel_traj', body)[:, :, 0],
             'smpl': recover_from_repr_smpl(rd_rec, 'smplx_params', body)[:, :, 0]}
    v_clean = root_clean[:, 1:] - root_clean[:, 0:-1]
    for name, r in roots.items():
        d[f'loss_root_pos_global_from_{name}'] = _mse(r, root_clean).mean()
    vels = {}
    for name, r in roots.items():
        vels[name] = r[:, 1:] - r[:, 0:-1]
        d[f'loss_root_vel_global_from_{name}'] = _mse(vels[name], v_clean).mean()
    bs = root_clean.shape[0]
    _, go_mat = glue.rot6d_to_angle_axis(rd_rec['smplx_rot_6d'].reshape(-1, 6), want_rotmat=True)
    go_mat = go_mat.reshape(bs, -1, 3, 3)
    rot_vel = _angular_velocity(go_mat[:, 0:-1], go_mat[:, 1:] - go_mat[:, 0:-1])
    d['loss_root_smplx_rot_vel'] = _mse(rot_vel, rd_clean['smplx_rot_vel'][:, 0:-1]).mean()
    tv = rd_rec['smplx_trans'][:, 1:] - rd_rec['smplx_trans'][:, 0:-1]
    d['loss_root_smplx_transl_vel'] = _mse(tv, rd_clean['smplx_trans_vel'][:, 0:-1]).mean()
    for name in roots:
        acc = vels[name][:, 1:] - vels[name][:, 0:-1]
        d[f'loss_root_smooth_from_{name}'] = torch.mean(acc ** 2)
    cv_clean = torch.cos(rd_clean['root_rot_angle'][:, 1:] * 2) - torch.cos(rd_clean['root_rot_angle'][:, 0:-1] * 2)
    cv_rec = torch.cos(rd_rec['root_rot_angle'][:, 1:] * 2) - torch.cos(rd_rec['root_rot_angle'][:, 0:-1] * 2)
    d['loss_root_rot_cos_vel_from_abs_traj'] = _mse(cv_clean, cv_rec).mean()
    d['loss_root_rot_cos_smooth_from_abs_traj'] = torch.mean((cv_rec[:, 1:] - cv_rec[:, 0:-1]) ** 2)
    if model.repr_abs_only:
        zero = torch.tensor(0.0, device=dev)
        d['loss_root_pos_global_from_rel_traj'] = zero
        d['loss_root_vel_global_from_rel_traj'] = zero.clone()
        d['loss_root_smooth_from_rel_traj'] = zero.clone()
    tri = lambda stem: d[f'{stem}_from_abs_traj'] + d[f'{stem}_from_rel_traj'] + d[f'{stem}_from_smpl']
    d["loss"] = (model.weight_loss_root_rec_repr * d['loss_repr_traj'] +
                 model.weight_loss_root_pos_global * tri('loss_root_pos_global') +
                 model.weight_loss_root_vel_global * tri('loss_root_vel_global') +
                 model.weight_loss_root_rot_vel_from_abs_traj * d['loss_root_rot_cos_vel_from_abs_traj'] +
                 model.weight_loss_root_smplx_transl_vel * d['loss_root_smplx_transl_vel'] +
                 model.weight_loss_root_smplx_rot_vel * d['loss_root_smplx_rot_vel'] +
                 model.weight_loss_root_smooth * tri('loss_root_smooth') +
                 model.weight_loss_root_rot_cos_smooth_from_abs_traj * d['loss_root_rot_cos_smooth_from_abs_traj'])
    return d
