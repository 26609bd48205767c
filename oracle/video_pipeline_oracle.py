"""Oracle (test infrastructure only): the video driver's multi-round TrajNet -> PoseNet inference of
test_prox_egobody.py:214-324 on the CPU, assembled from the other oracle modules (denoisers, samplers, kinematics, glue,
the 2-D projection guidance).  Flag set of the shipped PROX / EgoBody configs: sample_iter 2, iter2_cond_noisy_traj and
iter2_cond_noisy_pose False, early_stop, repr_abs_only, cond_fn_with_grad, grad_type='prox'.  Pinned by
tests/golden/video_pipeline.npz (the unmodified reference run through the same call sequence on windows of its own video
loader, tools/gen_golden.py:gen_video_pipeline).
"""
import torch

from . import diffusion_oracle as do
from . import glue_oracle as go
from . import kinematics_oracle as ko
from . import posenet_oracle, trajnet_oracle


def posenet_prox_step(tables, tmap, i, x_t, cond, sd_pose, mean_p, std_p, body_model, noise, camera, guide_last=100):
    """One p_sample_with_grad step with grad_type='prox' (gaussian_diffusion_posenet.py:436-480): the 2-D projection
    guidance at 3e5, then the skating guidance at 1e5, on steps <= 100 -> (x_{t-1}, x0).  camera: dict of transf_matrix,
    cam_R, cam_t, focal_length, camera_center, keypoints_2d (glue_oracle.guide_projection's inputs)."""
    B = x_t.shape[0]
    with torch.no_grad():
        x0 = posenet_oracle.posenet_forward(sd_pose, x_t, cond, torch.full((B,), tmap[i], dtype=torch.long))
    g = None
    if i <= guide_last:
        gp, _ = go.guide_projection(x0, mean_p, std_p, body_model, camera['transf_matrix'], camera['cam_R'], camera['cam_t'],
                                    camera['focal_length'], camera['camera_center'], camera['keypoints_2d'])
        g = [(3e5, gp)]
        gs = ko.guide_skating(x0, mean_p, std_p, body_model)
        if gs.dim() != 0:
            g.append((1e5, gs))
    return do.p_sample_step(tables, i, x_t, x0, noise, g), x0


def video_pose_cond(src_cl, traj_full, vis_mask=None):
    """test_prox_egobody.py:290-313 on a channels-last source [B,Tp,294] -> [B,294,1,Tp]: channels [0,22) <- traj_full;
    with vis_mask ([B,>=Tp,294], the rounds < mask_iter_num) the row is multiplied by vis_mask[:, 0:Tp] and the contact
    channels are zeroed."""
    cond = src_cl.clone()
    cond[:, :, 0:22] = traj_full
    if vis_mask is not None:
        cond = cond * vis_mask[:, 0:cond.shape[1]]
        cond[:, :, -4:] = 0.
    return torch.permute(cond, (0, 2, 1)).unsqueeze(-2).contiguous()


def run_video_rounds(sd_pose, sd_traj, sd_ctrl, ds_pose, ds_traj, body_model, pose, traj, pose_steps, traj_steps, rounds,
                     noise_pose, noise_traj, camera, pose_respacing='', teacher=None, teacher_steps=()):
    """The video driver's rounds (test_prox_egobody.py:214-324) with the shipped flags (iter2_cond_noisy_traj and
    iter2_cond_noisy_pose False, early_stop, grad_type='prox'): the trajectory composite builds on traj['motion_repr_noisy']
    (round 0's composite replaces it), TrajNet's condition becomes the previous TrajNet output, and the PoseNet condition is
    the visibility-masked noisy rows in round 0 and the previous PoseNet output afterwards.  pose / traj: the loader's
    batches (CPU tensors: pose motion_repr_noisy [B,144,294] and mask_vec_vis [B,145,294]; traj motion_repr_noisy and
    cond); camera: see posenet_prox_step.  Returns one dict per round as ``run_rounds``, with the same teacher mechanism
    (teacher keys r{k}_val_pose, r{k}_xt{i})."""
    tp, mp_ = do.create_diffusion('cosine', pose_steps, pose_respacing)
    tt, mt_ = do.create_diffusion('cosine', traj_steps, '')
    mean_p, std_p = torch.from_numpy(ds_pose.Mean), torch.from_numpy(ds_pose.Std)
    B, T = traj['cond'].shape[0], traj['cond'].shape[1]
    base, cond_traj = traj['motion_repr_noisy'], traj['cond']
    noisy_p = pose['motion_repr_noisy'][:, 0:-1]
    n_pose = len(tp['betas'])
    out = []
    val_pose = None
    for it in range(rounds):
        x_T = noise_traj.randn(B, T, 13)
        if it == 0:
            fn = lambda x, t, c=cond_traj: trajnet_oracle.trajnet_forward(sd_traj, x, c, torch.full((B,), t, dtype=torch.long))
        else:
            cc = go.pose_to_control_cond(val_pose, T, 272)
            fn = lambda x, t, c=cond_traj: trajnet_oracle.trajnet_forward(sd_ctrl, x, c, torch.full((B,), t, dtype=torch.long),
                                                                          control_cond=cc)
        with torch.no_grad():
            val_traj, _ = do.p_sample_loop(tt, mt_, fn, x_T, lambda i: noise_traj.randn_like(x_T))
        comp, traj_full = go.traj_to_full_repr(val_traj, base, ds_traj.Mean, ds_traj.Std, ds_pose.Mean, ds_pose.Std,
                                               body_model)
        if it == 0:
            base = comp
        if it < rounds - 1:
            cond_traj = val_traj
        src = noisy_p if it == 0 else val_pose[:, :, 0].permute(0, 2, 1)
        cond = video_pose_cond(src, traj_full, pose['mask_vec_vis'] if it == 0 else None)
        x = noise_pose.randn(B, 294, 1, T - 1)
        noises = {i: noise_pose.randn_like(x) for i in range(n_pose - 1, -1, -1)}  # the reference draws one per step, in order
        for i in range(n_pose - 1, -1, -1):
            x, x0 = posenet_prox_step(tp, mp_, i, x, cond, sd_pose, mean_p, std_p, body_model, noises[i], camera)
        res = {'val_traj': val_traj, 'traj_full': traj_full, 'cond': cond, 'val_pose': x0.detach()}  # early_stop: pred_xstart
        val_pose = res['val_pose']
        if teacher is not None:
            res['tf'] = {}
            for i in teacher_steps:
                xt = torch.from_numpy(teacher[f"r{it}_xt{i}"])
                x_next, x0_i = posenet_prox_step(tp, mp_, i, xt, cond, sd_pose, mean_p, std_p, body_model, noises[i], camera)
                res['tf'][i] = (x0_i if i == 0 else x_next).detach()
            val_pose = torch.from_numpy(teacher[f"r{it}_val_pose"])
        out.append(res)
    return out
