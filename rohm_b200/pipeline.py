"""The multi-round TrajNet -> PoseNet inference of the reference driver, device-resident.

``run_rounds`` replays test_amass_full.py:218-384 (one dataloader batch: optional trajectory infill mask, then
``sample_iter`` rounds of  TrajNet / TrajControl sampling -> inter-round glue -> PoseNet condition assembly with occlusion
masks -> guided PoseNet sampling)  with the same call sequence, flags, batch-dict side effects and CPU-generator draws as
the driver, but without its host round trips: the per-clip numpy / scipy loop of :268-311 is ``rohm_traj_glue``, the
condition assembly of :313-370 is ``rohm_build_pose_cond``, the TrajControl condition of :256-258 is
``rohm_pose_to_control_cond``.  ``reconstruct_outputs`` is the post-loop block :386-428 (joints / vertices of the clean,
reconstructed and noisy motions) and ``result_dict`` the driver's pickle payload (:446-458).

``run_video_rounds``, ``reconstruct_video_outputs`` and ``video_result_dicts`` do the same for the PROX / EgoBody driver
(test_prox_egobody.py:214-384) on the windows of ``windows.encode_video``, any number of recordings per call.

The reference loop cannot be replaced "unchanged" because it is inline driver code, not a function; INTEGRATION.md shows the
5-line edit that swaps lines 218-384 for a call to ``run_rounds``.
"""
from types import SimpleNamespace

import numpy as np
import torch

from . import glue
from ._lib import RohmB200Error
from .motion_representation import REPR_DIM_DICT, REPR_LIST, recover_from_repr_smpl, split_repr

DEFAULTS = dict(sample_iter=2, cond_fn_with_grad=True, early_stop=False, timestep_respacing_eval='', input_noise=True,
                iter2_cond_noisy_traj=True, iter2_cond_noisy_pose=True, infill_traj=False, traj_mask_ratio=0.1,
                mask_scheme='lower', repr_abs_only=True)


def make_args(**kw):
    d = dict(DEFAULTS)
    d.update(kw)
    return SimpleNamespace(**d)


def run_rounds(args, model_posenet, model_trajnet, model_trajnet_control, diffusion_posenet, diffusion_trajnet,
               diffusion_trajnet_control, pose_dataset, traj_dataset, smplx_model, test_batch_pose, test_batch_traj,
               grad_type='amass', on_round=None):
    """One batch through ``args.sample_iter`` rounds.  Batch dicts hold CUDA tensors laid out as DataloaderAMASS emits them
    (pose: motion_repr_clean / motion_repr_noisy [B,144,294]; traj: cond [B,144,13], control_cond, motion_repr_clean /
    motion_repr_noisy [B,144,294]) and are mutated exactly as the driver mutates them.  Returns
    (val_output_pose [B,294,1,143], val_output_traj [B,144,traj_dim], traj_noisy_full [B,144,22]).

    test_batch_traj['lengths'] (optional, integer [B], multiples of 16 with 16 <= lengths[b] <= T = the padded trajectory
    batch's frame count): recording b has lengths[b] trajectory frames and lengths[b] - 1 pose frames inside the padded
    tensors.  It is checked before the first sampling step, test_batch_pose['lengths'] is set to lengths - 1, and both
    networks and every glue step run on the clips' own frames.  Shapes stay padded.  Real frames depend on their own clip
    only; frames past a clip are exactly zero in the three returned tensors and in the batch entries this function writes
    (pose 'cond', traj 'control_cond' and 'motion_repr_noisy'); whatever the padded frames of the inputs hold (NaN, Inf)
    never reaches a real frame.  Without guidance (cond_fn_with_grad=False, or steps before it starts) clip b equals the
    clip run as a one-clip batch with lengths=[lengths[b]] on the same noise, bit for bit.  The skating guidance
    normalises its loss over the real frames of the WHOLE batch (as the reference does over a batch), so with guidance on
    a clip's result depends on its batch-mates -- unless model_posenet.guidance_normaliser = 'clip', which normalises each
    clip over its own frames, so that guided clips also equal their one-clip runs bit for bit.  Those one-clip runs go through
    the same TrajNet engines; with batch_invariant = True on model_trajnet and model_trajnet_control they may be at the clip's
    own length in fresh engines, and still give the same bits.  mask_scheme='full' draws one uniform per clip as without lengths and
    places the window inside the clip: start = floor(u * (lengths[b] - 2)), end = min(start + 30, lengths[b] - 1).
    Refused with lengths: grad_type='prox', and infill_traj when its window [65, 65 + int(traj_mask_ratio * 145)) does not
    lie inside every clip.

    test_batch_traj['generators'] (optional, B distinct CUDA torch.Generator objects, rohm_b200.noise_streams): recording
    b's noise comes from generators[b] in every TrajNet, TrajControl and PoseNet loop of every round;
    test_batch_pose['generators'] is set to the same list.  Without guidance a recording's result then depends on the
    recording and its generator only, whatever batch or position it has.  mask_scheme='full' still makes the driver's one
    CPU uniform draw per batch (from torch's global CPU generator) to place its windows."""
    dev = test_batch_traj['cond'].device
    tfd = traj_dataset.traj_feat_dim
    pose_feat_dim = traj_dataset.pose_feat_dim
    if test_batch_traj.get('generators') is not None:
        from .noise_streams import check_generators
        check_generators(test_batch_traj, test_batch_traj['cond'].shape[0], dev)
        test_batch_pose['generators'] = test_batch_traj['generators']
    mask_traj = start = end = None
    len_t = len_p = lens = None  # int32 device lengths in trajectory / pose frames, and the ints
    if test_batch_traj.get('lengths') is not None:
        if grad_type == 'prox':
            # these rounds replay the AMASS driver; the PROX/EgoBody driver's rounds are not implemented here
            raise RohmB200Error("run_rounds: grad_type='prox' with test_batch_traj['lengths'] is out of scope (the rounds "
                                "replay the AMASS driver)")
        lens = model_trajnet.clip_lengths(test_batch_traj, test_batch_traj['cond'].shape)
        model_trajnet_control.clip_lengths(test_batch_traj, test_batch_traj['cond'].shape)
        B_, T_ = test_batch_traj['cond'].shape[0], test_batch_traj['cond'].shape[1]
        pose_lengths = test_batch_traj['lengths'].to(dev) - 1
        model_posenet.clip_lengths({'lengths': pose_lengths}, (B_, 294, 1, T_ - 1), grad_type=grad_type)
        if args.infill_traj and min(lens) < 65 + int(args.traj_mask_ratio * 145):
            raise RohmB200Error(f"run_rounds: infill_traj masks frames [65, {65 + int(args.traj_mask_ratio * 145)}) of every "
                                f"clip, which does not lie inside a clip of {min(lens)} frames")
        test_batch_pose['lengths'] = pose_lengths
        len_t = glue.device_lengths(lens, dev)
        len_p = glue.device_lengths([v - 1 for v in lens], dev)
    if args.infill_traj:  # :218-229
        clip_len, batch_size = test_batch_traj['cond'].shape[1], test_batch_traj['cond'].shape[0]
        mask_traj = torch.ones(batch_size, clip_len, device=dev)
        mask_len = int(args.traj_mask_ratio * 145)
        start = torch.ones([batch_size]).long() * 65
        end = start + mask_len
        mask_traj[:, 65:65 + mask_len] = 0
        mask_traj = mask_traj.unsqueeze(-1).repeat(1, 1, tfd)
        test_batch_traj['cond'][:, :, 0:tfd] = test_batch_traj['cond'][:, :, 0:tfd] * mask_traj

    val_output_traj = val_output_pose = traj_noisy_full = None
    for iter_idx in range(args.sample_iter):
        if args.iter2_cond_noisy_traj and args.infill_traj and iter_idx > 0:  # :233-237
            traj_vis = test_batch_traj['cond'][:, :, 0:tfd] * mask_traj
            traj_occ = val_output_traj * (1 - mask_traj)
            test_batch_traj['cond'][:, :, 0:tfd] = traj_vis + traj_occ

        # ---------------------------------------------------------------- trajectory network (:239-266)
        shape = list(test_batch_traj['motion_repr_clean'][:, :, 0:tfd].shape)
        if iter_idx == 0:
            _, val_output_traj = diffusion_trajnet.eval_losses(
                model=model_trajnet, batch=test_batch_traj, shape=shape, progress=False, clip_denoised=False,
                timestep_respacing=args.timestep_respacing_eval, cond_fn_with_grad=args.cond_fn_with_grad,
                compute_loss=False, smplx_model=smplx_model)
            traj_noisy_full = test_batch_traj['motion_repr_noisy'][:, :, 0:22].detach().clone()
            if lens is not None:
                for b, n in enumerate(lens):
                    traj_noisy_full[b, n:] = 0
        else:
            test_batch_traj['control_cond'] = glue.pose_to_control_cond(val_output_pose, shape[1], pose_feat_dim,
                                                                        lengths=len_p)
            _, val_output_traj = diffusion_trajnet_control.eval_losses(
                model=model_trajnet_control, batch=test_batch_traj, shape=shape, progress=False, clip_denoised=False,
                timestep_respacing=args.timestep_respacing_eval, cond_fn_with_grad=args.cond_fn_with_grad,
                compute_loss=False, smplx_model=smplx_model)

        # ---------------------------------------------------------------- inter-round glue (:268-311)
        composite, traj_rec_full = glue.traj_to_full_repr(smplx_model, val_output_traj,
                                                          test_batch_traj['motion_repr_clean'], traj_dataset, pose_dataset,
                                                          lengths=len_t)
        if iter_idx == 0:
            test_batch_traj['motion_repr_noisy'] = composite
        if iter_idx < args.sample_iter - 1 and not args.iter2_cond_noisy_traj:
            test_batch_traj['cond'] = val_output_traj

        # ---------------------------------------------------------------- PoseNet condition (:313-370)
        if iter_idx == 0:
            test_batch_pose['motion_repr_noisy'] = test_batch_pose['motion_repr_noisy'][:, 0:-1]
            test_batch_pose['motion_repr_clean'] = test_batch_pose['motion_repr_clean'][:, 0:-1]
        if not args.input_noise:
            src = test_batch_pose['motion_repr_clean']  # [B,143,294] in round 0, [B,294,1,143] afterwards: same values
        elif args.iter2_cond_noisy_pose or iter_idx == 0:
            src = test_batch_pose['motion_repr_noisy']
        else:
            src = val_output_pose
        bs, clip_len = traj_rec_full.shape[0], traj_rec_full.shape[1]
        replace_traj = not (args.mask_scheme == 'lower' and not args.input_noise)
        chan_keep = lo = hi = None
        zero_contact = False
        mask_iter_num = args.sample_iter if args.iter2_cond_noisy_pose else 1
        if iter_idx < mask_iter_num:
            if args.mask_scheme in ('lower', 'upper'):
                chan_keep = glue.channel_keep_mask(args.mask_scheme, pose_dataset.traj_feat_dim)
                zero_contact = True
            elif args.mask_scheme == 'full':
                if not args.infill_traj and lens is not None:  # the same draw, the window inside each clip
                    n_p = torch.tensor(lens, dtype=torch.float32) - 1  # pose frames per clip
                    start = (torch.FloatTensor(bs).uniform_(0, 1) * (n_p - 1)).long()
                    end = torch.minimum(start + 30, n_p.long())
                elif not args.infill_traj:  # same CPU-generator draw as the driver (:362)
                    start = torch.FloatTensor(bs).uniform_(0, clip_len - 1).long()
                    end = start + 30
                    end[end > clip_len] = clip_len
                lo, hi = start, end
                zero_contact = True
        test_batch_pose['cond'] = glue.build_pose_cond(src, traj_rec_full if replace_traj else None, chan_keep, lo, hi,
                                                       zero_contact, frames=clip_len, lengths=len_p)
        if iter_idx == 0:
            test_batch_pose['motion_repr_clean'] = torch.permute(test_batch_pose['motion_repr_clean'],
                                                                 (0, 2, 1)).unsqueeze(-2)

        # ---------------------------------------------------------------- PoseNet sampling (:372-384)
        shape = list(test_batch_pose['motion_repr_clean'].shape)
        _, val_output_pose = diffusion_posenet.eval_losses(
            model=model_posenet, batch=test_batch_pose, shape=shape, progress=False, clip_denoised=False,
            timestep_respacing=args.timestep_respacing_eval, cond_fn_with_grad=args.cond_fn_with_grad,
            early_stop=args.early_stop, compute_loss=False, grad_type=grad_type, smplx_model=smplx_model)
        if on_round is not None:
            # observer hook (tests): may return a tensor that replaces this round's PoseNet output for the next round
            repl = on_round(iter_idx, val_output_traj, traj_rec_full, test_batch_pose['cond'], val_output_pose)
            if repl is not None:
                val_output_pose = repl
    return val_output_pose, val_output_traj, traj_noisy_full


def reconstruct_outputs(args, pose_dataset, smplx_model, test_batch_pose, val_output_pose, traj_noisy_full,
                        return_verts=True, lengths=None):
    """test_amass_full.py:386-428: de-normalise the clean / reconstructed / noisy motions and recover joints (and
    vertices) from them.  Everything stays on the device; returns a dict of tensors.

    lengths (default test_batch_pose.get('lengths'); integer [B], pose frames per clip): only the clips' own frames are
    computed.  Every per-frame entry of the dict is then a list of B tensors [lengths[b], ...], the joints and vertices
    views into one packed allocation ([sum of lengths, 22, 3] joints, the pitched [sum of lengths, V, 3] vertex buffer),
    and out['frame_offsets'] (int64 [B+1]) gives each clip's first packed row."""
    dev = val_output_pose.device
    mean, std = glue.stats_on(pose_dataset, dev)
    if lengths is None:
        lengths = test_batch_pose.get('lengths')
    lens = None
    if lengths is not None:
        lens = lengths if getattr(lengths, "_rohm_layout", None) is not None else \
            glue.device_lengths([int(v) for v in lengths.tolist()], dev)
        glue.clip_layout(lens, val_output_pose.shape[0], val_output_pose.shape[-1], "reconstruct_outputs")
    per_clip = (lambda t: t) if lens is None else (lambda t: None if t is None else glue.split_clips(t, lens))
    rows = (lambda t: t) if lens is None else (lambda t: [t[b, :n] for b, n in enumerate(lens._rohm_layout[1])])
    out = {}
    if lens is not None:
        out['frame_offsets'] = lens._rohm_layout[2].to(torch.int64)
    clean = test_batch_pose['motion_repr_clean'][:, :, 0].permute(0, 2, 1) * std + mean
    rec = val_output_pose[:, :, 0].permute(0, 2, 1) * std + mean
    out['motion_repr_clean'], out['motion_repr_rec'] = rows(clean), rows(rec)
    res = recover_from_repr_smpl(split_repr(clean), 'smplx_params', smplx_model, return_verts=return_verts, lengths=lens)
    res = res if return_verts else (res, None)
    out['rec_ric_data_clean'], out['smpl_verts_clean'] = per_clip(res[0]), per_clip(res[1])
    out['rec_ric_data_rec_from_abs_traj'] = per_clip(recover_from_repr_smpl(split_repr(rec), 'joint_abs_traj', smplx_model,
                                                                            lengths=lens))
    res = recover_from_repr_smpl(split_repr(rec), 'smplx_params', smplx_model, return_verts=return_verts, lengths=lens)
    res = res if return_verts else (res, None)
    out['rec_ric_data_rec_from_smpl'], out['smpl_verts_rec'] = per_clip(res[0]), per_clip(res[1])
    if args.input_noise:
        noisy = test_batch_pose['motion_repr_noisy'].clone()
        noisy[:, :, 0:22] = traj_noisy_full[:, 0:-1, :]
        noisy = noisy * std + mean
        out['motion_repr_noisy'] = rows(noisy)
        res = recover_from_repr_smpl(split_repr(noisy), 'smplx_params', smplx_model, return_verts=return_verts,
                                     lengths=lens)
        res = res if return_verts else (res, None)
        out['rec_ric_data_noisy'], out['smpl_verts_noisy'] = per_clip(res[0]), per_clip(res[1])
    return out


VIDEO_POSE_KEYS = ('mask_vec_vis', 'keypoints_2d', 'transf_matrix', 'focal_length', 'camera_center')


def run_video_rounds(args, model_posenet, model_trajnet, model_trajnet_control, diffusion_posenet, diffusion_trajnet,
                     diffusion_trajnet_control, pose_dataset, traj_dataset, smplx_model, test_batch_pose, test_batch_traj,
                     on_round=None):
    """test_prox_egobody.py:214-324: ``args.sample_iter`` rounds of TrajNet / TrajControl -> glue -> guided PoseNet
    (grad_type='prox') over the W video windows of ``windows.encode_video`` (any number of recordings), mutating the two
    batch dicts as the driver does.  Returns (val_output_pose [W,294,1,143], val_output_traj [W,144,traj_dim]).

    It differs from ``run_rounds`` (the AMASS driver) in three places: the trajectory composite is built on
    test_batch_traj['motion_repr_noisy'] (round 0 stores it back there, so round 1 builds on round 0's composite); the
    PoseNet condition is the noisy pose rows (round 0, and every round with iter2_cond_noisy_pose) or the previous PoseNet
    output, with channels [0,22) from the glue, multiplied by test_batch_pose['mask_vec_vis'][:, 0:-2] and with its contact
    channels zeroed in rounds < mask_iter_num (round 0 only unless iter2_cond_noisy_pose); and there is no occlusion scheme,
    infill mask, clean motion or input-noise flag.  Where the reference writes the trajectory block into the previous
    PoseNet output in place (round >= 1, iter2_cond_noisy_pose False), this builds a new tensor: nothing reads the
    aliased one afterwards, and an output already handed to ``on_round`` stays as it was.

    Flags read: sample_iter, iter2_cond_noisy_traj, iter2_cond_noisy_pose, early_stop, cond_fn_with_grad,
    timestep_respacing_eval.  test_batch_traj['generators'] is honoured as in ``run_rounds``; with per-window generators,
    model_posenet.guidance_normaliser = 'clip' and batch-invariant TrajNets, a window's rounds depend on that window only.
    Refused before any sampling step: test_batch_traj['lengths'] (video windows are whole), a missing pose-batch key the
    driver reads (VIDEO_POSE_KEYS) and pose / trajectory batches with different window counts."""
    if test_batch_traj.get('lengths') is not None:
        raise RohmB200Error("run_video_rounds: test_batch_traj['lengths'] is refused: video windows are whole clips")
    missing = [k for k in VIDEO_POSE_KEYS if test_batch_pose.get(k) is None]
    if missing:
        raise RohmB200Error(f"run_video_rounds: test_batch_pose lacks {missing} (the video driver reads them)")
    W = test_batch_traj['motion_repr_noisy'].shape[0]
    if test_batch_pose['motion_repr_noisy'].shape[0] != W:
        raise RohmB200Error(f"run_video_rounds: the trajectory batch holds {W} windows, the pose batch "
                            f"{test_batch_pose['motion_repr_noisy'].shape[0]}")
    dev = test_batch_traj['motion_repr_noisy'].device
    tfd, pose_feat_dim = traj_dataset.traj_feat_dim, traj_dataset.pose_feat_dim
    if test_batch_traj.get('generators') is not None:
        from .noise_streams import check_generators
        check_generators(test_batch_traj, W, dev)
        test_batch_pose['generators'] = test_batch_traj['generators']
    mask_iter_num = args.sample_iter if args.iter2_cond_noisy_pose else 1
    val_output_traj = val_output_pose = None
    for iter_idx in range(args.sample_iter):
        # ---------------------------------------------------------------- trajectory network (:216-242)
        shape = list(test_batch_traj['motion_repr_noisy'][:, :, 0:tfd].shape)
        if iter_idx == 0:
            _, val_output_traj = diffusion_trajnet.eval_losses(
                model=model_trajnet, batch=test_batch_traj, shape=shape, progress=False, clip_denoised=False,
                timestep_respacing=args.timestep_respacing_eval, cond_fn_with_grad=args.cond_fn_with_grad,
                compute_loss=False, smplx_model=smplx_model)
        else:
            test_batch_traj['control_cond'] = glue.pose_to_control_cond(val_output_pose, shape[1], pose_feat_dim)
            _, val_output_traj = diffusion_trajnet_control.eval_losses(
                model=model_trajnet_control, batch=test_batch_traj, shape=shape, progress=False, clip_denoised=False,
                timestep_respacing=args.timestep_respacing_eval, cond_fn_with_grad=args.cond_fn_with_grad,
                compute_loss=False, smplx_model=smplx_model)

        # ---------------------------------------------------------------- inter-round glue (:244-287)
        composite, traj_rec_full = glue.traj_to_full_repr(smplx_model, val_output_traj, test_batch_traj['motion_repr_noisy'],
                                                          traj_dataset, pose_dataset)
        if iter_idx == 0:
            test_batch_traj['motion_repr_noisy'] = composite
        if iter_idx < args.sample_iter - 1 and not args.iter2_cond_noisy_traj:
            test_batch_traj['cond'] = val_output_traj

        # ---------------------------------------------------------------- PoseNet condition (:290-313)
        if iter_idx == 0:
            test_batch_pose['motion_repr_noisy'] = test_batch_pose['motion_repr_noisy'][:, 0:-1]
        src = test_batch_pose['motion_repr_noisy'] if (args.iter2_cond_noisy_pose or iter_idx == 0) else val_output_pose
        clip_len = traj_rec_full.shape[1]
        if iter_idx < mask_iter_num:
            cond = glue.build_pose_cond(src, traj_rec_full, zero_contact=True, frames=clip_len,
                                        vis_mask=test_batch_pose['mask_vec_vis'])
        else:
            cond = glue.build_pose_cond(src, traj_rec_full, frames=clip_len)
        test_batch_pose['cond'] = cond
        if iter_idx == 0:
            test_batch_pose['motion_repr_noisy'] = torch.permute(test_batch_pose['motion_repr_noisy'],
                                                                 (0, 2, 1)).unsqueeze(-2)

        # ---------------------------------------------------------------- PoseNet sampling (:315-324)
        shape = list(test_batch_pose['motion_repr_noisy'].shape)
        _, val_output_pose = diffusion_posenet.eval_losses(
            model=model_posenet, batch=test_batch_pose, shape=shape, progress=False, clip_denoised=False,
            timestep_respacing=args.timestep_respacing_eval, cond_fn_with_grad=args.cond_fn_with_grad,
            early_stop=args.early_stop, compute_loss=False, grad_type='prox', smplx_model=smplx_model)
        if on_round is not None:
            # observer hook (tests): may return a tensor that replaces this round's PoseNet output for the next round
            repl = on_round(iter_idx, val_output_traj, traj_rec_full, test_batch_pose['cond'], val_output_pose)
            if repl is not None:
                val_output_pose = repl
    return val_output_pose, val_output_traj


def reconstruct_video_outputs(pose_dataset, smplx_model, test_batch_pose, val_output_pose, return_verts=True):
    """test_prox_egobody.py:326-354 on the device: de-normalise the noisy input (test_batch_pose['motion_repr_noisy'] as
    ``run_video_rounds`` leaves it, [W,294,1,Tp]) and the PoseNet output, and recover joints (and vertices) of the noisy
    motion from its SMPL-X parameters and of the reconstruction from its absolute trajectory and from its SMPL-X
    parameters.  Returns a dict of device tensors."""
    noisy = test_batch_pose['motion_repr_noisy']
    if noisy.dim() != 4 or tuple(noisy.shape) != tuple(val_output_pose.shape):
        raise RohmB200Error(f"reconstruct_video_outputs: test_batch_pose['motion_repr_noisy'] must be the [W, 294, 1, Tp] "
                            f"rows run_video_rounds leaves, like val_output_pose {tuple(val_output_pose.shape)}; got "
                            f"{tuple(noisy.shape)}")
    mean, std = glue.stats_on(pose_dataset, val_output_pose.device)
    noisy = noisy[:, :, 0].permute(0, 2, 1) * std + mean
    rec = val_output_pose[:, :, 0].permute(0, 2, 1) * std + mean
    out = {'motion_repr_noisy': noisy, 'motion_repr_rec': rec}
    res = recover_from_repr_smpl(split_repr(noisy), 'smplx_params', smplx_model, return_verts=return_verts)
    res = res if return_verts else (res, None)
    out['rec_ric_data_noisy'], out['smpl_verts_noisy'] = res
    out['rec_ric_data_rec_from_abs_traj'] = recover_from_repr_smpl(split_repr(rec), 'joint_abs_traj', smplx_model)
    res = recover_from_repr_smpl(split_repr(rec), 'smplx_params', smplx_model, return_verts=return_verts)
    res = res if return_verts else (res, None)
    out['rec_ric_data_rec_from_smpl'], out['smpl_verts_rec'] = res
    return out


def video_result_dicts(windows, outputs, test_batch_pose, frame_names=None):
    """The pickle payload of test_prox_egobody.py:356-384, one dict (numpy) per recording of ``windows`` (the Windows of
    ``windows.encode_video``), holding that recording's windows in start order, each once.  outputs: the dict of
    ``reconstruct_video_outputs``; test_batch_pose: the pose batch after ``run_video_rounds``.  frame_names (optional, one
    list of frame names per recording) fills 'frame_name_list' [n, clip_len] from each window's start; recording_name and
    gender_gt stay with the caller, who knows them.

    Two deliberate differences from the reference: it stores only its last batch's frame names (the same as these whenever
    a recording fits in one batch), and its ``len // batch_size + 1`` loop appends a wrapped-around duplicate batch when
    the window count is a multiple of the batch size; here every window appears once."""
    W, R = len(windows), len(windows.lengths)
    if frame_names is not None and len(frame_names) != R:
        raise RohmB200Error(f"video_result_dicts: frame_names must hold one name list per recording ({R}), got "
                            f"{len(frame_names)}")
    host = lambda t: t.detach().cpu().numpy()
    per_window = {'trans_scene2cano_list': host(test_batch_pose['transf_matrix']),
                  'rec_ric_data_noisy_list': host(outputs['rec_ric_data_noisy']),
                  'rec_ric_data_rec_list_from_abs_traj': host(outputs['rec_ric_data_rec_from_abs_traj']),
                  'rec_ric_data_rec_list_from_smpl': host(outputs['rec_ric_data_rec_from_smpl']),
                  'joints_input_scene_coord_list': host(test_batch_pose['noisy_joints_scene_coord']),
                  'motion_repr_noisy_list': host(outputs['motion_repr_noisy']),
                  'motion_repr_rec_list': host(outputs['motion_repr_rec']),
                  'mask_joint_vis_list': host(test_batch_pose['mask_joint_vis'][:, 0:-2])}
    if test_batch_pose.get('gt_joints_scene_coord') is not None:
        per_window['joints_gt_scene_coord_list'] = host(test_batch_pose['gt_joints_scene_coord'])
    bad = [k for k, v in per_window.items() if v.shape[0] != W]
    if bad:
        raise RohmB200Error(f"video_result_dicts: {bad} do not hold the {W} windows")
    rec, start = host(windows.recording).astype(np.int64), host(windows.start).astype(np.int64)
    payloads = []
    for r in range(R):
        idx = np.flatnonzero(rec == r)
        idx = idx[np.argsort(start[idx], kind='stable')]
        save = {k: v[idx] for k, v in per_window.items()}
        save['repr_name_list'], save['repr_dim_dict'] = REPR_LIST, REPR_DIM_DICT
        if frame_names is not None:
            names = np.asarray(frame_names[r])
            save['frame_name_list'] = np.asarray([names[s:s + windows.clip_len] for s in start[idx]]).reshape(
                len(idx), windows.clip_len)
        payloads.append(save)
    return payloads


def result_dict(args, outputs_per_batch):
    """The pickle payload of test_amass_full.py:446-458 (numpy, concatenated over batches).  Batches reconstructed with
    lengths give lists of per-clip arrays for the ``*_list`` keys instead."""
    if any(isinstance(o['motion_repr_rec'], list) for o in outputs_per_batch):
        cat = lambda key: [c.detach().cpu().numpy() for o in outputs_per_batch
                           for c in (o[key] if isinstance(o[key], list) else list(o[key]))]
    else:
        cat = lambda key: np.concatenate([o[key].detach().cpu().numpy() for o in outputs_per_batch], axis=0)
    save = {'mask_scheme': args.mask_scheme, 'repr_name_list': REPR_LIST, 'repr_dim_dict': REPR_DIM_DICT,
            'rec_ric_data_clean_list': cat('rec_ric_data_clean'),
            'rec_ric_data_rec_list_from_abs_traj': cat('rec_ric_data_rec_from_abs_traj'),
            'rec_ric_data_rec_list_from_smpl': cat('rec_ric_data_rec_from_smpl'),
            'motion_repr_clean_list': cat('motion_repr_clean'), 'motion_repr_rec_list': cat('motion_repr_rec')}
    if args.input_noise:
        save['rec_ric_data_noisy_list'] = cat('rec_ric_data_noisy')
        save['motion_repr_noisy_list'] = cat('motion_repr_noisy')
    return save
