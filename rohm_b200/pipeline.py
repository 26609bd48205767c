"""The multi-round TrajNet -> PoseNet inference of the reference driver, device-resident.

``run_rounds`` replays test_amass_full.py:218-384 (one dataloader batch: optional trajectory infill mask, then
``sample_iter`` rounds of  TrajNet / TrajControl sampling -> inter-round glue -> PoseNet condition assembly with occlusion
masks -> guided PoseNet sampling)  with the same call sequence, flags, batch-dict side effects and CPU-generator draws as
the driver, but without its host round trips: the per-clip numpy / scipy loop of :268-311 is ``rohm_traj_glue``, the
condition assembly of :313-370 is ``rohm_build_pose_cond``, the TrajControl condition of :256-258 is
``rohm_pose_to_control_cond``.  ``reconstruct_outputs`` is the post-loop block :386-428 (joints / vertices of the clean,
reconstructed and noisy motions) and ``result_dict`` the driver's pickle payload (:446-458).

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
