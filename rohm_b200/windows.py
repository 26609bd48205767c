"""Whole recordings in and out of the rounds (SURVEY.md 8f row N4, sliding-window batching).

``encode`` cuts packed recordings into the reference's windows of ``clip_len`` frames (dataloader_video.py:160-183 with
overlap 2, dataloader_amass.py:105-131 with overlap 0), canonicalises each (cano_seq_smplx), encodes its 294-channel
representation (get_repr_smplx) and assembles the batch dicts ``pipeline.run_rounds`` takes, as DataloaderAMASS.__getitem__
builds them without input noise (dataloader_amass.py:319-341).  ``to_recordings`` maps each window's joints back to the
world frame of its recording (the inverse of transf_matrix, eval_prox_egobody.py:177-182).  Both are one kernel launch
(rohm_window_encode / rohm_window_to_world); tensors stay on the GPU.

Only full windows are cut, so a recording shorter than ``clip_len`` gives none, and the frames after a recording's last
window are not covered.  A window's results cover its first clip_len - 2 frames (the PoseNet frames): with overlap 2
consecutive windows tile the recording, with overlap 0 each leaves a 2-frame gap.  ``to_recordings`` reports which frames
a window covers and does not fill the others.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, glue
from ._lib import RohmB200Error

MAX_CLIP_LEN = 160  # one CTA of one thread per window frame
# channels of the 294-wide row the TrajNet condition keeps with repr_abs_only (dataloader_amass.py:337)
ABS_TRAJ_CHANNELS = (0, 2, 3, 6, 7, 8, 9, 10, 11, 12, 16, 17, 18)
PARAMS = (('global_orient', 3), ('transl', 3), ('betas', 10), ('body_pose', 63))


def window_table(lengths, clip_len=145, overlap=2):
    """[(recording, first frame)] of every window, in order: window k of a recording starts at k * (clip_len - overlap)
    and is cut while it ends inside the recording."""
    stride = clip_len - overlap
    return [(r, s) for r, n in enumerate(lengths) for s in range(0, int(n) - clip_len + 1, stride)]


class Windows:
    """The windows of one ``encode`` call: ``recording`` / ``start`` (int32 device [W]), ``transf`` (world -> canonical
    [W,4,4]), and the recordings' ``lengths`` (ints), ``offsets`` (int32 device [R+1]), ``clip_len`` and ``overlap``."""

    def __init__(self, recording, start, transf, lengths, offsets, clip_len, overlap):
        self.recording, self.start, self.transf = recording, start, transf
        self.lengths, self.offsets, self.clip_len, self.overlap = lengths, offsets, clip_len, overlap

    def __len__(self):
        return int(self.recording.shape[0])


def _check_shape(clip_len, overlap):
    if not 3 <= clip_len <= MAX_CLIP_LEN or not 0 <= overlap <= 2:
        raise RohmB200Error(f"windows: clip_len={clip_len}, overlap={overlap}; windows of 3 to {MAX_CLIP_LEN} frames with an "
                            "overlap of 0 to 2 frames (so that no recording frame lies in two windows' pose frames)")


def encode(body_model, params, lengths, pose_dataset, traj_dataset, clip_len=145, overlap=2):
    """params: SMPL-X parameters of R recordings packed frame after frame (CUDA tensors global_orient [N,3], transl [N,3],
    betas [N,10], body_pose [N,63] axis-angle, N = sum of lengths, z up); lengths: frames per recording (ints).  World joints
    come from ``body_model`` (FK only).  Returns (test_batch_traj, test_batch_pose, windows):

    * test_batch_traj: motion_repr_clean / motion_repr_noisy [W, clip_len-1, 294] z-scored with traj_dataset's statistics,
      cond [W, clip_len-1, 13] (the repr_abs_only channels; the first traj_feat_dim channels otherwise) and control_cond
      [W, clip_len-1, pose_feat_dim];
    * test_batch_pose: motion_repr_clean / motion_repr_noisy z-scored with pose_dataset's statistics;
    * windows: the window table and transf (``Windows``), for ``to_recordings``.

    Each window's rows depend on its own frames only: the same in any batch, order or packing of recordings."""
    p, lengths = _packed_params(params, lengths, clip_len, overlap)
    joints = None
    if window_table(lengths, clip_len, overlap):
        joints = body_model(transl=p['transl'], global_orient=p['global_orient'], body_pose=p['body_pose'],
                            betas=p['betas'], return_verts=False).joints[:, 0:22].contiguous()
    return _encode(p, joints, lengths, pose_dataset, traj_dataset, clip_len, overlap)


def encode_joints(params, joints, lengths, pose_dataset, traj_dataset, clip_len=145, overlap=2):
    """``encode`` with the recordings' 22-joint world positions given (joints [N,22,3], packed like params), as the
    reference loaders read them from preprocessed files."""
    p, lengths = _packed_params(params, lengths, clip_len, overlap)
    joints = glue._f32c(joints, "windows.encode_joints: joints")
    if joints.numel() != sum(lengths) * 66:
        raise RohmB200Error(f"windows.encode_joints: joints must hold [{sum(lengths)}, 22, 3], got {tuple(joints.shape)}")
    return _encode(p, joints, lengths, pose_dataset, traj_dataset, clip_len, overlap)


def _packed_params(params, lengths, clip_len, overlap):
    _check_shape(clip_len, overlap)
    lengths = tuple(int(n) for n in lengths)
    if not lengths or min(lengths) < 0:
        raise RohmB200Error(f"windows.encode: lengths must be one frame count >= 0 per recording, got {lengths}")
    total = sum(lengths)
    p = {}
    for name, width in PARAMS:
        t = glue._f32c(params[name], f"windows.encode: params['{name}']")
        if t.numel() != total * width:
            raise RohmB200Error(f"windows.encode: params['{name}'] must hold [{total}, {width}] (the packed recordings), got "
                                f"{tuple(t.shape)}")
        p[name] = t.reshape(total, width)
    return p, lengths


def _encode(p, joints, lengths, pose_dataset, traj_dataset, clip_len, overlap):
    dev = p['transl'].device
    tm, ts = glue.stats_on(traj_dataset, dev)
    pm, ps = glue.stats_on(pose_dataset, dev)
    if any(t.numel() != glue.BODY_FEAT_DIM for t in (tm, ts, pm, ps)):
        raise RohmB200Error("windows.encode: the datasets' Mean / Std must have 294 entries")
    W, T1 = len(window_table(lengths, clip_len, overlap)), clip_len - 1
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    offsets = torch.from_numpy(off).to(dev)
    rec = torch.empty(W, dtype=torch.int32, device=dev)
    start = torch.empty(W, dtype=torch.int32, device=dev)
    transf = torch.empty(W, 4, 4, device=dev)
    rt = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    rp = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    if W > 0:
        lib, ctx = _lib.load(), _lib.ctx(dev.index)
        n = C.c_int(0)
        rc = lib.rohm_window_encode(ctx, glue._p(p['global_orient']), glue._p(p['transl']), glue._p(p['betas']),
                                    glue._p(p['body_pose']), glue._p(joints), (C.c_int * len(off))(*off.tolist()),
                                    glue._p(offsets), len(lengths), clip_len, overlap, glue._p(tm), glue._p(ts),
                                    glue._p(pm), glue._p(ps), W, C.byref(n), glue._p(rec), glue._p(start), glue._p(transf),
                                    glue._p(rt), glue._p(rp), glue._stream(dev))
        _lib.check(rc, ctx)
        if n.value != W:
            raise RohmB200Error(f"windows.encode: the library cut {n.value} windows, the window rule {W}")
    tfd, pfd = traj_dataset.traj_feat_dim, traj_dataset.pose_feat_dim
    cond = rt[..., list(ABS_TRAJ_CHANNELS)] if tfd == len(ABS_TRAJ_CHANNELS) else rt[..., 0:tfd].clone()
    test_batch_traj = {'motion_repr_clean': rt, 'motion_repr_noisy': rt.clone(), 'cond': cond,
                       'control_cond': rt[..., -pfd:].contiguous()}
    test_batch_pose = {'motion_repr_clean': rp, 'motion_repr_noisy': rp.clone()}
    return test_batch_traj, test_batch_pose, Windows(rec, start, transf, lengths, offsets, clip_len, overlap)


def to_recordings(windows, joints):
    """joints: each window's clip_len - 2 pose frames in its canonical frame, [W, clip_len-2, 22, 3] or packed
    [W*(clip_len-2), 22, 3] (e.g. reconstruct_outputs' rec_ric_data_rec_from_smpl) -> (world, covered): per recording
    world-frame joints [lengths[r], 22, 3] and a bool mask [lengths[r]] of the frames a window covers.  Frames no window
    covers are zero."""
    W, P = len(windows), windows.clip_len - 2
    dev = windows.offsets.device
    j = glue._f32c(joints, "windows.to_recordings: joints")
    if j.numel() != W * P * 22 * 3:
        raise RohmB200Error(f"windows.to_recordings: joints must hold [{W} * {P}, 22, 3] (pose frames of every window), got "
                            f"{tuple(j.shape)}")
    total = sum(windows.lengths)
    world = torch.empty(total, 22, 3, device=dev)
    covered = torch.empty(total, dtype=torch.uint8, device=dev)
    if total > 0:
        lib, ctx = _lib.load(), _lib.ctx(dev.index)
        rc = lib.rohm_window_to_world(ctx, glue._p(j), glue._p(windows.recording), glue._p(windows.start),
                                      glue._p(windows.transf), W, windows.clip_len, glue._p(windows.offsets), total,
                                      glue._p(world), glue._p(covered), glue._stream(dev))
        _lib.check(rc, ctx)
    n = list(windows.lengths)
    return list(torch.split(world, n)), list(torch.split(covered.bool(), n))
