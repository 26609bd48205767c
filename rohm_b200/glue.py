"""Device-side replacements for what the reference drivers do around the sampling loops on the host
(SURVEY.md 8f rows N1, N3, N4): the inter-round glue of test_amass_full.py:256-311, the PoseNet condition assembly with
its occlusion masks (:313-370) and the rotation / representation recovery helpers the drivers call
(data_loaders/motion_representation.py:285-398, data_loaders/common/quaternion.py:482-501,
utils/konia_transform.py:317-340).  Every function is a checked wrapper around one C-ABI entry of librohm_b200.so;
tensors stay on the GPU, nothing synchronises.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import RohmB200Error

BODY_FEAT_DIM = 294
TRAJ_FULL_DIM = 22

# joints whose features the 'lower' / 'upper' occlusion schemes blank out (test_amass_full.py:340, 351)
_MASK_JOINTS = {'lower': (1, 2, 4, 5, 7, 8, 10, 11), 'upper': (3, 6, 9, 12, 13, 14, 15, 16, 17, 18, 19, 20)}


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _f32c(t, name):
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise RohmB200Error(f"{name}: expected a CUDA tensor (rohm_b200 has no CPU path)")
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.contiguous().float()


def stats_on(dataset, device):
    """(Mean, Std) of a dataset object as cached fp32 device tensors."""
    cache = dataset.__dict__.setdefault("_rohm_stats", {}) if hasattr(dataset, "__dict__") else {}
    key = str(device)
    if key not in cache:
        cache[key] = (torch.from_numpy(np.ascontiguousarray(dataset.Mean, dtype=np.float32)).to(device),
                      torch.from_numpy(np.ascontiguousarray(dataset.Std, dtype=np.float32)).to(device))
    return cache[key]


def device_lengths(values, device):
    """Per-clip frame counts (ints) as the int32 device tensor [B] the ``lengths`` arguments of this module take, with its
    packed layout attached so that no call has to read it back from the device."""
    t = torch.tensor(values, dtype=torch.int32, device=device)
    _attach_layout(t, values)
    return t


def _attach_layout(lengths, values):
    values = tuple(int(v) for v in values)
    off = np.concatenate([[0], np.cumsum(values)]).astype(np.int32)
    lengths._rohm_layout = (lengths._version, values, torch.from_numpy(off).to(lengths.device), int(off[-1]))


def clip_layout(lengths, B, T, name, least=1):
    """Checks a ``lengths`` argument (int32 CUDA tensor [B], least <= lengths[b] <= T) and returns (clip_off, total): the
    exclusive prefix sum as an int32 device tensor [B+1] (frame t of clip b is packed row clip_off[b] + t) and the number
    of frames in the clips.  Tensors from ``device_lengths`` carry the layout; any other is read back once."""
    if (not isinstance(lengths, torch.Tensor) or lengths.dtype != torch.int32 or lengths.device.type != "cuda" or
            tuple(lengths.shape) != (B,) or not lengths.is_contiguous()):
        raise RohmB200Error(f"{name}: lengths must be a contiguous int32 CUDA tensor of shape [{B}], got "
                            f"{getattr(lengths, 'dtype', type(lengths))} {tuple(getattr(lengths, 'shape', ()))}")
    lay = getattr(lengths, "_rohm_layout", None)
    if lay is None or lay[0] != lengths._version:
        _attach_layout(lengths, lengths.tolist())
        lay = lengths._rohm_layout
    bad = [(b, v) for b, v in enumerate(lay[1]) if not least <= v <= T]
    if bad:
        raise RohmB200Error(f"{name}: lengths must lie in [{least}, {T}]; lengths[{bad[0][0]}] = {bad[0][1]}")
    return lay[2], lay[3]


def split_clips(packed, lengths):
    """Packed rows [sum of lengths, ...] -> one view [lengths[b], ...] per clip."""
    return list(torch.split(packed, list(lengths._rohm_layout[1]), dim=0))


def traj_to_full_repr(body_model, traj_out, repr_clean, traj_dataset, pose_dataset, lengths=None):
    """test_amass_full.py:268-311.  traj_out [B,T,13|22] (TrajNet output), repr_clean [B,T,294] (the trajectory batch's
    motion_repr_clean), both z-scored with traj_dataset's statistics -> (composite [B,T,294] -- what the driver stores as
    motion_repr_clean_root_rec / motion_repr_noisy --, traj_rec_full [B,T-1,22] z-scored with pose_dataset's statistics).
    lengths (int32 device [B], 2 <= lengths[b] <= T trajectory frames): FK runs over the clips' own frames only, the NaN
    repair and the velocity pairs stay inside each clip, and composite rows >= lengths[b] / traj_rec_full rows >=
    lengths[b] - 1 are zeros; a clip's rows equal the call on that clip alone, bit for bit."""
    from .body_model import kernels_for
    traj_out, repr_clean = _f32c(traj_out, "traj_out"), _f32c(repr_clean, "repr_clean")
    B, T, D = traj_out.shape
    if tuple(repr_clean.shape) != (B, T, BODY_FEAT_DIM):
        raise RohmB200Error(f"traj_to_full_repr: repr_clean must be [{B}, {T}, {BODY_FEAT_DIM}], got {tuple(repr_clean.shape)}")
    dev = traj_out.device
    tm, ts = stats_on(traj_dataset, dev)
    pm, ps = stats_on(pose_dataset, dev)
    if lengths is not None:
        clip_off, total = clip_layout(lengths, B, T, "traj_to_full_repr", least=2)
        k = kernels_for(body_model, dev, total, with_vertices=False)
        return k.traj_glue(traj_out, repr_clean, tm, ts, pm, ps, lengths=(lengths, clip_off, total))
    k = kernels_for(body_model, dev, B * T, with_vertices=False)
    return k.traj_glue(traj_out, repr_clean, tm, ts, pm, ps)


def traj_repr_from_joints(joints, global_orient_aa, transl, mean, std, lengths=None, frames=None):
    """get_repr_smplx's 22 trajectory channels (motion_representation.py:187-282) from joints [B,T,22,3], axis-angle global
    orientations [B,T,3] and translations [B,T,3] -> [B,T-1,22], z-scored with mean / std (device tensors, >= 22 entries).
    lengths (int32 device [B], 2 <= lengths[b] <= T = ``frames``): the three inputs hold the clips packed ([sum of lengths,
    ...]); the output keeps the padded shape [B,T-1,22] with zeros from row lengths[b] - 1."""
    joints, go, tr = _f32c(joints, "joints"), _f32c(global_orient_aa, "global_orient_aa"), _f32c(transl, "transl")
    lib, ctx = _lib.load(), _lib.ctx(joints.device.index)
    clip_off = None
    if lengths is not None:
        B, T = int(lengths.shape[0]), int(frames)
        clip_off, total = clip_layout(lengths, B, T, "traj_repr_from_joints", least=2)
        if joints.shape[0] != total or go.numel() != total * 3 or tr.numel() != total * 3:
            raise RohmB200Error(f"traj_repr_from_joints: with lengths the inputs hold the {total} packed frames of the clips")
    else:
        B, T = joints.shape[0], joints.shape[1]
    out = torch.empty(B, T - 1, TRAJ_FULL_DIM, device=joints.device)
    rc = lib.rohm_traj_repr_from_joints(ctx, _p(joints), _p(go), _p(tr), _p(mean), _p(std), B, T, _p(lengths), _p(clip_off),
                                        _p(out), _stream(joints.device))
    _lib.check(rc, ctx)
    return out


def pose_to_control_cond(pose_out, T, pose_feat_dim=272, lengths=None):
    """test_amass_full.py:256-258: control_cond [B,T,pose_feat_dim] from the PoseNet output [B,294,1,T-1].
    lengths (int32 device [B], pose frames per clip): the frame repeated into control frame lengths[b] is the clip's own
    last pose frame, later control frames are zeros and the output is never read past a clip."""
    pose_out = _f32c(pose_out, "pose_out")
    B, Cc, _, Tp = pose_out.shape
    out = torch.empty(B, T, pose_feat_dim, device=pose_out.device)
    lib, ctx = _lib.load(), _lib.ctx(pose_out.device.index)
    if lengths is not None:
        clip_layout(lengths, B, Tp, "pose_to_control_cond")
    rc = lib.rohm_pose_to_control_cond(ctx, _p(pose_out), B, Tp, T, Cc - pose_feat_dim, pose_feat_dim, _p(lengths), _p(out),
                                       _stream(pose_out.device))
    _lib.check(rc, ctx)
    return out


def channel_keep_mask(mask_scheme, traj_feat_dim=22):
    """294-byte keep mask of the 'lower' / 'upper' occlusion schemes (test_amass_full.py:338-358): for the masked joints the
    local position, local velocity and 6-D pose channels are zeroed."""
    keep = np.ones(BODY_FEAT_DIM, dtype=np.uint8)
    if mask_scheme in _MASK_JOINTS:
        ids = np.asarray(_MASK_JOINTS[mask_scheme])
        for k in range(3):
            keep[traj_feat_dim + ids * 3 + k] = 0
            keep[traj_feat_dim + 22 * 3 + ids * 3 + k] = 0
        for k in range(6):
            keep[traj_feat_dim + 22 * 3 + 22 * 3 + (ids - 1) * 6 + k] = 0
    elif mask_scheme not in (None, 'full', 'none', 'video'):
        raise RohmB200Error(f"unknown mask_scheme {mask_scheme!r}")
    return keep


def build_pose_cond(src, traj_full=None, chan_keep=None, frame_lo=None, frame_hi=None, zero_contact=False, frames=None,
                    lengths=None, vis_mask=None):
    """PoseNet condition [B,294,1,Tp] (test_amass_full.py:320-370): ``src`` is [B,Ts,294] (driver tensors) or [B,294,1,Ts]
    (a previous PoseNet output), Tp = ``frames`` (default Ts); channels [0,22) <- traj_full [B,Tp,22]; channels >= 22 are
    zeroed where chan_keep == 0, inside [frame_lo[b], frame_hi[b]) and (zero_contact) in the contact channels.
    lengths (int32 device [B], pose frames per clip): frames past a clip are zeros, src / traj_full are not read there.
    vis_mask (float32 CUDA [B,vis_T,294], vis_T >= Tp; the video loader's mask_vec_vis, test_prox_egobody.py:302-309): after
    the occlusion zeroing every channel of frame t < Tp is multiplied by vis_mask[b,t] -- a multiply, so -x * 0 = -0.0,
    NaN * 1 = NaN and Inf * 0 = NaN as in the reference -- and the contact zeroing comes after it.  Not with lengths."""
    src = _f32c(src, "src")
    if src.dim() == 4:
        B, Cc, _, Ts = src.shape
        channel_major = 1
    else:
        B, Ts, Cc = src.shape
        channel_major = 0
    if Cc != BODY_FEAT_DIM:
        raise RohmB200Error(f"build_pose_cond: expected {BODY_FEAT_DIM} channels, got {Cc}")
    Tp = Ts if frames is None else int(frames)
    dev = src.device
    if traj_full is not None:
        traj_full = _f32c(traj_full, "traj_full")
        if tuple(traj_full.shape) != (B, Tp, TRAJ_FULL_DIM):
            raise RohmB200Error(f"build_pose_cond: traj_full must be [{B}, {Tp}, 22], got {tuple(traj_full.shape)}")
    keep_t = None
    if chan_keep is not None:
        keep_t = (chan_keep if isinstance(chan_keep, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(chan_keep)))
        keep_t = keep_t.to(device=dev, dtype=torch.uint8).contiguous()
    lo_t = hi_t = None
    if frame_lo is not None:
        lo_t = torch.as_tensor(frame_lo).to(device=dev, dtype=torch.int32).contiguous()
        hi_t = torch.as_tensor(frame_hi).to(device=dev, dtype=torch.int32).contiguous()
    vis_T = 0
    if vis_mask is not None:
        if lengths is not None:
            raise RohmB200Error("build_pose_cond: vis_mask applies to whole clips; it is refused with lengths")
        if (not isinstance(vis_mask, torch.Tensor) or vis_mask.device != dev or vis_mask.dtype != torch.float32 or
                vis_mask.dim() != 3 or vis_mask.shape[0] != B or vis_mask.shape[1] < Tp or vis_mask.shape[2] != BODY_FEAT_DIM):
            raise RohmB200Error(f"build_pose_cond: vis_mask must be a float32 tensor [{B}, >={Tp}, {BODY_FEAT_DIM}] on {dev}, "
                                f"got {getattr(vis_mask, 'dtype', type(vis_mask))} {tuple(getattr(vis_mask, 'shape', ()))} "
                                f"on {getattr(vis_mask, 'device', None)}")
        vis_mask = vis_mask.contiguous()
        vis_T = int(vis_mask.shape[1])
    out = torch.empty(B, BODY_FEAT_DIM, 1, Tp, device=dev)
    lib, ctx = _lib.load(), _lib.ctx(dev.index)
    if lengths is not None:
        clip_layout(lengths, B, Tp, "build_pose_cond")
    rc = lib.rohm_build_pose_cond(ctx, _p(src), channel_major, Ts, _p(traj_full), _p(keep_t), _p(lo_t), _p(hi_t),
                                  int(bool(zero_contact)), B, Tp, _p(lengths), _p(vis_mask), vis_T, _p(out), _stream(dev))
    _lib.check(rc, ctx)
    return out


def rot6d_to_angle_axis(rot6d, want_rotmat=False):
    """rot6d_to_rotmat -> rotation_matrix_to_angle_axis (quaternion.py:482-501, konia_transform.py:317-340) on [..., 6]."""
    r = _f32c(rot6d, "rot6d").reshape(-1, 6)
    n = r.shape[0]
    aa = torch.empty(n, 3, device=r.device)
    rm = torch.empty(n, 3, 3, device=r.device) if want_rotmat else None
    lib, ctx = _lib.load(), _lib.ctx(r.device.index)
    rc = lib.rohm_rot6d_to_aa(ctx, _p(r), n, _p(aa), _p(rm), _stream(r.device))
    _lib.check(rc, ctx)
    aa = aa.reshape(tuple(rot6d.shape[:-1]) + (3,))
    return (aa, rm.reshape(tuple(rot6d.shape[:-1]) + (3, 3))) if want_rotmat else aa


def joints_from_traj_repr(x, mean, std, relative=False, channels_last=True, lengths=None):
    """recover_from_repr_smpl 'joint_abs_traj' / 'joint_rel_traj' (motion_representation.py:285-371) on a z-scored
    representation -> joints [B,T,22,3].  lengths (int32 device [B]): only the clips' own frames are computed, into packed
    joints [sum of lengths, 22, 3] (the absolute mode one thread per frame)."""
    x = _f32c(x, "x")
    if channels_last:
        B, T, _ = x.shape
    else:
        B, _, _, T = x.shape
    lib, ctx = _lib.load(), _lib.ctx(x.device.index)
    clip_off, total = None, 0
    if lengths is not None:
        clip_off, total = clip_layout(lengths, B, T, "joints_from_traj_repr")
        out = torch.empty(total, 22, 3, device=x.device)
    else:
        out = torch.empty(B, T, 22, 3, device=x.device)
    rc = lib.rohm_joints_from_traj(ctx, _p(x), int(bool(channels_last)), _p(mean), _p(std), B, T, _p(lengths), _p(clip_off),
                                   total, int(bool(relative)), _p(out), _stream(x.device))
    _lib.check(rc, ctx)
    return out
