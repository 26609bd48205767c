"""The evaluation metrics of the reference's eval_amass_full.py and eval_prox_egobody.py, computed on the device.

``amass`` takes the dict of ``pipeline.reconstruct_outputs`` (with or without ``lengths``), ``video`` the outputs of
``pipeline.reconstruct_video_outputs`` with the pose batch and ``Windows`` of ``windows.encode_video``, and
``from_payload`` the reference's own pickle dicts (or ``pipeline.result_dict`` / ``video_result_dicts``), so that results
written by the reference can be evaluated without it.  One CTA per clip or window computes the per-frame values in
float32 exactly as the reference's numpy does (DESIGN §4.16) and their float64 sums in a fixed order; a second launch
sums clips per recording in window order and over the recordings in the order given.

Each call returns a dict: per clip (``'clips'``) or per recording (``'recordings'``) a dict of metric -> float, the same
for ``'all'``, and ``'frames'``, the per-frame device tensors the reference keeps.  Values are in metres and m/s^2 as the
arrays are; the scripts print distances x1000 and the PROX/EgoBody penetration distance as ``-mean x 1000``.  Means are
float64 sums over float64 counts: the reference's float32 ``np.mean`` differs from them by its own rounding (about 5e-6
relative); ratios of counts are the reference's bit for bit.

Deviation: a recording without windows reports NaN with count 0 (the reference fails on ``np.concatenate([])``).
"""
import numpy as np
import torch

from . import _lib, glue
from ._lib import RohmB200Error

MASK_SCHEMES = ('lower', 'full')
DATASETS = ('prox', 'egobody')
LOWER_OCCLUDED = (1, 2, 4, 5, 7, 8, 10, 11)  # eval_amass_full.py:76
FULL_START, FULL_FRAMES = 65, 145  # eval_amass_full.py:83-85: occluded frames [65, 65 + int(ratio * 145))
ALL_JOINTS = (1 << 22) - 1
AMASS_SUMS = ('mpjpe', 'mpjpe_vis', 'mpjpe_occ', 'accel', 'pene_dist')
AMASS_COUNTS = ('mpjpe', 'mpjpe_vis', 'mpjpe_occ', 'contact_match', 'contact', 'skating_gt', 'skating_rec', 'skating',
                'accel', 'pene_freq', 'pene')
VIDEO_SUMS = ('acc', 'acc_error', 'gmpjpe', 'mpjpe', 'vis_num', 'vis_den', 'occ_num', 'occ_den', 'pene_freq',
              'pene_dist')


def _div(a, b):
    return float(a) / float(b) if b else float('nan')


def _cuda_f32(t, name, shape):
    """t as a contiguous float32 CUDA tensor whose shape matches `shape` (None: any extent)."""
    if not isinstance(t, torch.Tensor) or t.device.type != 'cuda':
        raise RohmB200Error(f"metrics: {name} must be a CUDA tensor, got {type(t).__name__}")
    if t.dim() != len(shape) or any(w is not None and t.shape[i] != w for i, w in enumerate(shape)):
        want = ", ".join("n" if w is None else str(w) for w in shape)
        raise RohmB200Error(f"metrics: {name} must be [{want}], got {tuple(t.shape)}")
    return t.contiguous().float()


def _reduce(sums, counts, order, group_off, n_groups, dev):
    """rohm_eval_reduce -> host (sums [G+1, ks] float64, counts [G+1, kc] int64); row G is over every group."""
    ks, kc = sums.shape[1], counts.shape[1]
    out_s = torch.empty(n_groups + 1, ks, dtype=torch.float64, device=dev)
    out_c = torch.empty(n_groups + 1, kc, dtype=torch.int64, device=dev)
    lib, ctx = _lib.load(), _lib.ctx(dev.index)
    _lib.check(lib.rohm_eval_reduce(ctx, glue._p(sums), ks, glue._p(counts), kc, glue._p(order), glue._p(group_off),
                                    n_groups, glue._p(out_s), glue._p(out_c), glue._stream(dev)), ctx)
    return out_s.cpu().numpy(), out_c.cpu().numpy()


# ------------------------------------------------------------------------------------------------------------ AMASS
def _amass_values(s, c):
    s, c = dict(zip(AMASS_SUMS, s)), dict(zip(AMASS_COUNTS, c))
    return {'mpjpe_global': _div(s['mpjpe'], c['mpjpe']), 'mpjpe_global_vis': _div(s['mpjpe_vis'], c['mpjpe_vis']),
            'mpjpe_global_occ': _div(s['mpjpe_occ'], c['mpjpe_occ']),
            'contact_lbl_acc': _div(c['contact_match'], c['contact']),
            'skating_gt_ratio': _div(c['skating_gt'], c['skating']),
            'skating_rec_ratio': _div(c['skating_rec'], c['skating']), 'accel_error': _div(s['accel'], c['accel']),
            'ground_pene_freq': _div(c['pene_freq'], c['pene']), 'ground_pene_dist': _div(s['pene_dist'], c['pene'])}


def _occlusion(mask_scheme, traj_mask_ratio):
    if mask_scheme not in MASK_SCHEMES:
        raise RohmB200Error(f"metrics.amass: mask_scheme must be one of {MASK_SCHEMES}, got {mask_scheme!r}")
    if mask_scheme == 'lower':
        return sum(1 << j for j in LOWER_OCCLUDED), 0, 2 ** 31 - 1
    r = float(traj_mask_ratio)
    if not np.isfinite(r) or r < 0:
        raise RohmB200Error(f"metrics.amass: traj_mask_ratio must be finite and >= 0, got {traj_mask_ratio!r}")
    return ALL_JOINTS, FULL_START, min(FULL_START + int(r * FULL_FRAMES), 2 ** 31 - 1)


def amass(outputs, mask_scheme, traj_mask_ratio=0.0):
    """eval_amass_full.py:71-147 over the clips of ``reconstruct_outputs``: outputs['rec_ric_data_clean'] (G),
    ['rec_ric_data_rec_from_smpl'] (P), ['motion_repr_clean'] and ['motion_repr_rec'] (contact labels: the last 4
    channels), each a CUDA tensor [B,T,...] or, after ``lengths``, a list of B per-clip tensors [T_b,...].

    mask_scheme 'lower' splits the MPJPE into the visible joints and the occluded {1,2,4,5,7,8,10,11}; 'full' into the
    frames outside and inside [65, 65 + int(traj_mask_ratio * 145)), clamped to each clip (an empty set gives NaN).
    Skating of both G and P measures heights from the clean clip's lowest z, h0 (NaN if G holds one).  Returns
    {'clips': [per-clip metrics], 'all': metrics pooled over every clip's frames, 'frames': per-frame device tensors
    (mpjpe [.,22], accel_error [.,T-2,22], skating_gt / skating_rec [.,T-1] bool, contact_match [.,4] bool, pene_freq [.,2]
    bool, pene_dist [.,2], per clip as the inputs are), 'h0': [B]}."""
    occ_joints, lo, hi = _occlusion(mask_scheme, traj_mask_ratio)
    keys = ('rec_ric_data_clean', 'rec_ric_data_rec_from_smpl', 'motion_repr_clean', 'motion_repr_rec')
    missing = [k for k in keys if outputs.get(k) is None]
    if missing:
        raise RohmB200Error(f"metrics.amass: outputs lack {missing}")
    ragged = isinstance(outputs[keys[0]], (list, tuple))
    if ragged:
        clips = [list(outputs[k]) for k in keys]
        B = len(clips[0])
        if any(len(c) != B for c in clips):
            raise RohmB200Error("metrics.amass: the per-clip lists hold different clip counts")
        lens = []
        for b in range(B):
            T = clips[0][b].shape[0] if clips[0][b].dim() > 0 else 0
            for k, c in zip(keys, clips):
                _cuda_f32(c[b], f"{k}[{b}]", (T, 22, 3) if k.startswith('rec_ric') else (T, None))
            lens.append(T)
        width = clips[2][0].shape[1] if B else 294
        if any(c.shape[1] != width for c in clips[2] + clips[3]):
            raise RohmB200Error("metrics.amass: the motion representations have different channel counts")
        cat = lambda i: (torch.cat([t.float() for t in clips[i]]).contiguous() if B else None)
        G, P, RC, RR = cat(0), cat(1), cat(2), cat(3)
        dev = clips[0][0].device if B else torch.device('cuda', torch.cuda.current_device())
    else:
        G = _cuda_f32(outputs[keys[0]], keys[0], (None, None, 22, 3))
        B, T = G.shape[0], G.shape[1]
        P = _cuda_f32(outputs[keys[1]], keys[1], (B, T, 22, 3))
        RC = _cuda_f32(outputs[keys[2]], keys[2], (B, T, None))
        width = RC.shape[2]
        RR = _cuda_f32(outputs[keys[3]], keys[3], (B, T, width))
        lens = [T] * B
        dev = G.device
    if width < 4:
        raise RohmB200Error(f"metrics.amass: the motion representation needs the 4 contact channels, has {width}")
    if any(t is not None and t.device != dev for t in (G, P, RC, RR)):
        raise RohmB200Error("metrics.amass: the inputs live on different devices")
    N = sum(lens)
    off = torch.tensor(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), device=dev)
    f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    u8 = lambda *s: torch.empty(*s, dtype=torch.uint8, device=dev)
    h0, mpjpe, accerr, pene_dist = f32(B), f32(N, 22), f32(N, 22), f32(N, 2)
    sk_gt, sk_rec, contact, pene_freq = u8(N), u8(N), u8(N, 4), u8(N, 2)
    sums = torch.zeros(B, len(AMASS_SUMS), dtype=torch.float64, device=dev)
    counts = torch.zeros(B, len(AMASS_COUNTS), dtype=torch.int64, device=dev)
    lib, ctx = _lib.load(), _lib.ctx(dev.index)
    if B > 0:
        _lib.check(lib.rohm_eval_amass(ctx, glue._p(G), glue._p(P), glue._p(RC), glue._p(RR), width, glue._p(off), B,
                                       occ_joints, lo, hi, glue._p(h0), glue._p(mpjpe), glue._p(accerr),
                                       glue._p(sk_gt), glue._p(sk_rec), glue._p(contact), glue._p(pene_freq),
                                       glue._p(pene_dist), glue._p(sums), glue._p(counts), glue._stream(dev)), ctx)
    order = torch.arange(B, dtype=torch.int32, device=dev)
    group = torch.tensor([0, B], dtype=torch.int32, device=dev)
    tot_s, tot_c = _reduce(sums, counts, order, group, 1, dev)
    per_s, per_c = sums.cpu().numpy(), counts.cpu().numpy()

    def per_clip(t, drop=0):
        if ragged:
            return [x[:max(n - drop, 0)] for x, n in zip(torch.split(t, lens), lens)]
        v = t.view(B, lens[0] if B else 0, *t.shape[1:])
        return v[:, :max(v.shape[1] - drop, 0)]

    frames = {'mpjpe': per_clip(mpjpe), 'accel_error': per_clip(accerr, 2),
              'skating_gt': per_clip(sk_gt.bool(), 1), 'skating_rec': per_clip(sk_rec.bool(), 1),
              'contact_match': per_clip(contact.bool()), 'pene_freq': per_clip(pene_freq.bool()),
              'pene_dist': per_clip(pene_dist)}
    return {'clips': [_amass_values(per_s[b], per_c[b]) for b in range(B)], 'all': _amass_values(tot_s[1], tot_c[1]),
            'frames': frames, 'h0': h0}


# ------------------------------------------------------------------------------------------------------------ video
def _video_values(sums, skating, n_win, T, with_gt):
    s = dict(zip(VIDEO_SUMS, sums))
    out = {'skating': _div(skating, n_win * (T - 1)), 'acc': _div(s['acc'], n_win * (T - 2)),
           'ground_pene_freq': _div(s['pene_freq'], n_win * T), 'ground_pene_dist': _div(s['pene_dist'], n_win * T)}
    if with_gt:
        out.update(acc_error=_div(s['acc_error'], n_win * (T - 2)), gmpjpe=_div(s['gmpjpe'], n_win * T * 22),
                   mpjpe=_div(s['mpjpe'], n_win * T * 22), mpjpe_vis=_div(s['vis_num'], s['vis_den']),
                   mpjpe_occ=_div(s['occ_num'], s['occ_den']))
    return out


def _video(rec, transf, gt, mask, win_rec, order, n_per_rec, dataset, floor_height):
    """The video pass over W windows (rec [W,T,22,3] canonical, transf [W,4,4], gt [W,>=T,22,3] / mask [W,>=T,22] or
    None, win_rec int32 [W]); order: int32 [W], the windows of recording 0 in start order, then recording 1, ...;
    n_per_rec: host window counts."""
    if dataset not in DATASETS:
        raise RohmB200Error(f"metrics.video: dataset must be one of {DATASETS}, got {dataset!r}")
    R = len(n_per_rec)
    fl = np.asarray(floor_height, dtype=np.float64).reshape(-1) if floor_height is not None else np.zeros(0)
    if fl.shape[0] != R:
        raise RohmB200Error(f"metrics.video: floor_height must hold one height per recording ({R}), got {fl.shape[0]}")
    W, T = rec.shape[0], rec.shape[1]
    if T < 3:
        raise RohmB200Error(f"metrics.video: windows need at least 3 frames, got {T}")
    dev = rec.device
    if gt is None and mask is not None:
        mask = None  # the visibility split weighs the ground-truth MPJPE; without ground truth there is nothing to weigh
    f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    skate = torch.empty(W, T - 1, dtype=torch.uint8, device=dev)
    acc, pene_freq, pene_dist = f32(W, T - 2), f32(W, T), f32(W, T)
    accerr, gmpjpe, mpjpe = (f32(W, T - 2), f32(W, T, 22), f32(W, T, 22)) if gt is not None else (None, None, None)
    sums = torch.zeros(W, len(VIDEO_SUMS), dtype=torch.float64, device=dev)
    counts = torch.zeros(W, 1, dtype=torch.int64, device=dev)
    floors = torch.from_numpy(fl.astype(np.float32)).to(dev)
    lib, ctx = _lib.load(), _lib.ctx(dev.index)
    if W > 0:
        _lib.check(lib.rohm_eval_video(ctx, glue._p(rec), T, glue._p(transf), glue._p(gt),
                                       gt.shape[1] if gt is not None else 0, glue._p(mask),
                                       mask.shape[1] if mask is not None else 0, glue._p(win_rec), glue._p(floors), W,
                                       int(dataset == 'egobody'), glue._p(skate), glue._p(acc), glue._p(accerr),
                                       glue._p(gmpjpe), glue._p(mpjpe), glue._p(pene_freq), glue._p(pene_dist),
                                       glue._p(sums), glue._p(counts), glue._stream(dev)), ctx)
    goff = torch.tensor(np.concatenate([[0], np.cumsum(n_per_rec)]).astype(np.int32), device=dev)
    tot_s, tot_c = _reduce(sums, counts, order, goff, R, dev)
    with_gt = gt is not None
    recs = [_video_values(tot_s[r], tot_c[r, 0], n_per_rec[r], T, with_gt) for r in range(R)]
    frames = {'skating': skate.bool(), 'acc': acc, 'ground_pene_freq': pene_freq, 'ground_pene_dist': pene_dist}
    if with_gt:
        frames.update(acc_error=accerr, gmpjpe=gmpjpe, mpjpe=mpjpe)
    return {'recordings': recs, 'all': _video_values(tot_s[R], tot_c[R, 0], sum(n_per_rec), T, with_gt),
            'frames': frames, 'order': order}


def video(windows, outputs, test_batch_pose, dataset, floor_height):
    """eval_prox_egobody.py:172-272 and :453-490 over the windows of ``windows.encode_video``: outputs of
    ``reconstruct_video_outputs`` (rec_ric_data_rec_from_smpl [W,T,22,3], canonical), test_batch_pose after
    ``run_video_rounds`` (transf_matrix; for EgoBody with ground truth gt_joints_scene_coord and mask_joint_vis), dataset
    'prox' (z up) or 'egobody' (y up) and floor_height, one height per recording of ``windows`` (the reference's
    prox_floor_height / egobody_floor_height of the recording's scene).

    Per recording its windows count in start order; 'all' concatenates the recordings in order (the 2 frames shared by
    overlapping windows count twice, as in the reference).  Metrics: skating, acc (||acc||), ground_pene_freq,
    ground_pene_dist (the mean itself; the script prints -mean x 1000) and, with ground truth, acc_error, gmpjpe, mpjpe
    (root-relative), mpjpe_vis and mpjpe_occ.  'frames' holds the per-window device tensors in the windows' own order;
    'order' the window indices grouped by recording in start order."""
    R = len(windows.lengths)
    W = len(windows)
    keys = [k for k in ('transf_matrix',) if test_batch_pose.get(k) is None]
    if outputs.get('rec_ric_data_rec_from_smpl') is None or keys:
        raise RohmB200Error("metrics.video: needs outputs['rec_ric_data_rec_from_smpl'] and test_batch_pose"
                            "['transf_matrix']")
    rec = _cuda_f32(outputs['rec_ric_data_rec_from_smpl'], "rec_ric_data_rec_from_smpl", (W, None, 22, 3))
    T = rec.shape[1]
    transf = _cuda_f32(test_batch_pose['transf_matrix'], "transf_matrix", (W, 4, 4))
    gt = test_batch_pose.get('gt_joints_scene_coord')
    mask = None
    if gt is not None:
        gt = _cuda_f32(gt, "gt_joints_scene_coord", (W, None, 22, 3))
        mask = _cuda_f32(test_batch_pose['mask_joint_vis'], "mask_joint_vis", (W, None, 22))
        if gt.shape[1] < T or mask.shape[1] < T:
            raise RohmB200Error(f"metrics.video: ground truth and mask_joint_vis need {T} frames per window")
    if any(t is not None and t.device != rec.device for t in (transf, gt, mask, windows.recording)):
        raise RohmB200Error("metrics.video: the inputs and the windows live on different devices")
    from .windows import window_table
    n_per_rec = [0] * R
    for r, _ in window_table(windows.lengths, windows.clip_len, windows.overlap):
        n_per_rec[r] += 1
    if sum(n_per_rec) != W:
        raise RohmB200Error(f"metrics.video: the windows' recordings cut {sum(n_per_rec)} windows, the batch holds {W}")
    key = windows.recording.long() * (max(windows.lengths, default=0) + 1) + windows.start.long()
    order = torch.sort(key, stable=True).indices.to(torch.int32) if W else key.to(torch.int32)
    return _video(rec, transf, gt, mask, windows.recording.contiguous(), order, n_per_rec, dataset, floor_height)


# ------------------------------------------------------------------------------------------------------------ payloads
def _host_f32(a, name, shape):
    a = np.asarray(a)
    if a.ndim != len(shape) or any(w is not None and a.shape[i] != w for i, w in enumerate(shape)):
        want = ", ".join("n" if w is None else str(w) for w in shape)
        raise RohmB200Error(f"metrics.from_payload: {name} must be [{want}], got {a.shape}")
    return np.ascontiguousarray(a, dtype=np.float32)


def from_payload(payload, mask_scheme=None, traj_mask_ratio=0.0, dataset=None, floor_height=None, device=None):
    """The metrics of the reference's pickles, on the device.  payload: the dict eval_amass_full.py loads (or
    ``pipeline.result_dict``; per-clip lists after lengths) -> ``amass`` with mask_scheme (default payload['mask_scheme'])
    and traj_mask_ratio; or a list of the per-recording dicts eval_prox_egobody.py loads (or ``video_result_dicts``), in
    the order to concatenate them -> the ``video`` pass with dataset and floor_height (one per dict)."""
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    up = lambda a: torch.from_numpy(a).to(dev)
    if isinstance(payload, dict):
        scheme = mask_scheme if mask_scheme is not None else payload.get('mask_scheme')
        keys = {'rec_ric_data_clean': 'rec_ric_data_clean_list', 'rec_ric_data_rec_from_smpl':
                'rec_ric_data_rec_list_from_smpl', 'motion_repr_clean': 'motion_repr_clean_list',
                'motion_repr_rec': 'motion_repr_rec_list'}
        missing = [v for v in keys.values() if v not in payload]
        if missing:
            raise RohmB200Error(f"metrics.from_payload: the AMASS payload lacks {missing}")
        if isinstance(payload['rec_ric_data_clean_list'], (list, tuple)):
            outs = {k: [up(np.ascontiguousarray(a, dtype=np.float32)) for a in payload[v]] for k, v in keys.items()}
        else:
            outs = {k: up(_host_f32(payload[v], v, (None, None, 22, 3) if k.startswith('rec_ric') else
                                    (None, None, None))) for k, v in keys.items()}
        _occlusion(scheme, traj_mask_ratio)
        return amass(outs, scheme, traj_mask_ratio)
    payloads = list(payload)
    if dataset not in DATASETS:
        raise RohmB200Error(f"metrics.from_payload: dataset must be one of {DATASETS}, got {dataset!r}")
    fl = np.asarray(floor_height if floor_height is not None else [], dtype=np.float64).reshape(-1)
    if fl.shape[0] != len(payloads):
        raise RohmB200Error(f"metrics.from_payload: floor_height must hold one height per recording "
                            f"({len(payloads)}), got {fl.shape[0]}")
    recs, tfs, gts, masks, n_per_rec = [], [], [], [], []
    T = None
    with_gt = dataset == 'egobody' and any('joints_gt_scene_coord_list' in p for p in payloads)
    for i, p in enumerate(payloads):
        rec = _host_f32(p['rec_ric_data_rec_list_from_smpl'], f"[{i}]['rec_ric_data_rec_list_from_smpl']",
                        (None, T, 22, 3))
        T = rec.shape[1] if T is None else T
        n = rec.shape[0]
        recs.append(rec)
        tfs.append(_host_f32(p['trans_scene2cano_list'], f"[{i}]['trans_scene2cano_list']", (n, 4, 4)))
        if with_gt:
            g = _host_f32(p['joints_gt_scene_coord_list'], f"[{i}]['joints_gt_scene_coord_list']", (n, None, 22, 3))
            m = _host_f32(p['mask_joint_vis_list'], f"[{i}]['mask_joint_vis_list']", (n, None, 22))
            if g.shape[1] < T or m.shape[1] < T:
                raise RohmB200Error(f"metrics.from_payload: recording {i}'s ground truth or mask holds fewer than {T} "
                                    "frames")
            gts.append(g[:, :T])
            masks.append(m[:, :T])
        n_per_rec.append(n)
    T = 3 if T is None else T
    cat = lambda xs, shape: up(np.ascontiguousarray(np.concatenate(xs)) if xs else np.zeros((0,) + shape, np.float32))
    W = sum(n_per_rec)
    win_rec = up(np.repeat(np.arange(len(payloads)), n_per_rec).astype(np.int32))
    order = up(np.arange(W, dtype=np.int32))
    return _video(cat(recs, (T, 22, 3)), cat(tfs, (4, 4)), cat(gts, (T, 22, 3)) if with_gt else None,
                  cat(masks, (T, 22)) if with_gt else None, win_rec, order, n_per_rec, dataset, fl)
