"""numpy restatement of the evaluation metrics (eval_amass_full.py:71-147, eval_prox_egobody.py:150-490) that
rohm_b200.metrics computes on the device.

Per-frame values are float32 and follow the reference's numpy order of operations, written out: a norm over 3 channels
is sqrt((s0 + s1) + s2), which is what np.linalg.norm(x, axis=-1) computes for float32 rows of 3; a mean over 22 joints
is numpy's pairwise sum (8 accumulators over the first 16 values, combined as a tree, then the rest in order) divided
by 22.  The scene transform is the reference's own expression (points_coord_trans with np.linalg.inv).  Sums are
float64, so the means here are the float64 means of the float32 per-frame values, not the reference's float32 np.mean.
"""
import numpy as np

FPS = 30
LOWER_OCCLUDED = [1, 2, 4, 5, 7, 8, 10, 11]
FOOT = [7, 10, 8, 11]
F32 = np.float32


def norm3(x):
    """np.linalg.norm(x, axis=-1) of float32 rows of 3, as the explicit sum order the kernel uses."""
    x = np.asarray(x, F32)
    s = x * x
    return np.sqrt((s[..., 0] + s[..., 1]) + s[..., 2])


def norm2(x):
    x = np.asarray(x, F32)
    s = x * x
    return np.sqrt(s[..., 0] + s[..., 1])


def accel(x):
    """(x[t+2] - 2 x[t+1] + x[t]) * 900 along axis 1 in float32, left to right."""
    x = np.asarray(x, F32)
    return (((x[:, 2:] - F32(2) * x[:, 1:-1]) + x[:, :-2]) * F32(FPS ** 2)).astype(F32)


def mean22(v):
    """np.mean over the last axis (22 float32 values) in numpy's pairwise order."""
    v = np.asarray(v, F32)
    r = [v[..., j] + v[..., 8 + j] for j in range(8)]
    s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for j in range(16, v.shape[-1]):
        s = s + v[..., j]
    return (s / F32(22)).astype(F32)


def skating(foot, heights, horiz):
    """foot: [n,T,4,3] joints 7,10,8,11; heights [n,T,4] float32 (already relative to the floor); horiz: the 2 horizontal
    axes -> bool [n,T-1]."""
    d = foot[:, 1:][..., horiz] - foot[:, :-1][..., horiz]
    v = (norm2(d) * F32(FPS)).astype(F32)
    h = heights[:, :-1]
    left = (v[..., 0] > F32(0.1)) & (v[..., 1] > F32(0.1)) & (h[..., 0] < F32(0.15)) & (h[..., 1] < F32(0.1))
    right = (v[..., 2] > F32(0.1)) & (v[..., 3] > F32(0.1)) & (h[..., 2] < F32(0.15)) & (h[..., 3] < F32(0.1))
    return left & right


def amass_frames(G, P, label_clean, label_rec):
    """G, P [n,T,22,3]; contact labels [n,T,4] -> the per-frame arrays of eval_amass_full.py and h0 [n]."""
    G, P = np.asarray(G, F32), np.asarray(P, F32)
    h0 = G[..., 2].min(axis=-1).min(axis=-1)  # propagates NaN, as np.min does
    lr = np.asarray(label_rec, F32).copy()
    lr[lr > 0.5] = 1.0
    lr[lr <= 0.5] = 0.0
    hg = (G[:, :, FOOT, 2] - h0[:, None, None]).astype(F32)
    hp = (P[:, :, FOOT, 2] - h0[:, None, None]).astype(F32)
    pd = (P[:, :, [10, 11], 2] - h0[:, None, None]).astype(F32)
    pf = pd < F32(-0.05)
    pd[pd >= 0] = 0
    return {'h0': h0, 'mpjpe': norm3(G - P), 'contact_match': np.asarray(label_clean, F32) == lr,
            'skating_gt': skating(G[:, :, FOOT], hg, [0, 1]), 'skating_rec': skating(P[:, :, FOOT], hp, [0, 1]),
            'accel_error': norm3(accel(P) - accel(G)), 'pene_freq': pf, 'pene_dist': pd}


def amass_metrics(frames, mask_scheme, traj_mask_ratio=0.0):
    """float64 means / ratios of amass_frames' arrays (one batch of equal-length clips)."""
    e = frames['mpjpe'].astype(np.float64)
    T = e.shape[1]
    occ = np.zeros(e.shape, bool)
    if mask_scheme == 'lower':
        occ[:, :, LOWER_OCCLUDED] = True
    else:
        occ[:, 65:65 + int(traj_mask_ratio * 145)] = True
    mean = lambda a: a.sum() / a.size if a.size else np.nan
    return {'mpjpe_global': mean(e), 'mpjpe_global_vis': mean(e[~occ]), 'mpjpe_global_occ': mean(e[occ]),
            'contact_lbl_acc': mean(frames['contact_match']), 'skating_gt_ratio': mean(frames['skating_gt']),
            'skating_rec_ratio': mean(frames['skating_rec']),
            'accel_error': mean(frames['accel_error'].astype(np.float64)),
            'ground_pene_freq': mean(frames['pene_freq']),
            'ground_pene_dist': mean(frames['pene_dist'].astype(np.float64))} if T else {}


def scene_joints(P, transf):
    """eval_prox_egobody.py:178-182: points_coord_trans(x, np.linalg.inv(transf)) per window, float32."""
    out = np.empty_like(np.asarray(P, F32))
    for w in range(out.shape[0]):
        M = np.linalg.inv(np.asarray(transf[w], F32))
        x = np.asarray(P[w], F32).reshape(-1, 3)
        out[w] = (x.dot(M[:3, :3].transpose()) + M[:3, 3].reshape(1, -1)).reshape(out.shape[1:])
    return out


def video_frames(P, transf, dataset, floor, gt=None, mask=None):
    """One recording's windows: P [n,T,22,3] canonical, transf [n,4,4], floor (python float) and, for EgoBody with
    ground truth, gt [n,>=T,22,3] and mask [n,>=T,22] -> the per-window arrays eval_prox_egobody.py keeps."""
    S = scene_joints(P, transf)
    T = S.shape[1]
    up, horiz = (1, [0, 2]) if dataset == 'egobody' else (2, [0, 1])
    fl = F32(floor)
    out = {'skating': skating(S[:, :, FOOT], (S[:, :, FOOT, up] - fl).astype(F32), horiz),
           'acc': mean22(norm3(accel(S)))}
    pd = (S[:, :, [10, 11], up] - fl).astype(F32)
    out['ground_pene_freq'] = (pd < F32(-0.05)).mean(axis=-1)
    pd[pd >= 0] = 0
    out['ground_pene_dist'] = ((pd[..., 0] + pd[..., 1]) / F32(2)).astype(F32)
    if gt is not None:
        g = np.asarray(gt, F32)[:, :T]
        m = np.asarray(mask, F32)[:, :T]
        out['acc_error'] = mean22(norm3(accel(S) - accel(g)))
        out['gmpjpe'] = norm3(g - S)
        out['mpjpe'] = norm3((g - g[:, :, [0]]) - (S - S[:, :, [0]]))
        out['mpjpe_vis'] = (out['mpjpe'] * m).astype(F32)
        out['mpjpe_occ'] = (out['mpjpe'] * (F32(1) - m)).astype(F32)
        out['joint_mask'] = m
    return out


def video_metrics(per_recording):
    """per_recording: video_frames dicts in order -> ('all' metrics as float64 means, per-recording metrics).  An empty
    recording gives NaN."""
    def metrics(frames):
        cat = lambda k: (np.concatenate([f[k] for f in frames]).astype(np.float64) if frames and k in frames[0]
                         else np.zeros(0))
        mean = lambda a: a.sum() / a.size if a.size else np.nan
        out = {'skating': mean(cat('skating')), 'acc': mean(cat('acc')), 'ground_pene_freq': mean(cat('ground_pene_freq')),
               'ground_pene_dist': mean(cat('ground_pene_dist'))}
        if frames and 'gmpjpe' in frames[0]:
            m = cat('joint_mask')
            out.update(acc_error=mean(cat('acc_error')), gmpjpe=mean(cat('gmpjpe')), mpjpe=mean(cat('mpjpe')),
                       mpjpe_vis=cat('mpjpe_vis').sum() / m.sum(), mpjpe_occ=cat('mpjpe_occ').sum() / (1 - m).sum())
        return out
    return metrics([f for f in per_recording if f is not None]), [metrics([f] if f is not None else [])
                                                                   for f in per_recording]
