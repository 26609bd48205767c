"""Times rohm_b200.metrics on the device beside the numpy restatement (oracle/metrics_oracle.py) on one CPU thread:
metrics.amass over 2048 clips of 143 frames ('lower') and the video pass over 400 windows of 143 frames from 20 EgoBody
recordings with ground truth.  Device times are CUDA events around whole calls (kernels, the small host reads of the
sums and the Python around them), median of --iters after --warmup; prints one JSON line with the GPU's name and power
limit.

    python tools/eval_metrics_bench.py [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import metrics_oracle as mo  # noqa: E402
from rohm_b200 import metrics  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "?"
    except (OSError, subprocess.SubprocessError):
        return "?"


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    g = np.random.default_rng(0)
    B, T = 2048, 143
    G = g.normal(0, 0.5, (B, T, 22, 3)).astype(np.float32)
    P = (G + g.normal(0, 0.03, G.shape)).astype(np.float32)
    lc = (g.uniform(0, 1, (B, T, 4)) > 0.5).astype(np.float32)
    lr = g.uniform(0, 1, (B, T, 4)).astype(np.float32)
    rc, rr = np.zeros((B, T, 294), np.float32), np.zeros((B, T, 294), np.float32)
    rc[..., -4:], rr[..., -4:] = lc, lr
    out = {'rec_ric_data_clean': torch.from_numpy(G).to(dev), 'rec_ric_data_rec_from_smpl': torch.from_numpy(P).to(dev),
           'motion_repr_clean': torch.from_numpy(rc).to(dev), 'motion_repr_rec': torch.from_numpy(rr).to(dev)}
    amass_ms = timed(lambda: metrics.amass(out, 'lower'), args.iters, args.warmup)
    t0 = time.perf_counter()
    mo.amass_metrics(mo.amass_frames(G, P, lc, lr), 'lower')
    amass_cpu_ms = (time.perf_counter() - t0) * 1e3

    R, per = 20, 20
    payloads, floors = [], g.uniform(-1.5, -0.5, R)
    for r in range(R):
        rec = g.normal(0, 0.5, (per, T, 22, 3)).astype(np.float32)
        tf = np.repeat(np.eye(4, dtype=np.float32)[None], per, 0)
        tf[:, :3, 3] = g.normal(0, 1, (per, 3))
        payloads.append({'rec_ric_data_rec_list_from_smpl': rec, 'trans_scene2cano_list': tf,
                         'joints_gt_scene_coord_list': (g.normal(0, 0.5, (per, T + 2, 22, 3))).astype(np.float32),
                         'mask_joint_vis_list': (g.uniform(0, 1, (per, T, 22)) > 0.3).astype(np.float32)})
    # device-resident inputs, as metrics.video sees them after the rounds
    up = lambda k, cut=None: torch.from_numpy(np.concatenate([p[k][:, :cut] if cut else p[k] for p in payloads])).to(dev)
    rec, tf, gt, mask = (up('rec_ric_data_rec_list_from_smpl'), up('trans_scene2cano_list'),
                         up('joints_gt_scene_coord_list'), up('mask_joint_vis_list'))
    win_rec = torch.arange(R, dtype=torch.int32, device=dev).repeat_interleave(per)
    order = torch.arange(R * per, dtype=torch.int32, device=dev)
    video_ms = timed(lambda: metrics._video(rec, tf, gt, mask, win_rec, order, [per] * R, 'egobody', floors),
                     args.iters, args.warmup)
    t0 = time.perf_counter()
    mo.video_metrics([mo.video_frames(p['rec_ric_data_rec_list_from_smpl'], p['trans_scene2cano_list'], 'egobody',
                                      float(floors[r]), p['joints_gt_scene_coord_list'], p['mask_joint_vis_list'])
                      for r, p in enumerate(payloads)])
    video_cpu_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": gpu_info(),
                      "amass_clips": B, "amass_device_ms": round(amass_ms, 4), "amass_numpy_1thread_ms": round(amass_cpu_ms, 1),
                      "video_windows": R * per, "video_recordings": R, "video_device_ms": round(video_ms, 4),
                      "video_numpy_1thread_ms": round(video_cpu_ms, 1)}))


if __name__ == "__main__":
    main()
