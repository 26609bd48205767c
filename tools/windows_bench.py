"""Cost of sliding-window batching: rohm_b200.windows.encode (SMPL-X FK of every frame, then the window encoder) and
encode_joints (the encoder alone), encode with input noise (noise_given: preset noise tensors; noise_drawn: one CUDA
generator per window, the draws included; both add the noise kernel, FK of the W x 145 noisy rows and the canonical
encoder), and to_recordings, on R recordings of N frames cut into 145-frame windows with overlap 2.

    python tools/windows_bench.py [--recordings R] [--frames N] [--iters K] [--rounds M] [--oracle-windows V] [--json PATH]
    python tools/windows_bench.py --video [...]   # encode_video (PROX: camera map, undistorted keypoints, masks) vs encode

Each call is timed with CUDA events around --iters calls after warm-up calls; the median over --rounds is reported as
windows per second.  Next to it, the float64 CPU oracle's time per window (oracle/windows_oracle.py, one thread, over
--oracle-windows windows), labelled as the oracle: it restates the reference's per-clip numpy path, it is not the
reference.  Prints the card, its power limit and SM clocks read in the same run, then one JSON line.  Needs an H100;
writes nothing unless --json is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import windows_noise_oracle, windows_oracle, windows_video_oracle  # noqa: E402
from rohm_b200 import synthetic, windows  # noqa: E402
from rohm_b200.body_model import BodyModel  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def recordings(R, N, seed=0):
    g = np.random.default_rng(seed)
    t = np.arange(N, dtype=np.float64)
    out = {k: [] for k, _ in windows.PARAMS}
    for r in range(R):
        yaw = np.pi * np.sin(t / 300.0 + r) + 0.3 * np.sin(t / 23.0)
        out['global_orient'].append(np.stack([0.05 * np.sin(t / 11.0), 0.04 * np.cos(t / 17.0), yaw], -1))
        out['transl'].append(np.stack([2.0 * np.sin(t / 250.0), 2.0 * np.cos(t / 310.0) + r, 0.9 + 0.03 * np.sin(t / 9.0)], -1))
        out['betas'].append(np.repeat(0.5 * g.standard_normal((1, 10)), N, axis=0))
        out['body_pose'].append(0.15 * g.standard_normal((1, 63)) + 0.1 * np.sin(t[:, None] / 15.0 + np.arange(63)))
    return {k: np.concatenate(v).astype(np.float32) for k, v in out.items()}


def time_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recordings", type=int, default=20)
    ap.add_argument("--frames", type=int, default=3000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--oracle-windows", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--video", action="store_true", help="encode_video against encode, alternated per round")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = card()
    print("card, power limit, SM clock, max SM clock:", info)
    if a.video:
        return video(a, dev, info)
    ds_p, ds_t = synthetic.make_dataset('pose', seed=3, realistic_std=True), synthetic.make_dataset('traj', seed=3, realistic_std=True)
    bm = BodyModel.create('', device=dev, seed=0)
    host = recordings(a.recordings, a.frames)
    params = {k: torch.from_numpy(v).to(dev) for k, v in host.items()}
    lengths = [a.frames] * a.recordings
    joints = bm(**params, return_verts=False).joints[:, 0:22].contiguous()
    _, pose, win = windows.encode(bm, params, lengths, ds_p, ds_t)
    W = len(win)
    cano = torch.randn(W, 143, 22, 3, device=dev)
    g = torch.Generator(device=dev).manual_seed(1)
    level3 = {'transl': (0.03, (3,)), 'betas': (0.1, (10,)), 'global_orient': (3.0, (3,)), 'body_pose': (3.0, (21, 3))}
    n = {k: s * torch.randn((W, 145) + shape, generator=g, device=dev) for k, (s, shape) in level3.items()}
    given = windows.InputNoise.given(n['transl'], n['betas'], n['global_orient'], n['body_pose'])
    gens = [torch.Generator(device=dev).manual_seed(100 + w) for w in range(W)]
    calls = {"encode": lambda: windows.encode(bm, params, lengths, ds_p, ds_t),
             "encode_joints": lambda: windows.encode_joints(params, joints, lengths, ds_p, ds_t),
             "noise_given": lambda: windows.encode(bm, params, lengths, ds_p, ds_t, noise=given),
             "noise_drawn": lambda: windows.encode(bm, params, lengths, ds_p, ds_t, noise=windows.InputNoise.drawn(gens)),
             "to_recordings": lambda: windows.to_recordings(win, cano)}
    ms = {k: [] for k in calls}
    for _ in range(a.rounds):
        for k, fn in calls.items():
            ms[k].append(time_ms(fn, a.iters))
    res = {k: {"ms": statistics.median(v), "windows_per_s": W / (statistics.median(v) / 1e3)} for k, v in ms.items()}
    for k, v in res.items():
        print(f"{k:14s} {W} windows: {v['ms']:.3f} ms  ({v['windows_per_s']:.0f} windows/s)")
    # the float64 CPU oracle on the first windows, one thread
    torch.set_num_threads(1)
    jh = joints.cpu().numpy()
    table = windows.window_table(lengths)[:a.oracle_windows]
    t0 = time.perf_counter()
    for r, s in table:
        rows = slice(r * a.frames + s, r * a.frames + s + 145)
        m = windows_oracle.canonical_frame(jh[rows])
        windows_oracle.encode_window(jh[rows], host['global_orient'][rows], host['transl'][rows], host['betas'][rows],
                                     host['body_pose'][rows], m)
    oracle_ms = (time.perf_counter() - t0) * 1e3 / len(table)
    print(f"oracle (float64 numpy, CPU, 1 thread): {oracle_ms:.3f} ms per window")
    # the noisy path on the first recording's windows
    W0 = len(windows.window_table([a.frames]))
    nh = {k: v[:W0].cpu().numpy() for k, v in n.items()}
    model = synthetic.smplx_like_model(0)
    t0 = time.perf_counter()
    windows_noise_oracle.encode_noisy({k: v[:a.frames] for k, v in host.items()}, jh[:a.frames], [a.frames], nh, model)
    noisy_ms = (time.perf_counter() - t0) * 1e3 / W0
    print(f"oracle noisy path (float64, CPU, 1 thread): {noisy_ms:.3f} ms per window")
    line = {"card": info, "recordings": a.recordings, "frames": a.frames, "windows": W, **{k: v for k, v in res.items()},
            "oracle_cpu_ms_per_window": oracle_ms, "oracle_noisy_cpu_ms_per_window": noisy_ms}
    print(json.dumps(line))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(line, f, indent=1)


def video(a, dev, info):
    """encode_video on PROX-like recordings (a rotated camera, Kinect-like distortion, keypoints over the image) against
    encode on the same parameters; each call's host work is inside the timed region."""
    ds_p, ds_t = synthetic.make_dataset('pose', seed=3, realistic_std=True), synthetic.make_dataset('traj', seed=3, realistic_std=True)
    bm = BodyModel.create('', device=dev, seed=0)
    host = recordings(a.recordings, a.frames)
    params = {k: torch.from_numpy(v).to(dev) for k, v in host.items()}
    R, N = a.recordings, a.recordings * a.frames
    lengths = [a.frames] * R
    g = np.random.default_rng(2)
    c2w = np.repeat(np.eye(4)[None], R, 0)
    c2w[:, :3, :3] = np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]])
    c2w[:, :3, 3] = g.uniform(-1, 1, (R, 3))
    K = np.array([[1060.5, 0.0, 951.3], [0.0, 1060.4, 536.8], [0.0, 0.0, 1.0]])
    kp = np.concatenate([g.uniform(0, 1920, (N, 25, 1)), g.uniform(0, 1080, (N, 25, 1)), g.uniform(0, 1, (N, 25, 1))], -1)
    cam = dict(cam2world=c2w, focal_length=np.repeat([[1060.5, 1060.4]], R, 0), camera_center=np.repeat([[951.3, 536.8]], R, 0),
               camera_mtx=np.repeat(K[None], R, 0), dist=np.repeat([[0.0548, -0.0489, 0.0009, -0.0012, 0.0102]], R, 0),
               keypoints=torch.from_numpy(kp.astype(np.float32)).to(dev),
               depth_mask=torch.from_numpy((g.uniform(0, 1, (N, 25)) > 0.1).astype(np.float32)).to(dev),
               keypoints_float64=[False] * R)
    calls = {"encode_video": lambda: windows.encode_video(bm, params, lengths, 'prox', pose_dataset=ds_p, traj_dataset=ds_t,
                                                          **cam),
             "encode": lambda: windows.encode(bm, params, lengths, ds_p, ds_t)}
    W = len(windows.window_table(lengths))
    ms = {k: [] for k in calls}
    for _ in range(a.rounds):
        for k, fn in calls.items():
            ms[k].append(time_ms(fn, a.iters))
    res = {k: {"ms": statistics.median(v), "windows_per_s": W / (statistics.median(v) / 1e3)} for k, v in ms.items()}
    for k, v in res.items():
        print(f"{k:14s} {W} windows: {v['ms']:.3f} ms  ({v['windows_per_s']:.0f} windows/s)")
    torch.set_num_threads(1)
    jh = bm(**params, return_verts=False).joints[:, 0:22].cpu().numpy()
    table = windows.window_table(lengths)[:a.oracle_windows]
    t0 = time.perf_counter()
    for r, s in table:
        rows = slice(r * a.frames + s, r * a.frames + s + 145)
        windows_video_oracle.encode_window_video(jh[rows], {k: v[rows] for k, v in host.items()}, c2w[r], False)
        windows_video_oracle.keypoints_window(kp[rows].astype(np.float32), np.ones((145, 25)), True, K,
                                              cam['dist'][r], False)
    oracle_ms = (time.perf_counter() - t0) * 1e3 / len(table)
    print(f"oracle video path (float64 numpy, CPU, 1 thread): {oracle_ms:.3f} ms per window")
    line = {"card": info, "recordings": R, "frames": a.frames, "windows": W, **res,
            "oracle_video_cpu_ms_per_window": oracle_ms}
    print(json.dumps(line))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
