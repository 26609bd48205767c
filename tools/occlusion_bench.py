"""Times rohm_b200.occlusion on the device beside the numpy restatement (oracle/occlusion_oracle.py) on one CPU thread:
scene_depth of a synthetic scene of about 1M triangles at 1920x1080 (mostly few-pixel triangles, a few hundred beyond
the large-box threshold, a floor and walls), and joint_mask over 3000 frames of the synthetic SMPL-X-shaped body
(20 908 triangles; LBS included).  Device times are CUDA events around whole calls, median of --iters after --warmup;
the oracle runs on a subset (--oracle_tris triangles of the scene, --oracle_frames frames) and is scaled per item.
Prints one JSON line with the GPU's name and power limit.

    python tools/occlusion_bench.py [--iters 10] [--warmup 2]
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

from oracle import occlusion_oracle as oo  # noqa: E402
from rohm_b200 import occlusion, synthetic  # noqa: E402
from rohm_b200.body_model import BodyModel  # noqa: E402


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


def big_scene(n, seed=0):
    """n camera-facing triangles in the camera frame (identity cam2world): 99.9 % of 1-4 pixels, the rest of 40-400
    pixels across, plus a floor and two walls."""
    g = np.random.default_rng(seed)
    fx, fy, cx, cy = occlusion.PROX_RENDER_INTRINSICS
    W, H = occlusion.RENDER_SIZE
    size = np.where(g.uniform(size=n) < 0.999, g.uniform(1, 4, n), g.uniform(40, 400, n))
    c = np.stack([g.uniform(0, W, n), g.uniform(0, H, n)], -1)
    pts = c[:, None, :] + g.normal(0, 1, (n, 3, 2)) * size[:, None, None]
    z = g.uniform(1.0, 8.0, (n, 1)) + g.normal(0, 0.02, (n, 3))
    tri = np.stack([(pts[..., 0] - cx) / fx * z, (pts[..., 1] - cy) / fy * z, z], -1)
    big = np.array([[[-30, 1.2, 0.3], [30, 1.2, 60], [30, 1.2, 0.3]], [[-30, 1.2, 0.3], [-30, 1.2, 60], [30, 1.2, 60]],
                    [[-40, -30, 9], [40, 30, 9], [40, -30, 9]], [[-40, -30, 9], [-40, 30, 9], [40, 30, 9]]])
    tri = np.concatenate([tri, big])
    V = tri.reshape(-1, 3).astype(np.float32)
    F = np.arange(len(V)).reshape(-1, 3)
    a, b, d = (V[F[:, i]].astype(np.float64) for i in range(3))
    back = (np.cross(b - a, d - a) * a).sum(1) > 0
    F[back] = F[back][:, [0, 2, 1]]
    return V, F


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--triangles", type=int, default=1_000_000)
    ap.add_argument("--frames", type=int, default=3000)
    ap.add_argument("--oracle_tris", type=int, default=20_000)
    ap.add_argument("--oracle_frames", type=int, default=20)
    args = ap.parse_args()
    torch.set_num_threads(1)
    dev = torch.device("cuda:0")
    out = {"gpu": gpu_info()}

    V, F = big_scene(args.triangles)
    Vd, Fd = torch.from_numpy(V).to(dev), torch.from_numpy(F).to(dev)
    eye = np.eye(4)
    depth = occlusion.scene_depth(Vd, Fd, eye)
    out["scene_triangles"] = int(len(F))
    out["scene_depth_ms"] = timed(lambda: occlusion.scene_depth(Vd, Fd, eye), args.iters, args.warmup)
    out["scene_drawn_fraction"] = float((depth > 0).float().mean())
    sub = F[:args.oracle_tris]
    t0 = time.perf_counter()
    oo.scene_depth(V, sub, eye[:3], occlusion.PROX_RENDER_INTRINSICS, occlusion.RENDER_SIZE)
    out["oracle_scene_s_per_1M_triangles"] = (time.perf_counter() - t0) * 1e6 / len(sub)

    model = BodyModel.create('', device=dev, seed=0)
    faces = synthetic.smplx_like_faces(0)
    N = args.frames
    g = np.random.default_rng(1)
    p = {'global_orient': 0.3 * g.standard_normal((N, 3)), 'body_pose': 0.15 * g.standard_normal((N, 63)),
         'betas': 0.5 * g.standard_normal((N, 10)),
         'transl': np.stack([g.uniform(-0.8, 0.8, N), g.uniform(-0.4, 0.2, N), g.uniform(2.0, 4.0, N)], -1)}
    p = {k: torch.from_numpy(v.astype(np.float32)).to(dev) for k, v in p.items()}
    maps = depth[None].contiguous()
    K = np.array([[[1060.53, 0.0, 951.30], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]]])
    k = np.array([[0.0437, -0.0597, -0.0011, 0.0007, 0.0210]])
    mask = occlusion.joint_mask(model, faces, p, (N,), maps, [0], K, k)
    ms = timed(lambda: occlusion.joint_mask(model, faces, p, (N,), maps, [0], K, k), args.iters, args.warmup)
    out["mask_frames"] = N
    out["lbs_and_mask_ms"] = ms
    out["lbs_and_mask_us_per_frame"] = ms * 1e3 / N
    out["occluded_fraction"] = float((mask == 0).float().mean())
    n = args.oracle_frames
    body = model(**{a: b[:n] for a, b in p.items()}, return_verts=True)
    t0 = time.perf_counter()
    oo.joint_occlusion(body.joints.cpu().numpy(), body.vertices.cpu().numpy(), faces, np.zeros(n, int), K, k,
                       maps.cpu().numpy(), [0], occlusion.PROX_RENDER_INTRINSICS, occlusion.RENDER_SIZE)
    out["oracle_mask_ms_per_frame"] = (time.perf_counter() - t0) * 1e3 / n
    print(json.dumps(out))


if __name__ == "__main__":
    main()
