"""Long-clip measurement of the TrajNet engine (fp16 pairs, RoHM's configuration: mid_dim 512) and the round pipeline.

    python tools/long_traj_bench.py [--iters N] [--reps N] [--json PATH]

Prints the card and its power limit, then
  * per clip length T: B ~ 9216 / T clips (the token count of the trajcontrol benchmark's 64 x 144), the forward graph's
    time of TrajNet and of TrajNet+TrajControl (CUDA events over --iters replays), and the GroupNorm kernel's share of
    one forward from a separate torch.profiler run with graphs off;
  * the GroupNorm kernel alone at 1 clip x 4992 frames on the widest level (64 channels, 8 groups of 8, one partial plus
    the time projection) through the kernel test probe (tests/native/libkernel_probe.so), CUDA events
    around --reps back-to-back launches: one CTA per group (the shared-memory attribute raised), the size the engine chooses,
    and clusters of 8;
  * one 2-round pipeline.run_rounds at 1 clip x 4993 raw frames (TrajNet 4992 frames, 100 steps; PoseNet 4991 frames,
    50 respaced steps, guided), host clock around a synchronised run after a warm-up run, and the same at 145 raw frames;
    each reports which stages of which round are finite.
Needs an H100; writes nothing unless --json is given."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from rohm_b200 import synthetic  # noqa: E402
from rohm_b200.trajnet import TrajNet  # noqa: E402

MID = 512
CLIP_T = [144, 512, 1008, 1520, 1536, 2000, 4992]
FRAMES = 9216
GN_T, GN_C = 4992, 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def time_ms(fn, iters):
    """Mean device time of fn() over iters calls (CUDA events around the whole window)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def build(control, dev):
    m = TrajNet(time_dim=32, mid_dim=MID, cond_dim=13, traj_feat_dim=13, trajcontrol=control, device=dev,
                dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
    m.load_state_dict(synthetic.synth_state_dict(m, 2))
    return m.to(dev).eval()


def gn_share(m, batch, ts):
    """GroupNorm kernel time / all kernel time of one forward launched kernel by kernel (graphs off) under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    eng = m._engine
    eng.lib.rohm_trajnet_set_option(eng.handle, 0, 0)
    try:
        m(batch, ts)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m(batch, ts)
            torch.cuda.synchronize()
    finally:
        eng.lib.rohm_trajnet_set_option(eng.handle, 0, 1)
    gn = total = 0.0
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", 0.0)
        if e.device_type != torch.autograd.DeviceType.CUDA or t <= 0:
            continue
        total += t
        if "gn_mish_split_kernel" in e.key:
            gn += t
    return gn / 1e3, total / 1e3


def clip_lengths(dev, iters):
    nets = {c: build(c, dev) for c in (False, True)}
    rows = []
    for T in CLIP_T:
        B = max(1, round(FRAMES / T))
        r = {"T": T, "B": B}
        for control, m in nets.items():
            name = "trajcontrol" if control else "trajnet"
            g = torch.Generator().manual_seed(T)
            batch = {k: v.to(dev) for k, v in synthetic.trajnet_batch(B, T, 5, control=control).items()}
            batch['x_t'] = torch.randn(B, T, 13, generator=g).to(dev)
            ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
            for _ in range(3):  # engine, condition pyramid, graph capture
                m(batch, ts)
            torch.cuda.synchronize()
            ms = time_ms(lambda: m(batch, ts), iters)
            gn_ms, prof_ms = gn_share(m, batch, ts)
            r.update({f"{name}_forward_ms": ms, f"{name}_clip_forwards_per_s": B / ms * 1e3, f"{name}_gn_ms_profiled": gn_ms,
                      f"{name}_kernel_ms_profiled": prof_ms, f"{name}_gn_share": gn_ms / prof_ms})
            print(f"T={T:5d} B={B:3d} {name:11s}: forward {ms:8.3f} ms ({B / ms * 1e3:8.1f} clip forwards/s) | GroupNorm "
                  f"{gn_ms:7.3f} of {prof_ms:7.3f} ms of kernels ({100 * gn_ms / prof_ms:4.1f} %)", flush=True)
            m._engine = None
        rows.append(r)
    return rows


def group_norm_kernel(dev, reps):
    import kernel_probe as kp
    B, G = 1, 8
    Tp = GN_T + 32
    rows = B * Tp
    g = torch.Generator().manual_seed(1)
    rnd = lambda *s: torch.randn(*s, generator=g).to(dev)
    part, bias, gamma, beta, tp = rnd(rows * GN_C), rnd(GN_C), rnd(GN_C), rnd(GN_C), rnd(B, GN_C)
    hi = torch.empty(rows * GN_C, device=dev, dtype=torch.float16)
    lo = torch.empty_like(hi)
    slice_bytes = lambda n: -(-GN_T // n) * (GN_C // G) * 4
    chosen = kp.group_norm_cluster(GN_T, GN_C, G)
    res = []
    for label, n in (("one CTA per group", 1), ("chosen", chosen), ("clusters of 8", 8)):
        call = lambda k=reps: kp.group_norm(part, 1, rows * GN_C, bias, gamma, beta, tp, GN_C, None, None, None, hi, lo,
                                            GN_C, Tp, GN_T, B, n, 1, reps=k)
        assert call(5) == 0, n
        torch.cuda.synchronize()
        us = time_ms(call, 1) / reps * 1e3
        gbs = (GN_T * GN_C * 4 * 1 + GN_T * GN_C * 2 * 2) / (us * 1e-6) / 1e9  # one fp32 partial in, an fp16 pair out
        print(f"GroupNorm 1 x {GN_T} frames, {GN_C} channels, n={n} ({label}, {slice_bytes(n)} B of shared memory per "
              f"CTA): {us:8.2f} us ({gbs:6.1f} GB/s)", flush=True)
        res.append({"n": n, "label": label, "us": us, "gb_per_s": gbs})
    return res


def run_rounds(dev):
    import argparse as ap_
    from rohm_b200 import diffusion, pipeline
    from rohm_b200.body_model import BodyModel
    from rohm_b200.posenet import PoseNet
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    mp = PoseNet(dataset=ds_pose, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, device=dev,
                 traj_feat_dim=22)
    mp.load_state_dict(synthetic.synth_state_dict(mp, 1))
    mp = mp.to(dev).eval()
    mk = lambda c: TrajNet(time_dim=32, mid_dim=MID, cond_dim=13, traj_feat_dim=13, trajcontrol=c, device=dev,
                           dataset=ds_traj, repr_abs_only=True)
    mt, mc = mk(False), mk(True)
    mt.load_state_dict(synthetic.synth_state_dict(mt, 2))
    mc.load_state_dict(synthetic.synth_state_dict(mc, 4))
    mt, mc = mt.to(dev).eval(), mc.to(dev).eval()
    body = BodyModel.create('', device=dev, seed=0)
    a = ap_.Namespace(noise_schedule='cosine', sigma_small=True)
    dp = diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionPoseNet, 1000, 'ddim50', dev)
    dt = diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionTrajNet, 100, '', dev)
    dc = diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionTrajNet, 100, '', dev)
    args = pipeline.make_args(sample_iter=2, mask_scheme='lower')
    B = 1
    finite = []

    def on_round(it, val_traj, traj_full, cond, val_pose):  # which stage of which round stays finite
        finite.append({k: bool(torch.isfinite(v).all()) for k, v in (("val_traj", val_traj), ("traj_full", traj_full),
                                                                       ("val_pose", val_pose))})

    def once(frames):
        pose, traj = synthetic.pipeline_batches(B, 7, ds_pose, frames=frames, device=dev)
        finite.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipeline.run_rounds(args, mp, mt, mc, dp, dt, dc, ds_pose, ds_traj, body, pose, traj, on_round=on_round)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    res = []
    for frames in (144, 4992):  # the benchmark's clip length beside the longest, with the same settings
        once(frames)  # engines, graphs
        s = once(frames)
        print(f"run_rounds 1 x {frames + 1} raw frames, 2 rounds (TrajNet 100 steps, PoseNet 50 steps): {s:.3f} s; "
              f"finite per round: {finite}", flush=True)
        res.append({"frames_raw": frames + 1, "rounds": 2, "seconds": s, "finite": list(finite)})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_traj_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    c = card()
    print(f"card: {c} (name, power limit, max SM clock)", flush=True)
    res = {"card": c, "group_norm": group_norm_kernel(dev, a.reps), "clips": clip_lengths(dev, a.iters),
           "run_rounds": run_rounds(dev)}
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
