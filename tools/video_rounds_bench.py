"""Windows per second of the PROX / EgoBody video driver's rounds on the device (pipeline.run_video_rounds, then
reconstruct_video_outputs) in the shipped video configuration: 2 rounds, a 100-step TrajNet / TrajControl, 980 guided
PoseNet steps of the 1000-step schedule (early_stop, grad_type 'prox'), iter2_cond_noisy_traj / iter2_cond_noisy_pose False.

    python tools/video_rounds_bench.py [--rounds R] [--recordings N] [--frames F] [--json PATH]

Inputs: N synthetic PROX recordings of F frames (default 6 x 3000, 20 windows of 145 frames each) encoded by
windows.encode_video, synthetic weights.  Two cases:
  (a) the reference driver's batch: the 20 windows of one recording per call, every recording in turn;
  (b) every window of every recording in one call.
After one warm-up of each case, the two are timed alternately --rounds times (CUDA events around whole calls, including
the batch encoding and the reconstruction), and the median is reported as windows per second.  Prints the card, its
power limit and SM clocks read in the same run, then one JSON line.  Needs an H100; writes nothing unless --json is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rohm_b200 import diffusion, pipeline, synthetic, windows  # noqa: E402
from rohm_b200.body_model import BodyModel  # noqa: E402
from rohm_b200.posenet import PoseNet  # noqa: E402
from rohm_b200.trajnet import TrajNet  # noqa: E402

REFERENCE_BATCH = 20  # the reference video driver's batch_size (cfg_files/test_cfg/prox_rgb.yaml)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def recordings(n_rec, frames, dev):
    """Camera-frame SMPL-X fits of walking bodies 4.4 m in front of the camera, OpenPose-like keypoints and depth masks,
    one camera per recording."""
    g = np.random.default_rng(7)
    t = np.arange(frames, dtype=np.float64)
    params = {k: [] for k in ("global_orient", "transl", "betas", "body_pose")}
    for r in range(n_rec):
        yaw = np.pi * np.sin(t / 300.0 + r) + 0.3 * np.sin(t / 23.0)
        params["global_orient"].append(np.stack([0.05 * np.sin(t / 11.0), 0.04 * np.cos(t / 17.0), yaw], -1))
        params["transl"].append(np.stack([2.0 * np.sin(t / 250.0), 2.0 * np.cos(t / 310.0), 4.4 + 0.03 * np.sin(t / 9.0)], -1))
        params["betas"].append(np.repeat(0.5 * g.standard_normal((1, 10)), frames, axis=0))
        params["body_pose"].append(0.15 * g.standard_normal((1, 63)) + 0.1 * np.sin(t[:, None] / 15.0 + np.arange(63)))
    params = {k: torch.from_numpy(np.concatenate(v).astype(np.float32)).to(dev) for k, v in params.items()}
    N = n_rec * frames
    c2w = np.repeat(np.eye(4)[None], n_rec, 0)
    for r in range(n_rec):
        a = 0.7 + r
        c2w[r, :3, :3] = [[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]]
        c2w[r, :3, 3] = [0.3 * r, -1.2, 2.0 + 0.1 * r]
    kp = np.concatenate([g.uniform(0, 1920, (N, 25, 1)), g.uniform(0, 1080, (N, 25, 1)), g.uniform(0, 1, (N, 25, 1))],
                        -1).astype(np.float32)
    depth = (g.uniform(0, 1, (N, 25)) > 0.1).astype(np.float32)
    K = np.array([[1060.53, 0.0, 951.3], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]])
    cams = dict(cam2world=c2w, focal_length=np.repeat([[1060.53, 1060.38]], n_rec, 0),
                camera_center=np.repeat([[951.3, 536.77]], n_rec, 0), camera_mtx=np.repeat(K[None], n_rec, 0),
                dist=np.repeat([[0.0548, -0.0489, 0.0009, -0.0012, 0.0102]], n_rec, 0))
    return params, torch.from_numpy(kp).to(dev), torch.from_numpy(depth).to(dev), cams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--recordings", type=int, default=6)
    ap.add_argument("--frames", type=int, default=3000)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("video_rounds_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    c = card()
    print(f"card: {c} (name, power limit, SM clock, max SM clock)", flush=True)
    ds_p = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_t = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    mp = PoseNet(dataset=ds_p, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, device=dev,
                 traj_feat_dim=22)
    mp.load_state_dict(synthetic.synth_state_dict(mp, 1))
    mk = lambda ctl: TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=ctl, device=dev,
                                   dataset=ds_t, repr_abs_only=True)
    mt, mc = mk(False), mk(True)
    mt.load_state_dict(synthetic.synth_state_dict(mt, 2))
    mc.load_state_dict(synthetic.synth_state_dict(mc, 4))
    mp, mt, mc = mp.to(dev).eval(), mt.to(dev).eval(), mc.to(dev).eval()
    body = BodyModel.create('', device=dev, seed=0)
    da = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    dp = diffusion.create_gaussian_diffusion(da, diffusion, diffusion.SpacedDiffusionPoseNet, 1000, '', dev)
    dt = diffusion.create_gaussian_diffusion(da, diffusion, diffusion.SpacedDiffusionTrajNet, 100, '', dev)
    dc = diffusion.create_gaussian_diffusion(da, diffusion, diffusion.SpacedDiffusionTrajNet, 100, '', dev)
    args = pipeline.make_args(sample_iter=2, iter2_cond_noisy_traj=False, iter2_cond_noisy_pose=False, early_stop=True)
    params, kp, depth, cams = recordings(a.recordings, a.frames, dev)
    lengths = [a.frames] * a.recordings
    per_rec = windows.window_table([a.frames])
    W = len(per_rec) * a.recordings
    off = np.concatenate([[0], np.cumsum(lengths)])

    def encode(recs):
        rows = np.concatenate([np.arange(off[r], off[r + 1]) for r in recs])
        idx = torch.from_numpy(rows).to(dev)
        sel = lambda v: v[recs]
        return windows.encode_video(body, {k: v[idx] for k, v in params.items()}, [lengths[r] for r in recs], 'prox',
                                    keypoints=kp[idx], depth_mask=depth[idx], pose_dataset=ds_p, traj_dataset=ds_t,
                                    **{k: sel(v) for k, v in cams.items()})

    def call(recs):
        bt, bp, _ = encode(recs)
        vp, _ = pipeline.run_video_rounds(args, mp, mt, mc, dp, dt, dc, ds_p, ds_t, body, bp, bt)
        return pipeline.reconstruct_video_outputs(ds_p, body, bp, vp)

    def case_a():  # one recording's windows per call, as the reference driver batches them
        for r in range(a.recordings):
            call([r])

    def case_b():
        call(list(range(a.recordings)))

    if len(per_rec) > REFERENCE_BATCH:
        raise SystemExit(f"video_rounds_bench: a recording of {a.frames} frames has {len(per_rec)} windows, more than "
                         f"the reference's batch of {REFERENCE_BATCH}")

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3

    for fn in (case_a, case_b):  # warm-up: engines, graphs and body-model buffers of both batch sizes
        fn()
    times = {"a": [], "b": []}
    for _ in range(a.rounds):
        times["a"].append(timed(case_a))
        times["b"].append(timed(case_b))
        print(f"round: (a) {times['a'][-1]:.2f} s, (b) {times['b'][-1]:.2f} s for {W} windows", flush=True)
    ta, tb = statistics.median(times["a"]), statistics.median(times["b"])
    res = {"card": c, "windows": W, "recordings": a.recordings, "frames": a.frames, "rounds": a.rounds,
           "a_windows_per_call": len(per_rec), "a_s": ta, "b_s": tb, "a_windows_per_s": W / ta, "b_windows_per_s": W / tb,
           "b_over_a": ta / tb, "a_all_s": times["a"], "b_all_s": times["b"]}
    print(f"(a) {len(per_rec)} windows per call: {W / ta:.3f} windows/s | (b) {W} windows in one call: {W / tb:.3f} "
          f"windows/s | (b)/(a) x{ta / tb:.2f}", flush=True)
    print(json.dumps(res), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
