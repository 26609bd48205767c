"""Cost of per-clip noise streams (batch['generators']) against the single torch-generator stream.

    python tools/noise_streams_bench.py [--iters N] [--json PATH]

Three measurements, each alternating the two variants in the same process (single stream first, then per-clip, repeated
--rounds times; the median of the rounds is reported):
  (1) the update kernel alone over --iters back-to-back launches (CUDA events around the window): ddpm_step_philox_kernel
      (rohm_ddpm_step_philox) against clip_noise_kernel<true> (rohm_ddpm_step_philox_clips), for PoseNet 32 x 144 frames,
      TrajNet 64 x 144 frames x 13 channels and the 8-recording PoseNet mix of tools/ragged_bench.py (lengths given);
  (2) the fused PoseNet step graph (forward + update as one replay, 32 x 144) with and without per-clip streams;
  (3) clips/s of a 100-step respaced PoseNet p_sample_loop (32 x 144, RoHM's configuration) with and without
      generators: host clock around the loop, ended by a device synchronise, so the host cost of the streams shows.
Prints the card, its power limit and maximum SM clock from the same run, then one JSON line.  Needs an H100; writes
nothing unless --json is given."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ragged_bench import LENGTHS, card, time_ms  # noqa: E402
from rohm_b200 import diffusion, ops, synthetic  # noqa: E402
from rohm_b200.noise_streams import NoiseStreams  # noqa: E402
from rohm_b200.posenet import PoseNet  # noqa: E402


def gens(dev, B, seed=0):
    return [torch.Generator(device=dev).manual_seed(seed + b) for b in range(B)]


def alternate(fns, rounds):
    """{name: median over rounds} with the variants run one after another in every round."""
    got = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            got[k].append(fn())
    return {k: statistics.median(v) for k, v in got.items()}


def update_kernels(dev, iters, rounds):
    res = {}
    cases = {"posenet_32x144": ([32, 294, 1, 144], False, None),
             "trajnet_64x144x13": ([64, 144, 13], True, None),
             "posenet_mix8": ([len(LENGTHS), 294, 1, max(LENGTHS)], False, tuple(LENGTHS))}
    for name, (shape, cl, lengths) in cases.items():
        x0, xt = torch.randn(shape, device=dev), torch.randn(shape, device=dev)
        coef = torch.rand(8, device=dev)
        out = torch.empty_like(x0)
        s = NoiseStreams(gens(dev, shape[0]), dev)
        single = lambda: ops.ddpm_step_philox(x0, xt, coef, out=out)
        per_clip = lambda: ops.ddpm_step_philox_clips(x0, xt, coef, s, cl, lengths, out=out)
        r = alternate({"single_stream_us": lambda: 1e3 * time_ms(single, iters),
                       "per_clip_us": lambda: 1e3 * time_ms(per_clip, iters)}, rounds)
        s.close()
        res[name] = {k: round(v, 2) for k, v in r.items()}
    return res


def model(dev):
    m = PoseNet(dataset=synthetic.make_dataset('pose'), body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8,
                num_heads=4, device=dev, traj_feat_dim=22)
    m.load_state_dict({k: v.cpu() for k, v in synthetic.synth_state_dict(m, 1).items()})
    return m.to(dev).eval()


def step_graph(m, dev, iters, rounds):
    B, T = 32, 144
    cond = synthetic.posenet_batch(B, T, 3)['cond'].to(dev)
    x = torch.randn(B, 294, 1, T, device=dev)
    ts = torch.full((B,), 500, dtype=torch.int64, device=dev)
    coef = torch.rand(8, device=dev)
    e = m.prepare_cond(cond, None)
    s = NoiseStreams(gens(dev, B), dev)
    r = alternate({"single_stream_us": lambda: 1e3 * time_ms(lambda: e.sample_step(x, ts, coef), iters),
                   "per_clip_us": lambda: 1e3 * time_ms(lambda: e.sample_step(x, ts, coef, streams=s), iters)}, rounds)
    s.close()
    return {k: round(v, 1) for k, v in r.items()}


def loop_rate(m, dev, rounds):
    import argparse as ap
    B, T = 32, 144
    d = diffusion.create_gaussian_diffusion(ap.Namespace(noise_schedule='cosine', sigma_small=True), diffusion,
                                            diffusion.SpacedDiffusionPoseNet, 1000, '100', dev)
    cond = synthetic.posenet_batch(B, T, 3)['cond'].to(dev)

    def run(with_gens):
        batch = {'cond': cond}
        if with_gens:
            batch['generators'] = gens(dev, B)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        d.p_sample_loop(m, batch, [B, 294, 1, T], clip_denoised=False)
        torch.cuda.synchronize()
        return B / (time.perf_counter() - t0)

    run(False), run(True)  # graphs captured, condition embedded
    r = alternate({"single_stream_clips_per_s": lambda: run(False), "per_clip_clips_per_s": lambda: run(True)}, rounds)
    return {k: round(v, 1) for k, v in r.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=500)
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--json", default=None)
    a = p.parse_args()
    dev = torch.device("cuda:0")
    print("card:", card(), flush=True)
    m = model(dev)
    res = {"card": card(), "update_kernel": update_kernels(dev, a.iters, a.rounds),
           "posenet_step_graph_32x144": step_graph(m, dev, a.iters, a.rounds),
           "posenet_loop_100_steps_32x144": loop_rate(m, dev, a.rounds)}
    line = json.dumps(res)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
