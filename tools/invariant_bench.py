"""Cost of the batch-invariant TrajNet mode: the TrajNet + TrajControl forward graph (fp16 pairs, mid_dim 512) of the default
engine against the batch-invariant one (TrajNet.batch_invariant = True), same weights and inputs.

    python tools/invariant_bench.py [--iters N] [--rounds R] [--json PATH]

Shapes: 64 x 144 (the trajcontrol benchmark), 1 x 144, 2 x 4992, and the 8-recording mix of DESIGN 4.6 (4992, 1504, 896,
592, 400, 304, 208 and 144 frames as one batch with batch['lengths']).  Each shape gets fresh engines of its own size.  Per
round, the two modes are timed one after the other (CUDA events around --iters replays of the forward graph after warm-up
replays), and the median over --rounds is reported, with whether the two outputs are bit-identical.  Engine creation and
the condition pyramid stay outside the timed windows.  Prints the card, its power limit and SM clocks read in the same run,
then one JSON line.  Needs an H100; writes nothing unless --json is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rohm_b200 import synthetic, trajnet_engine  # noqa: E402
from rohm_b200.trajnet import TrajNet  # noqa: E402

MIX = (4992, 1504, 896, 592, 400, 304, 208, 144)
SHAPES = (("64x144", [144] * 64, False), ("1x144", [144], False), ("2x4992", [4992] * 2, False), ("mix8", list(MIX), True))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def time_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def model(dev, invariant):
    m = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=True, device=dev,
                dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
    m.load_state_dict(synthetic.synth_state_dict(m, 2))
    m.batch_invariant = invariant
    return m.to(dev).eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("invariant_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    c = card()
    print(f"card: {c} (name, power limit, SM clock, max SM clock)", flush=True)
    nets = {False: model(dev, False), True: model(dev, True)}
    res = {"card": c, "iters": a.iters, "rounds": a.rounds, "shapes": {}}
    for name, lengths, ragged in SHAPES:
        B, T = len(lengths), max(lengths)
        g = torch.Generator().manual_seed(5)
        batch = {k: v.to(dev) for k, v in synthetic.trajnet_batch(B, T, 3, control=True).items() if k != 'motion_repr_clean'}
        batch['x_t'] = torch.randn(B, T, 13, generator=g).to(dev)
        if ragged:
            batch['lengths'] = torch.tensor(lengths, device=dev)
        ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
        runs, outs = {}, {}
        for inv, m in nets.items():
            m.invalidate_engine()
            e, x, t = trajnet_engine.prepare(m, batch, ts)
            outs[inv] = e._forward_impl(x, t).clone()
            runs[inv] = (e, x, t)
        times = {False: [], True: []}
        for _ in range(a.rounds):
            for inv in (False, True):
                e, x, t = runs[inv]
                times[inv].append(time_ms(lambda: e._forward_impl(x, t), a.iters))
        d, i = statistics.median(times[False]), statistics.median(times[True])
        res["shapes"][name] = {"B": B, "T": T, "frames": sum(lengths), "default_ms": d, "invariant_ms": i,
                               "default_all_ms": times[False], "invariant_all_ms": times[True],
                               "bit_identical": bool(torch.equal(outs[False], outs[True]))}
        print(f"{name:7s} default {d:8.3f} ms | invariant {i:8.3f} ms | x{i / d:5.3f} | "
              f"bit-identical {res['shapes'][name]['bit_identical']}", flush=True)
        for m in nets.values():
            m.invalidate_engine()
    print(json.dumps(res), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
