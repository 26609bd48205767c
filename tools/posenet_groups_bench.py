"""PoseNet forward-graph time with the layer chain as one serial chain and as two concurrent clip groups (posenet.cu,
GroupPlan), on RoHM's configuration (fp16 pairs, d_model 512, 4 heads of 128, 8 layers).

    python tools/posenet_groups_bench.py [--T 144] [--batches 1,2,8,32,128] [--iters N] [--rounds R] [--json PATH]

For every batch size: the forward graph of each variant, timed with CUDA events around --iters replays after warm-up
replays, the variants alternated --rounds times (the reported figure is the median over rounds):
  serial      the serial layer chain (rohm_posenet_set_option(2, 1));
  split       two clip groups (rohm_posenet_set_option(2, 2); at B = 1 the serial chain);
  split_nopdl two clip groups with programmatic dependent launch off on every kernel (rohm_posenet_set_option(1, 0));
  auto        what the engine picks from the input (option 2 = 0, the default).
The outputs of every variant are compared bit for bit with the serial chain's.  These numbers are what the engine's rule
for choosing between the two rests on.  Prints the card and its power limit from the same run, then one JSON line.  Needs
an H100; writes nothing unless --json is given."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rohm_b200 import synthetic  # noqa: E402
from rohm_b200.posenet import PoseNet  # noqa: E402

VARIANTS = {"serial": (1, 1), "split": (2, 1), "split_nopdl": (2, 0), "auto": (0, 1)}  # name: (option 2, option 1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def graph_ms(e, x, ts, out, iters):
    for _ in range(3):
        e.forward(x, ts, out)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        e.forward(x, ts, out)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=144)
    ap.add_argument("--batches", default="1,2,8,32,128")
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("posenet_groups_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    batches = [int(b) for b in args.batches.split(",")]
    print(card(), flush=True)
    m = PoseNet(dataset=synthetic.make_dataset('pose'), body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8,
                num_heads=4, device=dev, traj_feat_dim=22)
    m.load_state_dict({k: v.cpu() for k, v in synthetic.synth_state_dict(m, 1).items()})
    m = m.to(dev).eval()
    m.engine(max(batches), args.T, dev)
    rows = []
    for B in batches:
        g = torch.Generator().manual_seed(B)
        x = torch.randn(B, 294, 1, args.T, generator=g).to(dev)
        ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
        e = m.prepare_cond(synthetic.posenet_batch(B, args.T, B)['cond'].to(dev))
        times = {k: [] for k in VARIANTS}
        outs = {}
        for _ in range(args.rounds):
            for name, (groups, pdl) in VARIANTS.items():
                assert e.lib.rohm_posenet_set_option(e.handle, 2, groups) == 0
                assert e.lib.rohm_posenet_set_option(e.handle, 1, pdl) == 0
                out = torch.empty_like(x)
                times[name].append(graph_ms(e, x, ts, out, args.iters))
                outs[name] = out
        assert e.lib.rohm_posenet_set_option(e.handle, 2, 0) == 0
        assert e.lib.rohm_posenet_set_option(e.handle, 1, 1) == 0
        same = all(torch.equal(o.view(torch.int32), outs["serial"].view(torch.int32)) for o in outs.values())
        row = {"B": B, "T": args.T, "bit_identical": same}
        for name, t in times.items():
            row[name + "_ms"] = statistics.median(t)
            row[name + "_spread_ms"] = max(t) - min(t)
        row["split_gain"] = row["serial_ms"] / row["split_ms"] - 1.0
        rows.append(row)
        print(json.dumps(row), flush=True)
    result = {"card": card(), "rows": rows}
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
