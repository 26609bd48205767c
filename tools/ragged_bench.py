"""Batches of recordings with different lengths through the PoseNet engine (fp16 pairs, RoHM's configuration: d_model 512,
4 heads of 128, 8 layers).

    python tools/ragged_bench.py [--iters N] [--json PATH]

The workload is a fixed mix of recording lengths between 145 and 4999 frames, 9044 frames in all.  Three timings of the
forward graph, each the mean of CUDA events around --iters replays after warm-up replays of the same graph:
  (a) the mix as one batch with batch['lengths'] (packed tokens, no padding rows);
  (b) every recording alone as a batch of one, summed over the recordings;
  (c) the mix padded to the longest recording, without lengths.  Its output is wrong (padded frames take part in
      attention), but it is what batching a mix costs without per-clip lengths.
Prints the card and its power limit from the same run, then one JSON line.  Needs an H100; writes nothing unless --json
is given."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rohm_b200 import synthetic  # noqa: E402
from rohm_b200.posenet import PoseNet  # noqa: E402

D, H, LAYERS = 512, 4, 8
LENGTHS = (4999, 1500, 900, 600, 400, 300, 200, 145)  # 9044 frames, 9052 tokens


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def time_ms(fn, iters, warmup=3):
    """Mean device time of fn() over iters calls (CUDA events around the whole window), after warmup calls."""
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


def forward_ms(m, x, cond, ts, lengths, iters):
    """The engine's forward graph for one batch: the condition is embedded once, every call is one graph replay."""
    e = m.prepare_cond(cond, lengths)
    out = torch.empty_like(x)
    return time_ms(lambda: e.forward(x, ts, out), iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if a.iters < 20:
        raise SystemExit("ragged_bench: --iters must be at least 20")
    if not torch.cuda.is_available():
        raise SystemExit("ragged_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    c = card()
    print(f"card: {c} (name, power limit, max SM clock)", flush=True)
    ds = synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=D, ff_size=1024, num_layers=LAYERS, num_heads=H, device=dev,
                traj_feat_dim=22)
    m.load_state_dict(synthetic.synth_state_dict(m, 1))
    m.to(dev).eval()
    B, T = len(LENGTHS), max(LENGTHS)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 294, 1, T, generator=g).to(dev)
    cond = synthetic.posenet_batch(B, T, 3)['cond'].to(dev)
    ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
    m.engine(B, T, dev)  # one engine sized for the padded batch serves all three

    ragged = forward_ms(m, x, cond, ts, LENGTHS, a.iters)
    alone = []
    for b, L in enumerate(LENGTHS):
        alone.append(forward_ms(m, x[b:b + 1, ..., :L].contiguous(), cond[b:b + 1, ..., :L].contiguous(), ts[b:b + 1],
                                None, a.iters))
    padded = forward_ms(m, x, cond, ts, None, a.iters)
    res = {"card": c, "lengths": list(LENGTHS), "frames": sum(LENGTHS), "tokens": sum(L + 1 for L in LENGTHS),
           "padded_tokens": B * (T + 1), "iters": a.iters, "ragged_ms": ragged, "alone_ms": alone,
           "alone_sum_ms": sum(alone), "padded_ms": padded}
    print(f"(a) ragged batch {ragged:8.3f} ms | (b) each recording alone {sum(alone):8.3f} ms summed | "
          f"(c) padded to {T} frames {padded:8.3f} ms", flush=True)
    print(json.dumps(res), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
