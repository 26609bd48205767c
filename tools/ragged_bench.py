"""Batches of recordings with different lengths through the PoseNet engine (fp16 pairs, RoHM's configuration: d_model 512,
4 heads of 128, 8 layers) or the TrajNet + TrajControl engine (fp16 pairs, mid_dim 512).

    python tools/ragged_bench.py [--net posenet|trajcontrol] [--iters N] [--json PATH]

The PoseNet workload is a fixed mix of recording lengths between 145 and 4999 frames, 9044 frames in all; the
TrajControl one a mix between 144 and 4992 frames (multiples of 16, TrajNet's rule), 9040 frames in all.  Three timings
of the forward graph, each the mean of CUDA events around --iters replays after warm-up replays of the same graph:
  (a) the mix as one batch with batch['lengths'] (packed clips, no padding rows past each clip's own);
  (b) every recording alone as a batch of one, summed over the recordings;
  (c) the mix padded to the longest recording, without lengths.  Its output is wrong (padded frames take part in
      attention, or in TrajNet's GroupNorm statistics and convolutions), but it is what batching a mix costs without
      per-clip lengths.
Engine creation and the condition embedding stay outside the timed windows (the TrajNet engine is rebuilt whenever T
changes).
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
TRAJ_LENGTHS = (4992, 1504, 896, 592, 400, 304, 208, 144)  # 9040 frames


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


def traj_forward_ms(m, batch, ts, iters):
    """The TrajNet engine's forward graph for one batch: engine and condition pyramid made first, then graph replays."""
    from rohm_b200 import trajnet_engine
    e, x, t = trajnet_engine.prepare(m, batch, ts)
    return time_ms(lambda: e._forward_impl(x, t), iters)


def trajcontrol(dev, iters):
    from rohm_b200.trajnet import TrajNet
    m = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=True, device=dev,
                dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
    m.load_state_dict(synthetic.synth_state_dict(m, 2))
    m.to(dev).eval()
    B, T = len(TRAJ_LENGTHS), max(TRAJ_LENGTHS)
    g = torch.Generator().manual_seed(5)
    batch = {k: v.to(dev) for k, v in synthetic.trajnet_batch(B, T, 3, control=True).items() if k != 'motion_repr_clean'}
    batch['x_t'] = torch.randn(B, T, 13, generator=g).to(dev)
    ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
    ragged = traj_forward_ms(m, dict(batch, lengths=torch.tensor(TRAJ_LENGTHS, device=dev)), ts, iters)
    alone = [traj_forward_ms(m, {k: v[b:b + 1, :L].contiguous() for k, v in batch.items()}, ts[b:b + 1], iters)
             for b, L in enumerate(TRAJ_LENGTHS)]
    padded = traj_forward_ms(m, batch, ts, iters)
    return {"net": "trajcontrol", "lengths": list(TRAJ_LENGTHS), "frames": sum(TRAJ_LENGTHS), "padded_frames": B * T,
            "ragged_ms": ragged, "alone_ms": alone, "alone_sum_ms": sum(alone), "padded_ms": padded}, T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", choices=("posenet", "trajcontrol"), default="posenet")
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
    if a.net == "trajcontrol":
        res, T = trajcontrol(dev, a.iters)
        res = dict(card=c, iters=a.iters, **res)
        report(res, T, a.json)
        return
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
    report(res, T, a.json)


def report(res, T, path):
    print(f"(a) ragged batch {res['ragged_ms']:8.3f} ms | (b) each recording alone {res['alone_sum_ms']:8.3f} ms summed | "
          f"(c) padded to {T} frames {res['padded_ms']:8.3f} ms", flush=True)
    print(json.dumps(res), flush=True)
    if path:
        with open(path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
