"""Cost of per-clip guidance normalisers (PoseNet.guidance_normaliser = 'clip') against the batch-wide ones.

    python tools/clip_guidance_bench.py [--iters N] [--rounds R] [--json PATH]

Times the two guidance calls of one guided step -- the skating term (rohm_skating_guidance: forward kinematics, loss and
VJP launches) and the 2-D projection term (rohm_projection_guidance) -- with per_clip = 0 and per_clip = 1, on
  (1) 32 clips x 143 frames (RoHM's PoseNet batch), and
  (2) the 8-recording mix of tools/ragged_bench.py (DESIGN 4.6; 4999 ... 145 frames).  The batch-wide projection term
      takes no lengths, so on the mix it runs over the padded batch; per clip it runs with lengths.  The skating term
      takes lengths in both modes.
Each figure is the mean device time over --iters back-to-back calls (CUDA events around the window) after a warm-up; the
two modes alternate inside every round and the median of --rounds rounds is reported.  Prints the card, its power limit
and maximum SM clock from the same run, then one JSON line.  Needs an H100; writes nothing unless --json is given."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ragged_bench import LENGTHS, card, time_ms  # noqa: E402
from rohm_b200 import synthetic  # noqa: E402
from rohm_b200.body_model import BodyModel, kernels_for  # noqa: E402


def camera(B, T, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    aff = torch.zeros(B, 3, 4)
    aff[:, :, :3] = torch.tensor([[1., 0, 0], [0, 0, -1], [0, 1, 0]])
    aff[:, :, 3] = torch.tensor([0.2, 1.0, 5.0]) + 0.1 * torch.randn(B, 3, generator=g)
    focal, center = torch.tensor([[1000., 990.]]).repeat(B, 1), torch.tensor([[900., 500.]]).repeat(B, 1)
    kp = torch.cat([900 + 300 * torch.randn(B, T, 22, 1, generator=g), 500 + 200 * torch.randn(B, T, 22, 1, generator=g),
                    torch.rand(B, T, 22, 1, generator=g)], dim=-1)
    return [t.to(dev).contiguous() for t in (aff, focal, center, kp)]


def case(k, mean, std, x, lengths, dev, iters, rounds):
    B, T = x.shape[0], x.shape[-1]
    L = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
    aff, focal, center, kp = camera(B, T, dev)
    fns = {
        "skating_batch_us": lambda: k.skating_guidance(x, mean, std, lengths=L),
        "skating_clip_us": lambda: k.skating_guidance(x, mean, std, lengths=L, per_clip=True),
        "projection_batch_us": lambda: k.projection_guidance(x, mean, std, aff, focal, center, kp),
        "projection_clip_us": lambda: k.projection_guidance(x, mean, std, aff, focal, center, kp, lengths=L, per_clip=True),
    }
    got = {name: [] for name in fns}
    for _ in range(rounds):
        for name, fn in fns.items():
            got[name].append(1e3 * time_ms(fn, iters))
    return {name: round(statistics.median(v), 2) for name, v in got.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_guidance_bench: needs a CUDA device (an H100)")
    dev = torch.device("cuda:0")
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    mean, std = torch.from_numpy(ds.Mean).to(dev), torch.from_numpy(ds.Std).to(dev)
    bm = BodyModel.create('', device=dev, seed=0)
    mix = list(LENGTHS)
    k = kernels_for(bm, dev, max(32 * 143, len(mix) * max(mix)), with_vertices=False)
    res = {"card": card()}
    x = synthetic.plausible_motion(32, 143, 1, ds).to(dev).contiguous()
    res["b32_t143"] = case(k, mean, std, x, None, dev, a.iters, a.rounds)
    xm = torch.zeros(len(mix), 294, 1, max(mix))
    for b, n in enumerate(mix):
        xm[b:b + 1, ..., :n] = synthetic.plausible_motion(1, n, 10 + b, ds)
    res["mix8"] = case(k, mean, std, xm.to(dev).contiguous(), mix, dev, a.iters, a.rounds)
    res["mix8"]["lengths"] = mix
    print(f"card (name, power limit, max SM clock): {res['card']}")
    for name in ("b32_t143", "mix8"):
        r = res[name]
        print(f"{name}: skating batch {r['skating_batch_us']} us, clip {r['skating_clip_us']} us | "
              f"projection batch {r['projection_batch_us']} us, clip {r['projection_clip_us']} us")
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
