"""Long-clip measurement of the PoseNet engine (fp16 pairs, RoHM's configuration: d_model 512, 4 heads of 128, 8 layers).

    python tools/long_clip_bench.py [--iters N] [--json PATH]

Prints the card and its power limit, then
  * per clip length T: B ~ 4640 / (T + 1) clips (about the token count of the benchmark's 32 x 145), the forward graph's
    time (CUDA events over --iters replays), the attention share of one event-timed forward (engine.profile) and the
    attention rate, counting 4 S^2 D flops per clip and layer (S = T + 1);
  * kernel against kernel through the kernel test probe (tests/native/libkernel_probe.so), CUDA events around --reps
    back-to-back launches: the SIMT kernel against the streaming wgmma kernel where both run (161 - 212 tokens), and the
    streaming kernel against the 160-key wgmma kernel where that one runs (<= 160 tokens).
Needs an H100; writes nothing unless --json is given."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from rohm_b200 import synthetic  # noqa: E402
from rohm_b200.posenet import PoseNet  # noqa: E402

D, H, LAYERS = 512, 4, 8
CLIP_T = [144, 160, 200, 211, 256, 512, 1000, 2000, 4999]
KERNEL_PAIRS = [("simt", "stream", [161, 201, 212]), ("stream", "wgmma", [64, 145, 160])]
TOKENS = 4640


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


def clip_lengths(dev, iters):
    ds = synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=D, ff_size=1024, num_layers=LAYERS, num_heads=H, device=dev,
                traj_feat_dim=22)
    m.load_state_dict(synthetic.synth_state_dict(m, 1))
    m.to(dev).eval()
    rows = []
    for T in CLIP_T:
        S = T + 1
        B = max(1, round(TOKENS / S))
        g = torch.Generator().manual_seed(T)
        x = torch.randn(B, 294, 1, T, generator=g).to(dev)
        cond = synthetic.posenet_batch(B, T, 3)['cond'].to(dev)
        ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
        batch = {'x_t': x, 'cond': cond}
        for _ in range(3):  # engine, condition embedding, graph capture
            m(batch, ts)
        torch.cuda.synchronize()
        ms = time_ms(lambda: m(batch, ts), iters)
        e = m.prepare_cond(cond)
        prof_ms, _ = e.profile(x, ts)
        torch.cuda.synchronize()
        attn_ms = prof_ms["attention"]
        total_prof = sum(prof_ms.values())
        flops = 4.0 * S * S * D * B * LAYERS
        r = {"T": T, "B": B, "tokens": B * S, "forward_ms": ms, "clips_per_s_forward": B / ms * 1e3,
             "attention_ms_profiled": attn_ms, "attention_share": attn_ms / total_prof,
             "attention_tflops": flops / (attn_ms * 1e-3) / 1e12}
        print(f"T={T:5d} B={B:3d}: forward {ms:8.3f} ms | attention {attn_ms:7.3f} of {total_prof:7.3f} ms profiled "
              f"({100 * r['attention_share']:4.1f} %) | attention {r['attention_tflops']:6.1f} TFLOP/s", flush=True)
        rows.append(r)
    return rows


def kernels(dev, reps):
    import kernel_probe as kp
    ids = {"simt": kp.ATTN_SIMT, "stream": kp.ATTN_WGMMA_STREAM, "wgmma": kp.ATTN_WGMMA}
    rows = []
    for first, second, lengths in KERNEL_PAIRS:
        for S in lengths:
            B = max(1, round(TOKENS / S))
            g = torch.Generator().manual_seed(S)
            qkv = torch.randn(B * S, 3 * D, generator=g).to(dev)
            hi, lo = kp.split(kp.KIND_F16, qkv)
            ctx_hi = torch.empty(B * S, D, dtype=torch.float16, device=dev)
            ctx_lo = torch.empty_like(ctx_hi)
            scale = 1.0 / math.sqrt(D // H)
            r = {"S": S, "B": B}
            for name in (first, second):
                call = lambda n=reps: kp.attention(hi, lo, ctx_hi, ctx_lo, B, S, D, H, scale, kp.KIND_F16, ids[name], reps=n)
                assert call(5) == 0, (name, S)
                torch.cuda.synchronize()
                r[name + "_us"] = time_ms(call, 1) / reps * 1e3
                r[name + "_tflops"] = 4.0 * S * S * D * B / (r[name + "_us"] * 1e-6) / 1e12
            print(f"S={S:4d} B={B:3d}: {first} {r[first + '_us']:8.2f} us ({r[first + '_tflops']:5.1f} TFLOP/s) | "
                  f"{second} {r[second + '_us']:8.2f} us ({r[second + '_tflops']:5.1f} TFLOP/s) per layer", flush=True)
            rows.append(r)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_clip_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    c = card()
    print(f"card: {c} (name, power limit, max SM clock)", flush=True)
    res = {"card": c, "kernels": kernels(dev, a.reps), "clips": clip_lengths(dev, a.iters)}
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
