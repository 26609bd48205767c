"""GEMM timing on the PoseNet shapes that DESIGN §4.1 quotes: fp16 pairs, M = 4640 rows (32 clips x 145 tokens).

    python tools/gemm_bench.py [--reps N]

Prints the card and its power limit, then per shape the time of one launch through the kernel test probe
(tests/native/libkernel_probe.so): bias, the TMA-store epilogue, CUDA events around --reps back-to-back launches after a
warm-up, and the algorithmic rate (2 M N K per launch).  Needs an H100; writes nothing."""
import argparse
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kernel_probe as kp  # noqa: E402

M = 4640
# name, N, K, activation, output (fp16 "pair" or "fp32")
SHAPES = [("QKV", 1536, 512, kp.ACT_NONE, "pair"), ("FFN1 + GELU", 1024, 512, kp.ACT_GELU, "pair"),
          ("out-proj", 512, 512, kp.ACT_NONE, "fp32"), ("FFN2", 512, 1024, kp.ACT_NONE, "fp32")]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    return q.stdout.strip().splitlines()[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    print(f"card: {card()} (name, power limit)", flush=True)
    g = torch.Generator().manual_seed(0)
    for name, N, K, act, form in SHAPES:
        A = kp.Operand(kp.KIND_F16, torch.randn(M, K, generator=g).to(dev))
        W = kp.Weight(kp.KIND_F16, [(torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev)], 128)
        bias = torch.randn(N, generator=g).to(dev)
        out = oh = ol = None
        if form == "pair":
            oh, ol = torch.empty(M, N, dtype=torch.float16, device=dev), torch.empty(M, N, dtype=torch.float16, device=dev)
        else:
            out = torch.empty(M, N, device=dev)

        def launch(reps):
            return kp.gemm(kp.KIND_F16, W, [A.seg(W.kblocks[0])], M, N, out=out, out_hi=oh, out_lo=ol, bias=bias, act=act,
                           tma_store=True, reps=reps)

        rc, params = launch(10)  # warm-up
        assert rc == 0 and params.tma_store == 1, (name, rc)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc, _ = launch(a.reps)
        e1.record()
        torch.cuda.synchronize()
        assert rc == 0, (name, rc)
        us = e0.elapsed_time(e1) * 1e3 / a.reps
        print(f"{name:12s} N {N:4d} K {K:4d} ({form} out): {us:7.2f} us per launch, "
              f"{2.0 * M * N * K / us * 1e-6:6.1f} TFLOP/s", flush=True)


if __name__ == "__main__":
    main()
