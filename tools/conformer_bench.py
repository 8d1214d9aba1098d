"""Step time of the rotary Conformer against the transformer of the same size (GPU only).

    python tools/conformer_bench.py [--steps 10] [--warmup 3] [--rounds 3]

Times 16 x 20 s batches (T = 999 frames) of ``wav2vec2_conformer_rope`` and ``wav2vec2_large_ll60k`` in one process,
alternating the two models round by round, then one profiled pass of each (per-category device time, the library's five
categories). The card name and power limit head the output: a time means nothing without them.

Counted from the shapes, a Conformer layer does about 1.9x the GEMM work per frame of a transformer-large layer
(4 D F + 7 D^2 multiply-adds against 2 D F + 4 D^2); a step time well above twice the transformer's would point at a
non-GEMM bottleneck.
"""
from __future__ import annotations

import argparse
import ctypes as C
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

MODELS = ("wav2vec2_conformer_rope", "wav2vec2_large_ll60k")
CATEGORIES = ("gemm", "attention", "conv0", "layernorm", "misc")


def card():
    import torch

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - the report still names the card
        q = f"nvidia-smi unavailable ({e})"
    return torch.cuda.get_device_name(0), q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=20.0)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.expert import UpstreamExpert

    if not torch.cuda.is_available():
        raise SystemExit("tools/conformer_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    L = int(args.seconds * 16000)
    g = torch.Generator(device="cuda").manual_seed(0)
    wavs = [torch.randn(L, device="cuda", generator=g) for _ in range(args.batch)]
    experts = {n: UpstreamExpert(name=n, seed=0).to("cuda") for n in MODELS}
    for n, ex in experts.items():
        with torch.no_grad():
            for _ in range(args.warmup):
                ex(wavs)
        torch.cuda.synchronize()
    times = {n: [] for n in MODELS}
    for r in range(args.rounds):
        for n, ex in experts.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.no_grad():
                for _ in range(args.steps):
                    ex(wavs)
            torch.cuda.synchronize()
            times[n].append((time.perf_counter() - t0) * 1e3 / args.steps)
    print(f"# {args.batch} x {args.seconds:g} s, T = {experts[MODELS[0]].num_frames(L)}; ms per step, "
          f"{args.rounds} alternating rounds of {args.steps} steps")
    for n in MODELS:
        print(f"{n:28s} " + " ".join(f"{t:8.2f}" for t in times[n]))
    ratio = min(times[MODELS[0]]) / min(times[MODELS[1]])
    print(f"conformer / transformer (best rounds): {ratio:.2f}")
    print("# profiled pass (launches timed one by one: lanes run back to back), ms per step by category")
    print(f"{'':28s} " + " ".join(f"{c:>10s}" for c in CATEGORIES) + "  launches")
    for n, ex in experts.items():
        native = ex._native
        s3lib.check(native.lib.s3b_profile_enable(native.handle, 1))
        with torch.no_grad():
            for _ in range(args.steps):
                ex(wavs)
        ms, fl, ln = (C.c_double * 5)(), (C.c_double * 5)(), (C.c_int64 * 5)()
        s3lib.check(native.lib.s3b_profile_read(native.handle, ms, fl, ln, 1))
        s3lib.check(native.lib.s3b_profile_enable(native.handle, 0))
        print(f"{n:28s} " + " ".join(f"{ms[i] / args.steps:10.2f}" for i in range(5)) +
              f"  {sum(ln) // args.steps}")


if __name__ == "__main__":
    main()
