"""Step time and profile of XLS-R 1B / 2B against wav2vec2_large_ll60k (GPU only).

    python tools/xls_r_bench.py [--steps 5] [--warmup 2] [--rounds 2] [--batch 16]

Times 16 x 20 s batches (T = 999 frames) of the three models in one process, alternating them round by round, then one
profiled pass of each: device time per category (s3b_profile_read), algorithmic GEMM TFLOP/s and attention time and
TFLOP/s, whose head width is the model's (64 for wav2vec2_large_ll60k, 80 for XLS-R 1B, 120 for XLS-R 2B). A model that
does not fit at the requested batch runs at the largest batch that does, and the report says which. The card name and
power limit head the output: a time means nothing without them.
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

CATEGORIES = ("gemm", "attention", "conv0", "layernorm", "misc")
HEAD_WIDTH = {"wav2vec2_large_ll60k": 64, "xls_r_1b": 80, "xls_r_2b": 120}


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
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=20.0)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.configs import ARCHS, XLS_R
    from s3prl_b200.upstream.expert import UpstreamExpert

    if not torch.cuda.is_available():
        raise SystemExit("tools/xls_r_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    L = int(args.seconds * 16000)
    g = torch.Generator(device="cuda").manual_seed(0)
    wavs = [torch.randn(L, device="cuda", generator=g) for _ in range(args.batch)]
    archs = {"wav2vec2_large_ll60k": ARCHS["wav2vec2_large_ll60k"], **XLS_R}
    experts, batch = {}, {}
    for n, a in archs.items():
        ex = UpstreamExpert(name=n if n in ARCHS else "wav2vec2_local", arch=a, seed=0).to("cuda")
        b = args.batch
        while b >= 1:
            try:
                with torch.no_grad():
                    for _ in range(args.warmup):
                        ex(wavs[:b])
                torch.cuda.synchronize()
                break
            except (s3lib.S3BError, torch.cuda.OutOfMemoryError) as e:
                print(f"# {n}: batch {b} does not fit ({str(e)[:80]}); halving")
                b //= 2
        experts[n], batch[n] = ex, b
    times = {n: [] for n in experts}
    for _ in range(args.rounds):
        for n, ex in experts.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.no_grad():
                for _ in range(args.steps):
                    ex(wavs[: batch[n]])
            torch.cuda.synchronize()
            times[n].append((time.perf_counter() - t0) * 1e3 / args.steps)
    T = experts["wav2vec2_large_ll60k"].num_frames(L)
    print(f"# {args.seconds:g} s utterances, T = {T}; ms per step, {args.rounds} alternating rounds of {args.steps} steps")
    for n in experts:
        print(f"{n:22s} batch {batch[n]:2d} " + " ".join(f"{t:9.2f}" for t in times[n]))
    print("# profiled pass (launches timed one by one), ms per step by category; algorithmic TFLOP/s of GEMM and "
          "attention")
    print(f"{'':22s} " + " ".join(f"{c:>10s}" for c in CATEGORIES) + "   GEMM TF/s  attn(hd) TF/s  launches")
    for n, ex in experts.items():
        native = ex._native
        s3lib.check(native.lib.s3b_profile_enable(native.handle, 1))
        with torch.no_grad():
            for _ in range(args.steps):
                ex(wavs[: batch[n]])
        ms, fl, ln = (C.c_double * 5)(), (C.c_double * 5)(), (C.c_int64 * 5)()
        s3lib.check(native.lib.s3b_profile_read(native.handle, ms, fl, ln, 1))
        s3lib.check(native.lib.s3b_profile_enable(native.handle, 0))
        tf = [fl[i] / (ms[i] * 1e-3) / 1e12 if ms[i] > 0 else 0.0 for i in range(5)]
        print(f"{n:22s} " + " ".join(f"{ms[i] / args.steps:10.2f}" for i in range(5)) +
              f"   {tf[0]:9.1f}  {tf[1]:7.1f} ({HEAD_WIDTH[n]:3d})  {sum(ln) // args.steps}")


if __name__ == "__main__":
    main()
