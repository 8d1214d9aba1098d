#!/usr/bin/env python
"""Per-shape timing of the production GEMM (s3b_gemm_bench) at the encoder's shapes, on the GPU only.

    python tools/gemm_shapes.py [--model base|large] [--iters N] [--repeats R] [--json FILE]
    S3B_LIB_PATH=/path/to/other/libs3prl_b200.so python tools/gemm_shapes.py     # another build of the same C ABI

For both operand schemes (f16q8, bf16x3), both row counts of bench.py's step (base, hubert_base 32 x 10 s: M = 7984 =
16 utterances x 499 frames, one of two lanes, and M = 15968, the whole batch in one lane; large, wav2vec2_large 16 x 20 s:
M = 7992 and 15984), the four encoder-layer GEMMs and both paired tile widths
(128, 256) plus the library's own choice ("auto"), it prints ms per launch (median of R repeats of N back-to-back
launches, CUDA events) and algorithmic TFLOP/s (2 M N K over that time). The card name and power limit head the output:
a time means nothing without them.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

# (name, N, K, gelu): gelu = fc1's epilogue (bias + GELU + operand planes), else bias + residual + fp32 like fc2
MODELS = {
    "base": dict(rows=[7984, 15968], shapes=[("qkv", 2304, 768, 0), ("out_proj", 768, 768, 0), ("fc1", 3072, 768, 1),
                                            ("fc2", 768, 3072, 0)]),
    "large": dict(rows=[7992, 15984], shapes=[("qkv", 3072, 1024, 0), ("out_proj", 1024, 1024, 0),
                                             ("fc1", 4096, 1024, 1), ("fc2", 1024, 4096, 0)]),
}
SCHEMES = ["f16q8", "bf16x3"]
WIDTHS = [0, 128, 256]  # 0 = the library's choice


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - the report still names the card
        q = f"nvidia-smi unavailable ({e})"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="base", choices=sorted(MODELS), help="base: hubert_base, large: wav2vec2_large")
    ap.add_argument("--iters", type=int, default=100, help="back-to-back launches per timing")
    ap.add_argument("--repeats", type=int, default=5, help="timings per point (the median is reported)")
    ap.add_argument("--json", default=None, help="also write every point to this file")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py needs a CUDA device (H100): nothing to time on this host")
    from s3prl_b200 import lib as s3lib

    lib = s3lib.load()
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}  library: {s3lib.lib_path()}")
    print(f"# {args.iters} launches per timing, median of {args.repeats}")
    print(f"{'scheme':7s} {'M':>6s} {'gemm':9s} {'N':>5s} {'K':>5s} {'tile':>5s} {'ms':>8s} {'TFLOP/s':>8s} {'spread%':>8s}")
    points = []
    saved = os.environ.get("S3B_GEMM_SCHEME")
    try:
        for scheme in SCHEMES:
            os.environ["S3B_GEMM_SCHEME"] = scheme  # read by the library at every call
            for M in MODELS[args.model]["rows"]:
                for gname, N, K, gelu in MODELS[args.model]["shapes"]:
                    for un in WIDTHS:
                        out = (C.c_float * 2)()
                        times = []
                        for _ in range(args.repeats):
                            s3lib.check(lib.s3b_gemm_bench(M, N, K, gelu, un, args.iters, out))
                            times.append(float(out[0]))
                        ms = statistics.median(times)
                        tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
                        spread = 100.0 * (max(times) - min(times)) / ms
                        width = int(out[1])
                        label = f"{width}" if un else f"{width}*"
                        print(f"{scheme:7s} {M:6d} {gname:9s} {N:5d} {K:5d} {label:>5s} {ms:8.4f} {tf:8.1f} {spread:8.1f}")
                        points.append(dict(scheme=scheme, M=M, gemm=gname, N=N, K=K, requested=un, tile=width, ms=ms,
                                           tflops=tf, times=times))
    finally:
        if saved is None:
            os.environ.pop("S3B_GEMM_SCHEME", None)
        else:
            os.environ["S3B_GEMM_SCHEME"] = saved
    print("# tile marked * = the library's own choice (requested 0)")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(model=args.model, card=name, power=power, lib=str(s3lib.lib_path()),
                                                   points=points),
                                              indent=1))


if __name__ == "__main__":
    main()
