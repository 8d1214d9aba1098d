#!/usr/bin/env python
"""Per-shape timing of the production GEMM (s3b_gemm_bench) at the encoder's shapes, on the GPU only.

    python tools/gemm_shapes.py [--model base|large] [--clusters auto,1,2,4] [--iters N] [--repeats R] [--json FILE]
    python tools/gemm_shapes.py --k-sweep [--clusters auto,1,2,4] [--iters N] [--repeats R] [--json FILE]
    S3B_LIB_PATH=/path/to/other/libs3prl_b200.so python tools/gemm_shapes.py     # another build of the same C ABI

For both operand schemes (f16q8, bf16x3), both row counts of bench.py's step (base, hubert_base 32 x 10 s: M = 7984 =
16 utterances x 499 frames, one of two lanes, and M = 15968, the whole batch in one lane; large, wav2vec2_large 16 x 20 s:
M = 7992 and 15984), the four encoder-layer GEMMs and both tile widths
(128, 256) plus the library's own choice ("auto"), it prints ms per launch (median of R repeats of N back-to-back
launches, CUDA events) and algorithmic TFLOP/s (2 M N K over that time). The card name and power limit head the output:
a time means nothing without them.

--clusters times every 128-wide point once per entry: auto = the library's choice of CTAs per cluster along N (the
CN column: CTAs that share each A tile by TMA multicast), 1 / 2 / 4 = S3B_GEMM_CLUSTER, which forces that size wherever
it divides the column tiles. The CN column shows the size a point ran with; other widths always run with 1.

The table also times a proxy of the conv stack (conv 1..6 at bench.py's shapes, 32 x 10 s for base, 16 x 20 s for large):
the linear with the conv's M, N = 512 and K = 1024 / 1536, with conv's bias + GELU + operand-plane epilogue.

--k-sweep times one shape (M = 7984, N = 2304, bias + residual + fp32 epilogue) at K = 256 .. 3072 for both schemes and
both widths, and fits the time of one round of tiles (ceil(tiles / SMs) rounds per launch) as fixed + per_k * K: the
fixed part is the per-tile cost that does not scale with K (epilogue, pipeline fill and drain).
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
# conv 1..6 rows of one step: batch x frames after each stride-2 conv (10 s -> 15999, ..., 499 frames); K = kw * 512
CONV_ROWS = {"base": (32, [15999, 7999, 3999, 1999, 999, 499]), "large": (16, [31999, 15999, 7999, 3999, 1999, 999])}
CONV_K = [1536, 1536, 1536, 1536, 1024, 1024]
SCHEMES = ["f16q8", "bf16x3"]
SWEEP_M, SWEEP_N, SWEEP_K = 7984, 2304, list(range(256, 3073, 256))
WIDTHS = [0, 128, 256]  # 0 = the library's choice
AUTO_CN = {"f16q8": 2, "bf16x3": 1}  # the library's cluster size for 128-wide linear tiles (model.cu: linear_params)


def set_cluster(cn):
    """S3B_GEMM_CLUSTER for the next calls (read by the library at every call); "auto" unsets it."""
    if cn == "auto":
        os.environ.pop("S3B_GEMM_CLUSTER", None)
    else:
        os.environ["S3B_GEMM_CLUSTER"] = cn


def cluster_used(cn, width, N, scheme):
    """CTAs per cluster the launch ran with: 128-wide tiles take the size where it divides N / 128."""
    size = AUTO_CN[scheme] if cn == "auto" else int(cn)
    return size if width == 128 and (N // 128) % size == 0 else 1


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - the report still names the card
        q = f"nvidia-smi unavailable ({e})"
    return name, q


def time_point(lib, s3lib, M, N, K, gelu, un, iters, repeats):
    out = (C.c_float * 2)()
    times = []
    for _ in range(repeats):
        s3lib.check(lib.s3b_gemm_bench(M, N, K, gelu, un, iters, out))
        times.append(float(out[0]))
    return statistics.median(times), times, int(out[1])


def k_sweep(lib, s3lib, args, sms):
    import numpy as np

    print(f"# K sweep: M = {SWEEP_M}, N = {SWEEP_N}, bias + residual + fp32; {sms} SMs")
    print(f"{'scheme':7s} {'tile':>5s} {'CN':>3s} {'K':>5s} {'ms':>8s} {'TFLOP/s':>8s} {'us/round':>9s}")
    points, fits = [], []
    for scheme in SCHEMES:
        os.environ["S3B_GEMM_SCHEME"] = scheme
        for un in (128, 256):
            for cn in args.clusters if un == 128 else args.clusters[:1]:
                set_cluster(cn)
                cn_used = cluster_used(cn, un, SWEEP_N, scheme)
                # a round: as many tiles as SMs (clusters that do not fit leave SMs idle: not counted here)
                rounds = -(-((SWEEP_M + 127) // 128) * (SWEEP_N // un) // sms)
                ks, us = [], []
                for K in SWEEP_K:
                    if scheme == "f16q8" and K % 128:
                        continue
                    ms, times, width = time_point(lib, s3lib, SWEEP_M, SWEEP_N, K, 0, un, args.iters, args.repeats)
                    per_round = ms * 1e3 / rounds
                    ks.append(K), us.append(per_round)
                    tf = 2.0 * SWEEP_M * SWEEP_N * K / (ms * 1e-3) / 1e12
                    print(f"{scheme:7s} {width:5d} {cn_used:3d} {K:5d} {ms:8.4f} {tf:8.1f} {per_round:9.2f}")
                    points.append(dict(scheme=scheme, tile=width, cn=cn_used, K=K, ms=ms, rounds=rounds, times=times))
                per_k, fixed = np.polyfit(np.array(ks, float), np.array(us, float), 1)
                fits.append(dict(scheme=scheme, tile=un, cn=cn_used, fixed_us=fixed, per_k_us=per_k, rounds=rounds))
    print("# fit per round of tiles: fixed_us + per_k_us * K   (mainloop share at K = 768 in the last column)")
    for f in fits:
        main768 = f["per_k_us"] * 768
        print(f"fit {f['scheme']:7s} {f['tile']:4d} CN {f['cn']}: fixed {f['fixed_us']:7.2f} us, per K "
              f"{f['per_k_us'] * 1e3:7.3f} ns  (K=768: fixed / mainloop = {f['fixed_us'] / main768:.2f})")
    return dict(points=points, fits=fits)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="base", choices=sorted(MODELS), help="base: hubert_base, large: wav2vec2_large")
    ap.add_argument("--iters", type=int, default=100, help="back-to-back launches per timing")
    ap.add_argument("--repeats", type=int, default=5, help="timings per point (the median is reported)")
    ap.add_argument("--json", default=None, help="also write every point to this file")
    ap.add_argument("--k-sweep", action="store_true", help="fit the per-tile fixed cost over K instead of the table")
    ap.add_argument("--clusters", default="auto", help="comma-separated: auto (the library's choice), 1, 2, 4")
    args = ap.parse_args()
    args.clusters = args.clusters.split(",")
    if any(c not in ("auto", "1", "2", "4") for c in args.clusters):
        raise SystemExit(f"--clusters takes auto, 1, 2 and 4, not {args.clusters}")

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py needs a CUDA device (H100): nothing to time on this host")
    from s3prl_b200 import lib as s3lib

    lib = s3lib.load()
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}  library: {s3lib.lib_path()}")
    print(f"# {args.iters} launches per timing, median of {args.repeats}")
    saved = {k: os.environ.get(k) for k in ("S3B_GEMM_SCHEME", "S3B_GEMM_CLUSTER")}

    def restore():
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v

    if args.k_sweep:
        try:
            res = k_sweep(lib, s3lib, args, torch.cuda.get_device_properties(0).multi_processor_count)
        finally:
            restore()
        if args.json:
            Path(args.json).parent.mkdir(parents=True, exist_ok=True)
            Path(args.json).write_text(json.dumps(dict(card=name, power=power, lib=str(s3lib.lib_path()), **res), indent=1))
        return
    print(f"{'scheme':7s} {'M':>6s} {'gemm':9s} {'N':>5s} {'K':>5s} {'tile':>5s} {'CN':>3s} {'ms':>8s} {'TFLOP/s':>8s} "
          f"{'spread%':>8s}")
    points = []
    nb, frames = CONV_ROWS[args.model]
    convs = [(nb * f, (f"conv{i + 1}", 512, k, 1)) for i, (f, k) in enumerate(zip(frames, CONV_K))]
    linears = [(M, shape) for M in MODELS[args.model]["rows"] for shape in MODELS[args.model]["shapes"]]
    try:
        for scheme in SCHEMES:
            os.environ["S3B_GEMM_SCHEME"] = scheme  # read by the library at every call
            for M, (gname, N, K, gelu) in linears + convs:
                for un in WIDTHS:
                    for cn in args.clusters if un != 256 else args.clusters[:1]:
                        set_cluster(cn)
                        ms, times, width = time_point(lib, s3lib, M, N, K, gelu, un, args.iters, args.repeats)
                        if width != 128 and cn != args.clusters[0]:
                            continue  # the library chose another width: the cluster setting does not apply
                        cn_used = cluster_used(cn, width, N, scheme)
                        tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
                        spread = 100.0 * (max(times) - min(times)) / ms
                        label = f"{width}" if un else f"{width}*"
                        print(f"{scheme:7s} {M:6d} {gname:9s} {N:5d} {K:5d} {label:>5s} {cn_used:3d} {ms:8.4f} {tf:8.1f} "
                              f"{spread:8.1f}")
                        points.append(dict(scheme=scheme, M=M, gemm=gname, N=N, K=K, requested=un, tile=width,
                                           cn=cn_used, ms=ms, tflops=tf, times=times))
    finally:
        restore()
    print("# tile marked * = the library's own choice (requested 0)")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(model=args.model, card=name, power=power, lib=str(s3lib.lib_path()),
                                                   points=points),
                                              indent=1))


if __name__ == "__main__":
    main()
