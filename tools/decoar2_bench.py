"""Step time and profile of DeCoAR 2.0 (decoar2) next to wav2vec2_base_960 (GPU only).

    python tools/decoar2_bench.py [--steps 20] [--warmup 3] [--rounds 3] [--batch 32] [--seconds 10]

The two models share the encoder (12 post-LN layers, 768 channels, pos_conv 128 / 16) and differ in the front end:
kaldi fbank + CMVN + every second frame into Linear(80, 768) against the waveform conv stack + LayerNorm(512) +
Linear(512, 768). At 32 x 10 s both give T = 499 frames, so the difference of the two step times is the front end.
Both are timed in one process, alternating round by round (host clock around `steps` forwards that end in a device
synchronise), then one profiled pass each: device milliseconds per step by category (s3b_profile_read; category 2 is
the front end: conv 0 for wav2vec2, the fbank frame and CMVN kernels for DeCoAR 2.0). The card name and power limit head
the output: a time means nothing without them.
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

CATEGORIES = ("gemm", "attention", "frontend", "layernorm", "misc")


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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=10.0)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.decoar2 import Decoar2Expert
    from s3prl_b200.upstream.expert import UpstreamExpert

    if not torch.cuda.is_available():
        raise SystemExit("tools/decoar2_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    L = int(args.seconds * 16000)
    g = torch.Generator(device="cuda").manual_seed(0)
    wavs = [torch.randn(L, device="cuda", generator=g) for _ in range(args.batch)]
    experts = {"decoar2": Decoar2Expert().to("cuda"),
               "wav2vec2_base_960": UpstreamExpert(name="wav2vec2_base_960", seed=0).to("cuda")}
    for ex in experts.values():
        with torch.no_grad():
            for _ in range(args.warmup):
                ex(wavs)
    torch.cuda.synchronize()
    times = {n: [] for n in experts}
    for _ in range(args.rounds):
        for n, ex in experts.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.no_grad():
                for _ in range(args.steps):
                    ex(wavs)
            torch.cuda.synchronize()
            times[n].append((time.perf_counter() - t0) * 1e3 / args.steps)
    print(f"# {args.batch} x {args.seconds:g} s, T = {experts['decoar2'].num_frames(L)} (decoar2) / "
          f"{experts['wav2vec2_base_960'].num_frames(L)} (wav2vec2_base_960); ms per step, {args.rounds} alternating "
          f"rounds of {args.steps} steps")
    for n in experts:
        print(f"{n:18s} " + " ".join(f"{t:9.2f}" for t in times[n]))
    print("# profiled pass (launches timed one by one), device ms per step by category")
    print(f"{'':18s} " + " ".join(f"{c:>10s}" for c in CATEGORIES) + "      total  launches")
    for n, ex in experts.items():
        native = ex._native
        s3lib.check(native.lib.s3b_profile_enable(native.handle, 1))
        with torch.no_grad():
            for _ in range(args.steps):
                ex(wavs)
        ms, fl, ln = (C.c_double * 5)(), (C.c_double * 5)(), (C.c_int64 * 5)()
        s3lib.check(native.lib.s3b_profile_read(native.handle, ms, fl, ln, 1))
        s3lib.check(native.lib.s3b_profile_enable(native.handle, 0))
        print(f"{n:18s} " + " ".join(f"{ms[i] / args.steps:10.3f}" for i in range(5)) +
              f" {sum(ms) / args.steps:10.3f}  {sum(ln) // args.steps}")


if __name__ == "__main__":
    main()
