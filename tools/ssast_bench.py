"""Step time and profile of SSAST (ssast_frame_base, ssast_patch_base) against hubert_base and against the reference
expert on the same GPU (GPU only).

    python tools/ssast_bench.py [--steps 5] [--warmup 2] [--rounds 2]

Workload: 32 x 10 s, fabricated checkpoints (seed 0), with window_secs 1 (speech commands: 10 windows of 101 / 110
tokens per utterance) and 10 (speaker identification: one window of 1001 / 1190 tokens). For each window, in one
process and alternating round by round (host clock around `steps` calls that end in a device synchronise):
  native     SsastExpert of both models, and UpstreamExpert("hubert_base") as the 768-wide yardstick
  reference  the reference's own s3prl.upstream.ssast.expert.UpstreamExpert on the GPU (fp32 torch; timm replaced by
             oracle/timm_shim.py when absent), loaded from the same file, same batch; needs the install under oracle/_ref.
             Its front end runs kaldi.fbank per window and utterance on the GPU, as the expert does.
Then one profiled pass of each native model: device ms per step by the library's categories (s3b_profile_read_ex).
For SSAST, "frontend" is the fbank, the patch operand and the token assembly, "gemm" holds the patch GEMM and the
encoder's linears, "misc" is the output layout step (the per-layer fold into the hidden states), and the GEMM rate is
the library's algorithmic FLOPs over the GEMM category's device time. The card name and power limit head the output.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "tools"))

from apc_bench import CATEGORIES, card  # noqa: E402

KINDS = {"ssast_frame_base": "frame", "ssast_patch_base": "patch"}


def reference_expert(kind: str, window_secs: float):
    import torch

    import ref_runtime
    import timm_shim

    from s3prl_b200.upstream.ssast import fabricate_ssast_state_dict

    if ref_runtime.reference_root() is None:
        return None
    ref_runtime.activate()
    timm_shim.install()
    from s3prl.upstream.ssast.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pth", delete=False)
    tmp.close()
    try:
        torch.save(fabricate_ssast_state_dict(0, kind), tmp.name)
        ex = UpstreamExpert(tmp.name, "base_" + kind[0], window_secs)
    finally:
        os.unlink(tmp.name)
    return ex.eval().cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.ssast import SsastExpert

    if not torch.cuda.is_available():
        raise SystemExit("tools/ssast_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    B, L = 32, 160000
    g = torch.Generator(device="cuda").manual_seed(0)
    wavs = [torch.randn(L, device="cuda", generator=g) * 0.1 for _ in range(B)]
    for window in (1.0, 10.0):
        models = {f"{n} w{window:g}": SsastExpert(name=n, kind=k, window_secs=window).to("cuda") for n, k in KINDS.items()}
        models["hubert_base"] = UpstreamExpert(name="hubert_base").to("cuda")
        for n, k in KINDS.items():
            ref = reference_expert(k, window)
            if ref is not None:
                models[f"reference {n} w{window:g}"] = ref
        if not any(n.startswith("reference") for n in models):
            print("# reference: not measured (no install under oracle/_ref)")
        with torch.no_grad():
            for ex in models.values():
                for _ in range(args.warmup):
                    ex(wavs)
        torch.cuda.synchronize()
        times = {n: [] for n in models}
        for _ in range(args.rounds):
            for n, ex in models.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with torch.no_grad():
                    for _ in range(args.steps):
                        ex(wavs)
                torch.cuda.synchronize()
                times[n].append((time.perf_counter() - t0) * 1e3 / args.steps)
        print(f"# {B} x {L // 16000} s, window_secs {window:g}: ms per step, {args.rounds} alternating rounds of "
              f"{args.steps} steps")
        for n in models:
            print(f"{n:34s} " + " ".join(f"{t:9.2f}" for t in times[n]))
        print("# profiled pass (launches timed one by one), device ms per step by category; GEMM TFLOP/s")
        print(f"{'':34s} " + " ".join(f"{c:>10s}" for c in CATEGORIES) + "      total  launches  gemm TFLOP/s")
        for n, ex in models.items():
            if n.startswith("reference"):
                continue
            native = ex._native
            s3lib.check(native.lib.s3b_profile_enable(native.handle, 1))
            with torch.no_grad():
                for _ in range(args.steps):
                    ex(wavs)
            nc = len(CATEGORIES)
            ms, fl, ln = (C.c_double * nc)(), (C.c_double * nc)(), (C.c_int64 * nc)()
            s3lib.check(native.lib.s3b_profile_read_ex(native.handle, nc, ms, fl, ln, 1))
            s3lib.check(native.lib.s3b_profile_enable(native.handle, 0))
            rate = fl[0] / (ms[0] * 1e-3) / 1e12 if ms[0] > 0 else 0.0
            print(f"{n:34s} " + " ".join(f"{ms[i] / args.steps:10.3f}" for i in range(nc)) +
                  f" {sum(ms) / args.steps:10.3f}  {sum(ln) // args.steps:8d}  {rate:12.1f}")
        del models
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
