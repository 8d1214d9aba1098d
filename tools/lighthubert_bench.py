"""Step time and profile of LightHuBERT (lighthubert_small, lighthubert_base, lighthubert_stage1) against hubert_base and
against the reference expert on the same GPU (GPU only).

    python tools/lighthubert_bench.py [--steps 5] [--warmup 2] [--rounds 2]

Workloads: 32 x 10 s (T = 499) and 16 x 20 s (T = 999), fabricated checkpoints (seed 0). For each workload, in one
process and alternating round by round (host clock around `steps` calls that end in a device synchronise):
  native     LighthubertExpert of each subnet, and UpstreamExpert("hubert_base") as the 768-wide HuBERT yardstick
  reference  the reference's own s3prl.upstream.lighthubert.expert.UpstreamExpert on the GPU (fp32 torch), loaded from
             the same supernet file, same batch; needs the install under oracle/_ref
Then one profiled pass of each native model: device ms per step by the library's categories (s3b_profile_read_ex).
"gemm" holds the conv stack's GEMMs, the encoder's linears and the pos_conv GEMM together; "layernorm" holds the conv
stack's LayerNorms, the encoder's and the pos_conv combine kernel. The card name and power limit head the output: a
time means nothing without them.
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

KINDS = {"lighthubert_small": "small", "lighthubert_base": "base", "lighthubert_stage1": "stage1"}


def reference_expert(kind: str):
    import torch

    import ref_runtime

    from s3prl_b200.upstream.lighthubert import fabricate_lighthubert_state_dict, lighthubert_config

    if ref_runtime.reference_root() is None:
        return None
    ref_runtime.activate()
    from s3prl.upstream.lighthubert.expert import UpstreamExpert

    cfg = lighthubert_config(kind)
    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"cfg": {"model": cfg}, "model": fabricate_lighthubert_state_dict(0, cfg)}, tmp.name)
        ex = UpstreamExpert(tmp.name)
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
    from s3prl_b200.upstream.lighthubert import LighthubertExpert

    if not torch.cuda.is_available():
        raise SystemExit("tools/lighthubert_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    models = {n: LighthubertExpert(name=n, kind=k).to("cuda") for n, k in KINDS.items()}
    models["hubert_base"] = UpstreamExpert(name="hubert_base").to("cuda")
    for n, k in KINDS.items():
        ref = reference_expert(k)
        if ref is not None:
            models[f"reference {n}"] = ref
    if not any(n.startswith("reference") for n in models):
        print("# reference: not measured (no install under oracle/_ref)")
    for B, seconds in ((32, 10), (16, 20)):
        L = seconds * 16000
        g = torch.Generator(device="cuda").manual_seed(0)
        wavs = [torch.randn(L, device="cuda", generator=g) * 0.1 for _ in range(B)]
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
        T = models["hubert_base"].num_frames(L)
        print(f"# {B} x {seconds} s, T = {T}: ms per step, {args.rounds} alternating rounds of {args.steps} steps")
        for n in models:
            print(f"{n:32s} " + " ".join(f"{t:9.2f}" for t in times[n]))
        print("# profiled pass (launches timed one by one), device ms per step by category")
        print(f"{'':32s} " + " ".join(f"{c:>10s}" for c in CATEGORIES) + "      total  launches")
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
            print(f"{n:32s} " + " ".join(f"{ms[i] / args.steps:10.3f}" for i in range(nc)) +
                  f" {sum(ms) / args.steps:10.3f}  {sum(ln) // args.steps}")
        del wavs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
