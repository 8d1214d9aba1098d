"""Step time and profile of MAE-AST (mae_ast_frame, mae_ast_patch) against hubert_base and against the reference
expert on the same GPU (GPU only).

    python tools/mae_ast_bench.py [--steps 5] [--warmup 2] [--rounds 2]

Workloads: 32 x 10 s and 16 x 20 s, fabricated checkpoints (seed 0, the believed released configuration). At 10 s the
frame model runs 499 tokens per utterance and the patch model 62 x 8 = 496. For each workload, in one process and
alternating round by round (host clock around `steps` calls that end in a device synchronise):
  native     MaeAstExpert of both models, and UpstreamExpert("hubert_base") as the 768-wide yardstick
  reference  the reference's own s3prl.upstream.mae_ast.expert.UpstreamExpert on the GPU (fp32 torch), loaded from the
             same file, same batch; needs the install under oracle/_ref. Its front end runs kaldi.fbank per utterance
             on the GPU, as the expert does.
Then one profiled pass of each native model: device ms per step by the library's categories (s3b_profile_read_ex).
For MAE-AST, "frontend" is the fbank-to-patch-operand kernel, "gemm" holds post_extract_proj and the encoder's
linears, "norm" the positions + encoder.layer_norm kernel and the layers' LayerNorms, and the GEMM rate is the
library's algorithmic FLOPs over the GEMM category's device time. The card name and power limit head the output.
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

KINDS = {"mae_ast_frame": "frame", "mae_ast_patch": "patch"}


def reference_expert(kind: str):
    import torch

    import ref_runtime

    from s3prl_b200.upstream.mae_ast import fabricate_mae_ast_state_dict

    if ref_runtime.reference_root() is None:
        return None
    ref_runtime.activate()
    from s3prl.upstream.mae_ast.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save(fabricate_mae_ast_state_dict(0, kind), tmp.name)
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
    from s3prl_b200.upstream.mae_ast import MaeAstExpert

    if not torch.cuda.is_available():
        raise SystemExit("tools/mae_ast_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    models = {n: MaeAstExpert(name=n, kind=k).to("cuda") for n, k in KINDS.items()}
    models["hubert_base"] = UpstreamExpert(name="hubert_base").to("cuda")
    for n, k in KINDS.items():
        ref = reference_expert(k)
        if ref is not None:
            models[f"reference {n}"] = ref
    if not any(n.startswith("reference") for n in models):
        print("# reference: not measured (no install under oracle/_ref)")
    g = torch.Generator(device="cuda").manual_seed(0)
    for B, L in ((32, 160000), (16, 320000)):
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
        print(f"# {B} x {L // 16000} s: ms per step, {args.rounds} alternating rounds of {args.steps} steps")
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
        del wavs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
