"""Step time and profile of NPC (npc) against the reference expert and against torch's conv1d stack (GPU only).

    python tools/npc_bench.py [--steps 10] [--warmup 2] [--rounds 3]

Workloads: 32 x 10 s (T = 998) and 16 x 20 s (T = 1998), the fabricated checkpoint (seed 0, npc_config()). For each, in
one process and alternating round by round (host clock around `steps` calls that end in a device synchronise):
  native     NpcExpert: fbank + CMVN kernels, three GEMMs per block (conv, linear, masked conv on its unmasked taps)
  reference  the reference's own s3prl.upstream.npc.expert.UpstreamExpert on the GPU (torchaudio fbank per utterance,
             torch Conv1d / BatchNorm1d, the masked convs over all their taps), loaded from the same checkpoint, same
             batch; needs the install under oracle/_ref
  conv1d     the reference's NPC module alone (torch.nn.functional.conv1d stack, eval mode) on the same features:
             the model without its front end
Then one profiled pass of the native model (device ms per step by category, s3b_profile_read_ex). The card name and
power limit head the output: a time means nothing without them.
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


def reference_expert(sd, config):
    import torch

    import ref_runtime

    if ref_runtime.reference_root() is None:
        return None
    ref_runtime.activate()
    from s3prl.upstream.npc.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"config": config, "model": sd}, tmp.name)
        ex = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    return ex.eval().cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.npc import NpcExpert, fabricate_npc_state_dict, npc_config

    if not torch.cuda.is_available():
        raise SystemExit("tools/npc_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    config = npc_config()
    sd = fabricate_npc_state_dict(0)
    native = NpcExpert(seed=0).to("cuda")
    ref = reference_expert(sd, config)
    if ref is None:
        print("# reference: not installed under oracle/_ref; the reference and conv1d rows are skipped")
    for batch, seconds in ((32, 10.0), (16, 20.0)):
        L = int(seconds * 16000)
        g = torch.Generator(device="cuda").manual_seed(0)
        wavs = [torch.randn(L, device="cuda", generator=g) for _ in range(batch)]
        T = native.num_frames(L)
        feats = torch.randn(batch, T, 80, device="cuda", generator=g)
        impls = {"native": lambda: native(wavs)}
        if ref is not None:
            impls["reference"] = lambda: ref(wavs)
            impls["conv1d"] = lambda: ref.model(feats, testing=True)
        with torch.no_grad():
            for f in impls.values():
                for _ in range(args.warmup):
                    f()
            torch.cuda.synchronize()
            times = {k: [] for k in impls}
            for _ in range(args.rounds):
                for k, f in impls.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(args.steps):
                        f()
                    torch.cuda.synchronize()
                    times[k].append((time.perf_counter() - t0) * 1e3 / args.steps)
        print(f"# {batch} x {seconds:g} s, T = {T}; ms per step, {args.rounds} alternating rounds of {args.steps} steps")
        for k, ts in times.items():
            print(f"{k:10s} " + " ".join(f"{t:9.2f}" for t in ts))
        h = native._native
        s3lib.check(h.lib.s3b_profile_enable(h.handle, 1))
        with torch.no_grad():
            for _ in range(args.steps):
                native(wavs)
        ms, fl, ln = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
        s3lib.check(h.lib.s3b_profile_read_ex(h.handle, 6, ms, fl, ln, 1))
        s3lib.check(h.lib.s3b_profile_enable(h.handle, 0))
        print("# native, profiled pass (launches timed one by one), device ms per step by category")
        print(" ".join(f"{c:>10s}" for c in CATEGORIES) + "      total  launches  GEMM TFLOP/s")
        print(" ".join(f"{ms[i] / args.steps:10.3f}" for i in range(6)) +
              f" {sum(ms) / args.steps:10.3f}  {sum(ln) // args.steps:8d}  {fl[0] / (ms[0] * 1e-3) / 1e12:12.1f}")


if __name__ == "__main__":
    main()
