"""Step time and profile of DeCoAR (decoar_layers) against the reference expert and against cuDNN's LSTM (GPU only).

    python tools/decoar_bench.py [--steps 5] [--warmup 2] [--rounds 3]

Workloads: 32 x 10 s (T = 998) and 16 x 20 s (T = 1998), the fabricated checkpoint (seed 0). For each, in one process
and alternating round by round (host clock around `steps` calls that end in a device synchronise):
  native      DecoarExpert(all_layers=True): fbank + CMVN kernels, GEMMs for post_extract_proj and the input
              projections, the grid-resident recurrence kernel (lstm.cu) for every layer and direction
  reference   the reference's own s3prl.upstream.decoar_layers.expert.UpstreamExpert on the GPU (torchaudio fbank per
              utterance, packed cuDNN LSTMs), loaded from the same checkpoint, same batch; needs oracle/_ref
  cudnn_lstm  post_extract_proj and the two 4-layer stacks as torch.nn.Linear / torch.nn.LSTM (cuDNN) on the same
              precomputed features: the model without its front end, cuDNN's LSTM in place of lstm.cu
Then one profiled pass of the native model (device ms per step by category, s3b_profile_read_ex; category 5 is the
recurrence kernel). The card name and power limit head the output: a time means nothing without them.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))

CATEGORIES = ("gemm", "attention", "frontend", "layernorm", "misc", "recurrence")


def card():
    import torch

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - the report still names the card
        q = f"nvidia-smi unavailable ({e})"
    return torch.cuda.get_device_name(0), q


def reference_expert(sd):
    import torch

    import ref_runtime

    if ref_runtime.reference_root() is None:
        return None
    ref_runtime.activate()
    from s3prl.upstream.decoar_layers.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"model": sd}, tmp.name)
        ex = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    return ex.eval().cuda()


class CudnnLstm:
    """post_extract_proj and the two LSTM stacks (torch.nn.LSTM, cuDNN) on precomputed padded features; the backward
    stack runs on the time-reversed features, as for utterances that fill the batch."""

    def __init__(self, sd):
        import torch

        self.proj = torch.nn.Linear(80, 1024).cuda().eval()
        self.proj.load_state_dict({k.split(".", 1)[1]: v for k, v in sd.items() if k.startswith("post_extract_proj.")})
        self.stacks = []
        for d in ("forward", "backward"):
            lstm = torch.nn.LSTM(1024, 1024, num_layers=4, batch_first=True)
            lstm.load_state_dict({k.split(".", 1)[1]: v for k, v in sd.items() if k.startswith(f"{d}_lstm.")})
            self.stacks.append(lstm.cuda().eval())

    def __call__(self, feats, lens):
        from torch.nn.utils.rnn import pack_padded_sequence

        x = self.proj(feats)
        outs = []
        for d, lstm in enumerate(self.stacks):
            xi = x.flip(1) if d == 1 else x
            y, _ = lstm(pack_padded_sequence(xi, lens, batch_first=True, enforce_sorted=False))
            outs.append(y)
        return outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.decoar import DecoarExpert, fabricate_decoar_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("tools/decoar_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    lib = s3lib.load()
    ok = C.c_int32(0)
    s3lib.check(lib.s3b_lstm_fits(C.byref(ok)))
    print(f"# recurrence kernel: s3b_lstm_fits = {ok.value} (128 co-resident CTAs, one per SM)")
    sd = fabricate_decoar_state_dict(0)
    native = DecoarExpert(all_layers=True, seed=0).to("cuda")
    ref = reference_expert(sd)
    if ref is None:
        print("# reference: not installed under oracle/_ref; its row is skipped")
    cudnn = CudnnLstm(sd)
    for batch, seconds in ((32, 10.0), (16, 20.0)):
        L = int(seconds * 16000)
        g = torch.Generator(device="cuda").manual_seed(0)
        wavs = [torch.randn(L, device="cuda", generator=g) for _ in range(batch)]
        T = native.num_frames(L)
        feats = torch.randn(batch, T, 80, device="cuda", generator=g)
        lens = [T] * batch
        impls = {"native": lambda: native(wavs), "cudnn_lstm": lambda: cudnn(feats, lens)}
        if ref is not None:
            impls["reference"] = lambda: ref(wavs)
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
            print(f"{k:11s} " + " ".join(f"{t:9.2f}" for t in ts))
        h = native._native
        s3lib.check(h.lib.s3b_profile_enable(h.handle, 1))
        with torch.no_grad():
            for _ in range(args.steps):
                native(wavs)
        ms, fl, ln = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
        s3lib.check(h.lib.s3b_profile_read_ex(h.handle, 6, ms, fl, ln, 1))
        s3lib.check(h.lib.s3b_profile_enable(h.handle, 0))
        print("# native, profiled pass (launches timed one by one), device ms per step by category")
        print(" ".join(f"{c:>10s}" for c in CATEGORIES) + "      total  launches")
        print(" ".join(f"{ms[i] / args.steps:10.3f}" for i in range(6)) +
              f" {sum(ms) / args.steps:10.3f}  {sum(ln) // args.steps}")
        rec_ms = ms[5] / args.steps
        print(f"# recurrence: {rec_ms / (sum(ms) / args.steps):.1%} of device time; "
              f"{fl[5] / args.steps / (rec_ms * 1e-3) / 1e12:.2f} TFLOP/s (8 H^2 per frame and direction)")


if __name__ == "__main__":
    main()
