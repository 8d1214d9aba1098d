"""Step time and profile of modified CPC (modified_cpc) against the reference expert and against torch's conv1d stack
with cuDNN's LSTM (GPU only).

    python tools/cpc_bench.py [--steps 10] [--warmup 2] [--rounds 3]

Workloads: 32 x 10 s (T = 1000) and 16 x 20 s (T = 2000), the fabricated checkpoint (seed 0, cpc_config()). For each,
in one process and alternating round by round (host clock around `steps` calls that end in a device synchronise):
  native     CpcExpert: conv 0 + ChannelNorm kernel, conv 1..4 on the wgmma GEMM with a norm kernel each, the LSTM's
             input GEMM and the cluster-resident recurrence
  reference  the reference's own s3prl.upstream.cpc.expert.UpstreamExpert on the GPU (torch Conv1d + ChannelNorm,
             nn.LSTM on cuDNN), loaded from the same checkpoint, same batch; needs the install under oracle/_ref
  torch      the same weights in plain torch: F.conv1d + the ChannelNorm arithmetic + ReLU, then nn.LSTM (cuDNN),
             written here and independent of the reference install
Then one profiled pass of the native model (device ms per step by category, s3b_profile_read_ex), and the number of
8-CTA recurrence clusters the card can hold against the number a batch needs. The card name and power limit head the
output: a time means nothing without them.
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
    from s3prl.upstream.cpc.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"config": config, "weights": sd}, tmp.name)
        ex = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    return ex.eval().cuda()


def torch_model(sd, num_layers):
    """F.conv1d + ChannelNorm + ReLU and cuDNN's nn.LSTM on the fabricated weights (fp32)."""
    import torch
    import torch.nn.functional as F

    from s3prl_b200.upstream.cpc import PADDINGS, STRIDES

    w = {k: v.cuda() for k, v in sd.items()}
    lstm = torch.nn.LSTM(256, 256, num_layers=num_layers, batch_first=True).cuda().eval()
    lstm.load_state_dict({k[len("gAR.baseNet."):]: v for k, v in w.items() if k.startswith("gAR.baseNet.")})

    def run(wav_pad):
        x = wav_pad.unsqueeze(1)
        for i, (s, p) in enumerate(zip(STRIDES, PADDINGS)):
            x = F.conv1d(x, w[f"gEncoder.conv{i}.weight"], w[f"gEncoder.conv{i}.bias"], stride=s, padding=p)
            x = (x - x.mean(dim=1, keepdim=True)) * torch.rsqrt(x.var(dim=1, keepdim=True) + 1e-5)
            x = torch.relu(x * w[f"gEncoder.batchNorm{i}.weight"] + w[f"gEncoder.batchNorm{i}.bias"])
        enc = x.transpose(1, 2)
        return enc, lstm(enc)[0]

    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.cpc import CpcExpert, cpc_config, fabricate_cpc_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("tools/cpc_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    config = cpc_config()
    sd = fabricate_cpc_state_dict(0)
    native = CpcExpert(seed=0).to("cuda")
    ref = reference_expert(sd, config)
    plain = torch_model(sd, config["nLevelsGRU"])
    if ref is None:
        print("# reference: not installed under oracle/_ref; the reference row is skipped")
    for batch, seconds in ((32, 10.0), (16, 20.0)):
        L = int(seconds * 16000)
        g = torch.Generator(device="cuda").manual_seed(0)
        wavs = [torch.randn(L, device="cuda", generator=g) * 0.1 for _ in range(batch)]
        wav_pad = torch.stack(wavs)
        T = native.num_frames(L)
        impls = {"native": lambda: native(wavs), "torch": lambda: plain(wav_pad)}
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
            nat = native(wavs)["hidden_states"]
            tor = plain(wav_pad)
        err = [((a.double() - b.double()).norm() / b.double().norm()).item() for a, b in zip(nat, tor)]
        print(f"# {batch} x {seconds:g} s, T = {T}; ms per step, {args.rounds} alternating rounds of {args.steps} steps"
              f" (native vs torch, relative: encoder {err[0]:.2e}, LSTM {err[1]:.2e})")
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
        n = C.c_int32()
        s3lib.check(h.lib.s3b_cpc_lstm_max_active_clusters(C.byref(n)))
        print(f"# recurrence: {n.value} clusters of 8 CTAs co-resident; {(batch + 3) // 4} needed by {batch} utterances "
              "(4 per cluster); with two lanes each lane needs half")


if __name__ == "__main__":
    main()
