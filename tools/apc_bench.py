"""Step time and profile of APC (apc) against the reference expert and against cuDNN's GRU (GPU only).

    python tools/apc_bench.py [--steps 10] [--warmup 2] [--rounds 3]

Workloads: 32 x 10 s (T = 998) and 16 x 20 s (T = 1998), the fabricated checkpoint (seed 0, residual). For each, in one
process and alternating round by round (host clock around `steps` calls that end in a device synchronise):
  native     ApcExpert: fbank + CMVN kernels, one GEMM per layer, the cluster recurrence kernel (gru.cu)
  reference  the reference's own s3prl.upstream.apc.expert.UpstreamExpert on the GPU (torchaudio fbank per utterance,
             packed cuDNN GRUs), loaded from the same checkpoint, same batch; needs the install under oracle/_ref
  cudnn_gru  three torch.nn.GRU(batch_first) layers with the residual on the same packed features: the model without
             its front end, cuDNN's recurrence in place of gru.cu
Then one profiled pass of the native model (device ms per step by category, s3b_profile_read_ex; category 5 is the
recurrence kernel) and cudaOccupancyMaxActiveClusters of the recurrence kernel. The card name and power limit head the
output: a time means nothing without them.
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


def reference_expert(sd, config):
    import torch

    import ref_runtime

    if ref_runtime.reference_root() is None:
        return None
    ref_runtime.activate()
    from s3prl.upstream.apc.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"config": config, "model": sd}, tmp.name)
        ex = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    return ex.eval().cuda()


class CudnnGru:
    """The APC GRU stack as torch.nn.GRU layers (cuDNN) on precomputed padded features."""

    def __init__(self, sd):
        import torch

        self.layers = []
        for l in range(3):
            gru = torch.nn.GRU(80 if l == 0 else 512, 512, batch_first=True)
            gru.load_state_dict({k.split(".", 2)[2]: v for k, v in sd.items() if k.startswith(f"rnn_layers.{l}.")})
            self.layers.append(gru.cuda().eval())

    def __call__(self, feats, lens):
        from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

        x, T, out = feats, feats.size(1), []
        for l, gru in enumerate(self.layers):
            y, _ = gru(pack_padded_sequence(x, lens, batch_first=True, enforce_sorted=False))
            y, _ = pad_packed_sequence(y, batch_first=True, total_length=T)
            if l > 0:
                y = y + x
            out.append(y)
            x = y
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch

    from s3prl_b200 import lib as s3lib
    from s3prl_b200.upstream.apc import ApcExpert, apc_config, fabricate_apc_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("tools/apc_bench.py needs a CUDA device")
    name, power = card()
    print(f"# {name}  power.limit, clocks.max.sm: {power}")
    lib = s3lib.load()
    n = C.c_int32(0)
    s3lib.check(lib.s3b_gru_max_active_clusters(C.byref(n)))
    print(f"# recurrence kernel: cudaOccupancyMaxActiveClusters = {n.value} clusters of 16 CTAs (4 utterances each)")
    sd = fabricate_apc_state_dict(0)
    native = ApcExpert(seed=0).to("cuda")
    ref = reference_expert(sd, apc_config())
    if ref is None:
        print("# reference: not installed under oracle/_ref; its row is skipped")
    cudnn = CudnnGru(sd)
    for batch, seconds in ((32, 10.0), (16, 20.0)):
        L = int(seconds * 16000)
        g = torch.Generator(device="cuda").manual_seed(0)
        wavs = [torch.randn(L, device="cuda", generator=g) for _ in range(batch)]
        T = native.num_frames(L)
        feats = torch.randn(batch, T, 80, device="cuda", generator=g)
        lens = [T] * batch
        impls = {"native": lambda: native(wavs), "cudnn_gru": lambda: cudnn(feats, lens)}
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
        print(" ".join(f"{c:>10s}" for c in CATEGORIES) + "      total  launches")
        print(" ".join(f"{ms[i] / args.steps:10.3f}" for i in range(6)) +
              f" {sum(ms) / args.steps:10.3f}  {sum(ln) // args.steps}")


if __name__ == "__main__":
    main()
