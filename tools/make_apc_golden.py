"""Writes the golden vectors of APC / VQ-APC (tests/golden/apc_ref*.pt, vq_apc_ref.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_apc_golden.py [--only apc_ref]

The fabricated checkpoint (s3prl_b200.upstream.apc.fabricate_apc_state_dict, seed 0, with apc_config) is saved as the
reference's ``{"config", "model"}`` file and loaded by the reference's own ``s3prl.upstream.apc.expert.UpstreamExpert``
(its constructor, strict load_state_dict, forward and hooks); seeded waveforms go through ``expert(wavs)``. The format
is that of tools/make_decoar2_golden.py: strided sub-samples of every hidden state plus per-layer norms. The names are
neither architecture names nor c<N>_* names, so the generic golden tests leave these files to tests/test_apc_cpu.py
(CPU oracle) and tests/test_apc_gpu.py (the CUDA path).
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))

import ref_runtime  # noqa: E402

from s3prl_b200.upstream.apc import apc_config, fabricate_apc_state_dict  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
# fixture -> (vq, waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    "apc_ref": (False, [[16000, 12345, 560], [8000, 8000]], 16, 2),  # 560 samples: m = 2
    "apc_ref_c2": (False, [[160000, 100003]], 16, 16),  # 10 s: T = 998
    "vq_apc_ref": (True, [[16000, 9001]], 16, 2),
}


def reference_expert(vq: bool):
    ref_runtime.activate()
    from s3prl.upstream.apc.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"config": apc_config(vq=vq), "model": fabricate_apc_state_dict(0, vq)}, tmp.name)
        expert = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    expert.eval()
    return expert


def make_fixture(fixture: str) -> None:
    vq, lens_cases, cstride, tstride = FIXTURES[fixture]
    expert = reference_expert(vq)
    out = {"arch": "vq_apc" if vq else "apc", "vq": vq, "weight_seed": 0, "channel_stride": cstride,
           "time_stride": tstride, "cases": []}
    for ci, lens in enumerate(lens_cases):
        g = torch.Generator().manual_seed(200 + ci)
        wavs = [torch.randn(n, generator=g) for n in lens]
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 200 + ci,
                "shape": tuple(hs[0].shape),
                "num_hidden": len(hs),
                "names": list(res["_hidden_states_info"]),
                "sub": torch.stack([h[:, (h.shape[1] - 1) % tstride :: tstride, ::cstride].contiguous() for h in hs]),
                "norms": torch.tensor([h.double().norm().item() for h in hs]),
                "abs_max": torch.tensor([h.abs().max().item() for h in hs]),
            }
        )
        print(f"{fixture} case {ci}: lens={lens} -> {len(hs)} x {tuple(hs[0].shape)}", flush=True)
    torch.save(out, GOLDEN / f"{fixture}.pt")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None, choices=sorted(FIXTURES))
    args = ap.parse_args()
    GOLDEN.mkdir(parents=True, exist_ok=True)
    for fixture in FIXTURES:
        if args.only in (None, fixture):
            make_fixture(fixture)


if __name__ == "__main__":
    main()
