"""Writes the golden vectors of DeCoAR (tests/golden/decoar_ref.pt, decoar_layers_ref*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_decoar_golden.py [--only decoar_ref]

The fabricated checkpoint (s3prl_b200.upstream.decoar.fabricate_decoar_state_dict, seed 0) is saved as the reference's
``{"model": state_dict}`` file and loaded by the reference's own ``s3prl.upstream.decoar.expert.UpstreamExpert`` or
``s3prl.upstream.decoar_layers.expert.UpstreamExpert`` (constructor, key renaming, load_state_dict, forward); seeded
waveforms go through ``expert(wavs)``. The format is that of tools/make_apc_golden.py: strided sub-samples of every
hidden state plus per-layer norms. The names are neither architecture names nor c<N>_* names, so the generic golden
tests leave these files to tests/test_decoar_cpu.py (CPU oracle) and tests/test_decoar_gpu.py (the CUDA path).
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

from s3prl_b200.upstream.decoar import fabricate_decoar_state_dict  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
# fixture -> (all_layers, waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    "decoar_ref": (False, [[16000, 12345, 560], [8000, 8000]], 32, 2),  # 560 samples: m = 2
    "decoar_layers_ref": (True, [[16000, 12345, 560], [8000, 8000]], 32, 2),
    "decoar_layers_ref_c2": (True, [[160000, 100003]], 32, 16),  # 10 s: T = 998
}


def reference_expert(all_layers: bool):
    ref_runtime.activate()
    if all_layers:
        from s3prl.upstream.decoar_layers.expert import UpstreamExpert
    else:
        from s3prl.upstream.decoar.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"model": fabricate_decoar_state_dict(0)}, tmp.name)
        expert = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    expert.eval()
    return expert


def make_fixture(fixture: str) -> None:
    all_layers, lens_cases, cstride, tstride = FIXTURES[fixture]
    expert = reference_expert(all_layers)
    out = {"arch": "decoar_layers" if all_layers else "decoar", "all_layers": all_layers, "weight_seed": 0,
           "channel_stride": cstride, "time_stride": tstride, "cases": []}
    for ci, lens in enumerate(lens_cases):
        g = torch.Generator().manual_seed(300 + ci)
        wavs = [torch.randn(n, generator=g) for n in lens]
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        assert torch.equal(res["last_hidden_state"], res["hidden_states"][-1])
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 300 + ci,
                "shape": tuple(hs[0].shape),
                "num_hidden": len(hs),
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
