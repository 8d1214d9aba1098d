"""Writes the golden vectors of DeCoAR 2.0 (tests/golden/decoar2_ref*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_decoar2_golden.py [--only decoar2_ref]

The fabricated checkpoint (s3prl_b200.upstream.decoar2.fabricate_decoar2_state_dict, seed 0) is saved as the
reference's ``{"model": state_dict}`` file and loaded by the reference's own
``s3prl.upstream.decoar2.expert.UpstreamExpert`` (its constructor, load_state_dict, forward and hooks); seeded waveforms
go through ``expert(wavs)``. The format is that of oracle/make_golden.py's model fixtures: strided sub-samples of every
hidden state plus per-layer norms. The names are neither architecture names nor c<N>_* names, so the generic golden
tests leave these files to tests/test_decoar2_cpu.py (CPU oracle) and tests/test_decoar2_gpu.py (the CUDA path).
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

from s3prl_b200.upstream.decoar2 import fabricate_decoar2_state_dict  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
# fixture -> (waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    "decoar2_ref": ([[16000, 12345, 800], [8000, 8000]], 14, 1),  # 800 samples: T_b = 2
    "decoar2_ref_c2": ([[160000, 100003]], 14, 8),  # 10 s: T = 499
}


def reference_expert(sd):
    ref_runtime.activate()
    from s3prl.upstream.decoar2.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"model": sd}, tmp.name)
        expert = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    missing = set(expert.model.state_dict()) ^ set(sd)
    assert not missing, f"fabricated keys differ from Decoar2().state_dict(): {sorted(missing)[:5]}"
    expert.eval()
    return expert


def make_fixture(fixture: str) -> None:
    lens_cases, cstride, tstride = FIXTURES[fixture]
    expert = reference_expert(fabricate_decoar2_state_dict(0))
    out = {"arch": "decoar2", "weight_seed": 0, "channel_stride": cstride, "time_stride": tstride, "cases": []}
    for ci, lens in enumerate(lens_cases):
        g = torch.Generator().manual_seed(100 + ci)
        wavs = [torch.randn(n, generator=g) for n in lens]
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 100 + ci,
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
