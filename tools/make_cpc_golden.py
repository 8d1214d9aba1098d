"""Writes the golden vectors of modified CPC (tests/golden/cpc_ref*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_cpc_golden.py [--only cpc_ref]

The fabricated checkpoint (s3prl_b200.upstream.cpc.fabricate_cpc_state_dict, seed 0) is saved as the reference's
``{"config", "weights"}`` file and loaded by the reference's own ``s3prl.upstream.cpc.expert.UpstreamExpert`` (its
constructor, config overlay, load_state_dict, forward and hooks); seeded waveforms go through ``expert(wavs)``. The
format is that of tools/make_npc_golden.py: strided sub-samples of every hidden state plus per-state norms and abs
maxima.
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

from s3prl_b200.upstream.cpc import cpc_config, fabricate_cpc_state_dict  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
# fixture -> (config overrides, waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    # 40 samples: an utterance shorter than one frame's receptive field; [159, 40]: T = 1
    "cpc_ref": ({}, [[16000, 12345, 100], [8000, 8000], [159, 40]], 16, 1),
    "cpc_ref_c2": ({}, [[160000, 100003]], 16, 8),  # 10 s: T = 1000
    "cpc_ref_variant": ({"nLevelsGRU": 2}, [[16000, 9001, 4000]], 16, 1),
}


def reference_expert(over: dict):
    ref_runtime.activate()
    from s3prl.upstream.cpc.expert import UpstreamExpert

    config = cpc_config(**over)
    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"config": config, "weights": fabricate_cpc_state_dict(0, config["nLevelsGRU"])}, tmp.name)
        expert = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    expert.eval()
    return expert


def make_fixture(fixture: str) -> None:
    over, lens_cases, cstride, tstride = FIXTURES[fixture]
    expert = reference_expert(over)
    out = {"arch": "cpc", "config": over, "weight_seed": 0, "channel_stride": cstride, "time_stride": tstride,
           "cases": []}
    for ci, lens in enumerate(lens_cases):
        g = torch.Generator().manual_seed(400 + ci)
        wavs = [torch.randn(n, generator=g) * 0.1 for n in lens]
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 400 + ci,
                "wav_scale": 0.1,
                "shape": tuple(hs[0].shape),
                "num_hidden": len(hs),
                "names": list(res["_hidden_states_info"]),
                "sub": torch.stack([h[:, (h.shape[1] - 1) % tstride :: tstride, ::cstride].contiguous() for h in hs]),
                "norms": torch.tensor([h.double().norm().item() for h in hs]),
                "abs_max": torch.tensor([h.abs().max().item() for h in hs]),
            }
        )
        print(f"{fixture} case {ci}: lens={lens} -> {len(hs)} x {tuple(hs[0].shape)}, abs max "
              f"{[round(v, 3) for v in out['cases'][-1]['abs_max'].tolist()]}", flush=True)
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
