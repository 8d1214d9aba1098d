"""Writes the golden vectors of LightHuBERT (tests/golden/lighthubert_*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_lighthubert_golden.py [--only lighthubert_small]

The fabricated supernet (s3prl_b200.upstream.lighthubert.fabricate_lighthubert_state_dict, seed 0) is saved as the
reference's ``{"cfg": {"model": ...}, "model": ...}`` file and loaded by the reference's own
``s3prl.upstream.lighthubert.expert.UpstreamExpert`` (its config, subnet choice, load_state_dict, set_sample_config
and forward); seeded waveforms go through ``expert(wavs)``. The format is that of tools/make_cpc_golden.py: strided
sub-samples of every hidden state plus per-state norms and abs maxima.
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

from s3prl_b200.upstream.lighthubert import fabricate_lighthubert_state_dict, lighthubert_config  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
_RAGGED = [[16000, 12345, 400], [8321, 8000]]  # T = 49 (odd) with a 1-frame utterance; T = 25 (odd)
# fixture -> (cfg["model"], waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    "lighthubert_small": (lighthubert_config("small"), _RAGGED, 32, 1),
    "lighthubert_base": (lighthubert_config("base"), _RAGGED, 32, 1),
    "lighthubert_stage1": (lighthubert_config("stage1"), _RAGGED, 32, 1),
    # student_hubert on a "small" supernet: max_subnet is 512 wide (local files only)
    "lighthubert_student_small": (lighthubert_config("stage1", supernet_type="small"), _RAGGED, 32, 1),
    "lighthubert_small_c2": (lighthubert_config("small"), [[160000, 100003]], 32, 8),  # 10 s: T = 499
    "lighthubert_variant_default": (lighthubert_config("small", extractor_mode="default"), [[16000, 9001]], 32, 1),
    "lighthubert_variant_bias": (lighthubert_config("base", conv_bias=True), [[16000, 9001]], 32, 1),
}


def reference_expert(cfg: dict):
    ref_runtime.activate()
    from s3prl.upstream.lighthubert.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save({"cfg": {"model": cfg}, "model": fabricate_lighthubert_state_dict(0, cfg)}, tmp.name)
        expert = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    expert.eval()
    return expert


def make_fixture(fixture: str) -> None:
    cfg, lens_cases, cstride, tstride = FIXTURES[fixture]
    expert = reference_expert(cfg)
    out = {"arch": "lighthubert", "config": cfg, "weight_seed": 0, "channel_stride": cstride, "time_stride": tstride,
           "cases": []}
    for ci, lens in enumerate(lens_cases):
        g = torch.Generator().manual_seed(500 + ci)
        wavs = [torch.randn(n, generator=g) * 0.1 for n in lens]
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 500 + ci,
                "wav_scale": 0.1,
                "shape": tuple(hs[0].shape),
                "num_hidden": len(hs),
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
