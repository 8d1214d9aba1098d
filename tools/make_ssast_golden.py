"""Writes the golden vectors of SSAST (tests/golden/ssast_*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_ssast_golden.py [--only ssast_frame]

The fabricated checkpoint (s3prl_b200.upstream.ssast.fabricate_ssast_state_dict, seed 0) is saved as the reference's
DataParallel file and loaded by the reference's own ``s3prl.upstream.ssast.expert.UpstreamExpert`` (its ASTModel
constructor with the positional re-gridding, its windowing, FeatureExtractor and forward); seeded waveforms go through
``expert(wavs)``. timm is replaced by oracle/timm_shim.py when it is not installed, and each golden records whether it
was. The format is that of tools/make_lighthubert_golden.py: strided sub-samples of every hidden state plus per-state
norms and abs maxima.
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
import timm_shim  # noqa: E402

from s3prl_b200.upstream.ssast import fabricate_ssast_state_dict  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
# 1 s windows: a 1-sample utterance and the window-boundary lengths (nseg 2, T = 101); then an utterance that ends two
# windows before the longest (nseg 3)
_SHORT = [[16001, 1, 15999, 16000], [40000, 9000]]
# 10 s windows: one window, then two with the second utterance inside the first
_LONG = [[160000, 37000], [170000, 5000]]
# fixture -> (kind, window_secs, waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    "ssast_frame": ("frame", 1.0, _SHORT, 192, 1),
    "ssast_patch": ("patch", 1.0, _SHORT, 768, 1),
    "ssast_frame_w10": ("frame", 10.0, _LONG, 192, 8),
    "ssast_patch_w10": ("patch", 10.0, _LONG, 768, 2),
}


def reference_expert(kind: str, window_secs: float):
    ref_runtime.activate()
    shim = timm_shim.install()
    from s3prl.upstream.ssast.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pth", delete=False)
    tmp.close()
    try:
        torch.save(fabricate_ssast_state_dict(0, kind), tmp.name)
        expert = UpstreamExpert(tmp.name, "base_" + kind[0], window_secs)
    finally:
        os.unlink(tmp.name)
    expert.eval()
    return expert, shim


def make_fixture(fixture: str) -> None:
    kind, window_secs, lens_cases, cstride, tstride = FIXTURES[fixture]
    expert, shim = reference_expert(kind, window_secs)
    out = {"arch": "ssast", "kind": kind, "window_secs": window_secs, "weight_seed": 0, "timm_shim": shim,
           "channel_stride": cstride, "time_stride": tstride, "cases": []}
    for ci, lens in enumerate(lens_cases):
        g = torch.Generator().manual_seed(700 + ci)
        wavs = [torch.randn(n, generator=g) * 0.1 for n in lens]
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 700 + ci,
                "wav_scale": 0.1,
                "shape": tuple(hs[0].shape),
                "num_hidden": len(hs),
                "sub": torch.stack([h[:, (h.shape[1] - 1) % tstride :: tstride, ::cstride].contiguous() for h in hs]),
                "norms": torch.tensor([h.double().norm().item() for h in hs]),
                "abs_max": torch.tensor([h.abs().max().item() for h in hs]),
            }
        )
        print(f"{fixture} case {ci}: lens={lens} -> {len(hs)} x {tuple(hs[0].shape)} (timm shim: {shim}), abs max "
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
