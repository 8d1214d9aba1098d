"""Writes the golden vectors of MAE-AST (tests/golden/mae_ast_*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_mae_ast_golden.py [--only mae_ast_frame]

The fabricated checkpoint (s3prl_b200.upstream.mae_ast.fabricate_mae_ast_state_dict) is saved as the reference's
``{"cfg", "model"}`` file and loaded by the reference's own ``s3prl.upstream.mae_ast.expert.UpstreamExpert`` (its
``MAE_AST`` with ``load_state_dict(strict=True)``, its fbank, padding mask and forward); seeded waveforms go through
``expert(wavs)``. The format is that of tools/make_ssast_golden.py: strided sub-samples of every hidden state plus
per-state norms and abs maxima, and the fabrication arguments.
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

from s3prl_b200.upstream.mae_ast import fabricate_mae_ast_state_dict  # noqa: E402

GOLDEN = ROOT / "tests" / "golden"
# n_b = 1 + (L - 400) // 160 frames. Frame model (kt 2): 16000 -> 99 (odd, a partly padded last patch), 9000 -> 54,
# 12345 -> 75 (odd), 400 -> 1 (one frame, one partly padded patch). Patch model (kt 16): 16000 -> 99 (a 3-frame last
# patch), 9000 -> 54, 5360 -> 32 (a multiple of 16), 400 -> 1.
_RAGGED = [[16000, 9000, 12345, 400], [5360, 16000]]
# every utterance as long as the longest: the reference's fast-exit mask
_EQUAL = [[16000, 16000, 16000], [4000, 4000]]
# fixture -> (kind, fabrication kwargs, waveform lengths per case, channel stride, time stride of the sub-sample). The
# channel strides are not divisors of 768, so the sub-sample visits many channels of each frequency patch.
FIXTURES = {
    "mae_ast_frame": ("frame", {}, _RAGGED, 37, 1),
    "mae_ast_patch": ("patch", {}, _RAGGED, 97, 1),
    "mae_ast_frame_c2": ("frame", {}, _EQUAL, 37, 1),
    "mae_ast_variant": ("patch", {"layers": 5, "layer_norm_first": True, "enc_sine_pos": False}, _RAGGED, 97, 1),
}
SEED = 0
MAX_TOKEN_LENGTH = 4096  # the table's rows; the released default (48000) only makes the file larger


def fabricate(kind: str, kwargs: dict) -> dict:
    return fabricate_mae_ast_state_dict(SEED, kind, max_token_length=MAX_TOKEN_LENGTH, **kwargs)


def reference_expert(kind: str, kwargs: dict):
    ref_runtime.activate()
    from s3prl.upstream.mae_ast.expert import UpstreamExpert

    tmp = tempfile.NamedTemporaryFile(suffix=".pt", delete=False)
    tmp.close()
    try:
        torch.save(fabricate(kind, kwargs), tmp.name)
        expert = UpstreamExpert(tmp.name)
    finally:
        os.unlink(tmp.name)
    expert.eval()
    return expert


def make_fixture(fixture: str) -> None:
    kind, kwargs, lens_cases, cstride, tstride = FIXTURES[fixture]
    expert = reference_expert(kind, kwargs)
    out = {"arch": "mae_ast", "kind": kind, "weight_seed": SEED, "fabricate": dict(kwargs),
           "max_token_length": MAX_TOKEN_LENGTH, "channel_stride": cstride, "time_stride": tstride, "cases": []}
    for ci, lens in enumerate(lens_cases):
        g = torch.Generator().manual_seed(900 + ci)
        wavs = [torch.randn(n, generator=g) * 0.1 for n in lens]
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 900 + ci,
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
