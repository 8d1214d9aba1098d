"""Writes the golden vectors of the rotary Conformer (tests/golden/conformer_rope*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_conformer_golden.py [--only conformer_rope]

Same procedure and format as oracle/make_golden.py's model fixtures (its make_model_fixture does the work: the
fabricated checkpoint, loaded and run by the reference's own UpstreamExpert, strided samples of every hidden state).
The fixture names are neither architecture names nor c<N>_* names, so the generic golden tests leave them to
tests/test_conformer_cpu.py (CPU oracle) and tests/test_conformer_gpu.py (the CUDA path).
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))

import make_golden  # noqa: E402

# fixture -> (architecture, waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    "conformer_rope": ("wav2vec2_conformer_rope", [[12000, 7001]], 13, 1),
    # BASELINE C3 length (16 x 20 s -> T = 999) on the batch the CPU reference affords
    "conformer_rope_c3": ("wav2vec2_conformer_rope", [[320000, 271828]], 26, 16),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None, choices=sorted(FIXTURES))
    args = ap.parse_args()
    make_golden.GOLDEN.mkdir(parents=True, exist_ok=True)
    make_golden.FULL_SIZE.update(FIXTURES)
    for fixture in FIXTURES:
        if args.only in (None, fixture):
            make_golden.make_model_fixture(None, fixture)


if __name__ == "__main__":
    main()
