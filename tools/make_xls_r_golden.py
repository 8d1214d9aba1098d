"""Writes the golden vectors of XLS-R 1B / 2B (tests/golden/xls_r_*.pt) by EXECUTING THE REFERENCE.

Run where the reference (s3prl) is available:

    PYTHONPATH=/path/to/s3prl python tools/make_xls_r_golden.py [--only xls_r_1b]

Same procedure and format as oracle/make_golden.py's model fixtures (its make_model_fixture does the work: the
fabricated checkpoint, loaded and run by the reference's own UpstreamExpert, strided samples of every hidden state).
The XLS-R configurations are not hub entries, so this process registers them in its own copy of the architecture table
before the fixture code looks them up. The fixture names are neither architecture names nor c<N>_* names, so the
generic golden tests leave them to tests/test_xls_r_cpu.py (CPU oracle) and tests/test_xls_r_gpu.py (the CUDA path).

The 2B reference holds its fp32 weights several times over (fabricated state dict, the checkpoint file the reference
loads, the model): about 30 GB of host memory and 9 GB of temporary disk.
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))

import make_golden  # noqa: E402

from s3prl_b200.upstream.configs import ARCHS, XLS_R  # noqa: E402

# fixture -> (architecture, waveform lengths per case, channel stride, time stride of the sub-sample)
FIXTURES = {
    "xls_r_1b": ("xls_r_1b", [[12000, 7001]], 26, 1),
    "xls_r_2b": ("xls_r_2b", [[12000, 7001]], 38, 1),
    # BASELINE C3 length (16 x 20 s -> T = 999) on the batch the CPU reference affords
    "xls_r_1b_c3": ("xls_r_1b", [[320000, 271828]], 52, 16),
    "xls_r_2b_c3": ("xls_r_2b", [[320000, 271828]], 76, 16),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None, choices=sorted(FIXTURES))
    args = ap.parse_args()
    ARCHS.update(XLS_R)  # this process only: make_model_fixture and reference_expert look architectures up by name
    make_golden.GOLDEN.mkdir(parents=True, exist_ok=True)
    make_golden.FULL_SIZE.update(FIXTURES)
    for fixture in FIXTURES:
        if args.only in (None, fixture):
            make_golden.make_model_fixture(None, fixture)


if __name__ == "__main__":
    main()
