"""Compile-time guard for the GEMM kernel (no GPU needed): ptxas must neither serialise its wgmma instructions nor
spill registers. Either regression costs a large share of the GEMM's throughput without changing any result, so no
numerical test can see it."""
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
GEMM_SRC = ROOT / "s3prl_b200" / "csrc" / "gemm_sm90.cu"


FRONTEND_SRC = ROOT / "s3prl_b200" / "csrc" / "frontend.cu"


def _ptxas_report(tmp_path, src=GEMM_SRC):
    """ptxas -v output of a source compiled with the library's own flags (sm_90a)."""
    from s3prl_b200 import build

    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas=-v", "-c", str(src), "-o", str(tmp_path / (src.stem + ".o"))]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed:\n{r.stderr}"
    return r.stderr


def test_gemm_wgmma_not_serialised_and_no_spills(tmp_path):
    log = _ptxas_report(tmp_path)
    serialised = [ln for ln in log.splitlines() if "C7520" in ln]
    assert not serialised, "ptxas serialises wgmma instructions:\n" + "\n".join(serialised)
    _assert_no_spills(log)


def test_frontend_no_spills(tmp_path):
    """The front-end kernels (conv 0's fp64 moments among them) keep everything in registers."""
    _assert_no_spills(_ptxas_report(tmp_path, FRONTEND_SRC))


def _assert_no_spills(log):
    # per entry function: "Compiling entry function '<name>'" ... "N bytes spill stores, M bytes spill loads"
    spills, current, entries = [], None, 0
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", ln)
        if m:
            current, entries = m.group(1), entries + 1
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current is not None and (int(m.group(1)) or int(m.group(2))):
            spills.append(f"{current}: {ln.strip()}")
    assert entries > 0, "no ptxas report parsed:\n" + log[-2000:]
    assert not spills, "register spills:\n" + "\n".join(spills)
