"""Block tests of non-GEMM kernel configurations that a served model runs and no other block table holds
(tests/test_kernel_coverage_cpu.py names them): the Conformer's depthwise conv at its served width, and the
positional conv's 32-column one-tap tiles (LightHuBERT student small: 16 groups of 32 channels) kept apart per group.
The positional conv's values at that configuration are checked against fp64 and the operand emulation by the rows of
test_gemm_layouts_gpu.POS_CONFIGS. Every check prints measured / bound."""
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent))

from test_conformer_gpu import DEPTHWISE_TS, _bn_params, _conv_native, _conv_ref  # noqa: E402
from test_conformer_gpu import _check_block as _check_rel  # noqa: E402
from test_gemm_layouts_gpu import _posconv  # noqa: E402
from test_xls_r_gpu import _check_block  # noqa: E402

pytestmark = pytest.mark.gpu

DEPTHWISE_SERVED = [(1024, 31)]  # (D, k): wav2vec2_conformer_rope's depthwise_conv_kernel_size at its encoder width
POS_APART = [(512, 16, 128)]  # (D, groups, k) of the one-tap tiles narrower than any other block test's


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("T", DEPTHWISE_TS)
@pytest.mark.parametrize("D,k", DEPTHWISE_SERVED)
def test_depthwise_served_width(s3b_lib, D, k, T, fmt):
    """GLU -> depthwise conv -> BatchNorm -> SiLU at the served (D, k), against fp64 with the bar of
    test_conformer_gpu.test_depthwise_block."""
    g = torch.Generator(device="cuda").manual_seed(T * 100 + k + D)
    x = torch.randn(2, T, 2 * D, device="cuda", generator=g)
    w = torch.randn(D, 1, k, device="cuda", generator=g) / k**0.5
    bn = _bn_params(D, g)
    out = _conv_native(s3b_lib, x, w, *bn, fmt)
    _check_rel(out, _conv_ref(x, w, *bn), f"depthwise D={D} T={T} k={k} fmt={fmt}")


@pytest.mark.parametrize("D,G,k", POS_APART)
def test_posconv_narrow_groups_stay_apart(s3b_lib, D, G, k):
    """test_xls_r_gpu.test_posconv_groups_stay_apart at 32 channels per group: groups 100x apart in magnitude, each
    checked against its own scale. The 64-wide A box of a tap reads the next group's 32 channels, which meet zero
    weights; an output column landing in the neighbouring group, or a non-zero weight there, shows as an error of the
    neighbour's size."""
    B, T = 1, 77
    cpg = D // G
    g = torch.Generator(device="cuda").manual_seed(D + k)
    x = torch.randn(B, T, D, device="cuda", generator=g)
    x.view(B, T, G, cpg).mul_(torch.tensor([100.0 if i % 2 else 0.01 for i in range(G)], device="cuda").view(1, 1, G, 1))
    w = torch.randn(D, cpg, k, device="cuda", generator=g) / (cpg * k) ** 0.5
    bias = torch.zeros(D, device="cuda")
    out = _posconv(x, w, bias, G, k, 1, 0) - x
    conv = F.conv1d(x.double().transpose(1, 2), w.double(), None, padding=k // 2, groups=G)[..., :T]
    ref = F.gelu(conv.transpose(1, 2))
    for gi in range(G):
        sl = slice(gi * cpg, (gi + 1) * cpg)
        _check_block(out[..., sl], ref[..., sl], f"posconv D={D} cpg={cpg} group {gi}")
