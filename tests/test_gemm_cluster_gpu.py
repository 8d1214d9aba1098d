"""Thread-block clusters in the 128-wide GEMM: the CTAs of a cluster take adjacent column tiles of the same rows and
load each A box once between them (TMA multicast). That changes where the operand bytes come from and nothing else, so
every output must be bit-identical to the launch without clusters (S3B_GEMM_CLUSTER=1), whatever the cluster size
(S3B_GEMM_CLUSTER=2 / 4, or the library's own choice with the variable unset).

Cases: the encoder linears of hubert_base, wav2vec2_large and the LightHuBERT subnets (some of an odd number of tiles,
where a forced cluster size falls back to 1), modified CPC's LSTM input GEMM, conv 1..6, NPC's tap convolutions (masked
ones too) and modified CPC's conv 1 and 4 (N = 256) in both operand schemes; M with a partial last row tile; conv batches whose
per-utterance row count is not a multiple of 128; n_tiles equal to the cluster size; launches with fewer clusters of
tiles than clusters that can be resident (M = 1, 129). Outputs start as NaN, so a tile that no cluster writes shows as
well."""
import pytest
import torch

import cpc_oracle as CO
from test_cpc_gpu import _cpc_conv
from test_gemm_layouts_gpu import _conv, _linear
from test_npc_gpu import _conv_inputs as _npc_inputs
from test_npc_gpu import _npc_conv

pytestmark = pytest.mark.gpu

SIZES = ["1", "2", "4", None]  # S3B_GEMM_CLUSTER; None = unset, the library's choice


def _runs(monkeypatch, fn):
    """fn() under every cluster setting; the outputs keyed by setting."""
    outs = {}
    for cn in SIZES:
        if cn is None:
            monkeypatch.delenv("S3B_GEMM_CLUSTER", raising=False)
        else:
            monkeypatch.setenv("S3B_GEMM_CLUSTER", cn)
        outs[cn] = fn()
    monkeypatch.delenv("S3B_GEMM_CLUSTER", raising=False)
    return outs


def _assert_identical(what, outs):
    base = outs["1"]
    assert torch.isfinite(base).all(), what
    for cn, out in outs.items():
        assert torch.equal(out, base), f"{what}: S3B_GEMM_CLUSTER={cn} differs from 1"


# (K, N): QKV, out_proj, fc1, fc2 of hubert_base and wav2vec2_large; N = 256 and 512 are n_tiles == 2 and 4; the same of
# LightHuBERT's 384-, 640- and 512-wide subnets, where N = 384, 1152, 640 and 1920 are an odd number of tiles (clusters
# of 2 or 4 fall back to 1); modified CPC's LSTM input GEMM
LINEAR_SHAPES = [(768, 2304), (768, 768), (768, 3072), (3072, 768), (1024, 3072), (1024, 1024), (1024, 4096),
                 (4096, 1024), (768, 256), (512, 512),
                 (384, 384), (384, 1152), (384, 1536), (1536, 384), (640, 640), (640, 1920), (640, 2560), (2560, 640),
                 (512, 1536), (512, 2048), (2048, 512), (256, 1024)]


@pytest.mark.parametrize("M", [1, 129, 1000, 4099])
@pytest.mark.parametrize("K,N", LINEAR_SHAPES)
@pytest.mark.parametrize("scheme", [0, 1])
def test_linear_clusters_bit_identical(s3b_lib, monkeypatch, scheme, K, N, M):
    """128-wide tiles in the epilogues of the encoder: bias + residual to fp32 (out_proj, fc2), bias + GELU to the
    scheme's operand planes (fc1)."""
    g = torch.Generator(device="cuda").manual_seed(M * 131 + K * 7 + N + scheme)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K**0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.5
    r = torch.randn(M, N, device="cuda", generator=g)

    def residual():
        out, o = _linear(a, w, b, r, scheme=scheme, tile_n=128)
        assert (o.scheme_used, o.tile_n_used) == (scheme, 128)
        return out

    def gelu_planes():
        return _linear(a, w, b, gelu=True, scheme=scheme, tile_n=128, out_fmt=scheme)[0]

    _assert_identical(f"linear s{scheme} M={M} K={K} N={N} residual", _runs(monkeypatch, residual))
    _assert_identical(f"linear s{scheme} M={M} K={K} N={N} gelu planes", _runs(monkeypatch, gelu_planes))


@pytest.mark.parametrize("Lout", [1, 129, 999])
@pytest.mark.parametrize("kw", [3, 2])
@pytest.mark.parametrize("scheme", [0, 1])
def test_conv_clusters_bit_identical(s3b_lib, monkeypatch, scheme, kw, Lout):
    """Conv1d(512, 512, kw, stride 2) over three utterances (N = 512: four 128-wide tiles), GELU to fp32 and to the
    scheme's operand planes, as conv 1..6 run it."""
    B = 3
    Lin = 2 * (Lout - 1) + kw + 1  # one sample more than Lout needs: the odd tail of a real conv input
    g = torch.Generator(device="cuda").manual_seed(Lout * 17 + kw + scheme)
    x = torch.randn(B, Lin, 512, device="cuda", generator=g)
    w = torch.randn(512, 512, kw, device="cuda", generator=g) / (512 * kw) ** 0.5
    bias = torch.randn(512, device="cuda", generator=g) * 0.1
    for out_fmt in (-1, scheme):
        _assert_identical(f"conv s{scheme} kw={kw} Lout={Lout} fmt={out_fmt}",
                          _runs(monkeypatch, lambda: _conv(x, w, bias, Lin, kw, True, scheme, out_fmt)))


@pytest.mark.parametrize("T", [129, 999])
@pytest.mark.parametrize("cin,k,mask", [(80, 3, 0), (512, 3, 0), (512, 1, 0), (512, 15, 7), (512, 15, 13)])
@pytest.mark.parametrize("scheme", [0, 1])
def test_npc_conv_clusters_bit_identical(s3b_lib, monkeypatch, scheme, cin, k, mask, T):
    """NPC's same-padded tap convolutions (N = 512: four 128-wide tiles) over three utterances, with the masked
    convs' skip over the band (a_gap), tanh and a residual added after it, as its blocks run them."""
    x, w, bias, res = _npc_inputs(T, cin, k, mask, "unit", T + cin + k + mask + scheme)
    _assert_identical(f"npc conv s{scheme} c_in={cin} k={k} mask={mask} T={T}",
                      _runs(monkeypatch, lambda: _npc_conv(s3b_lib, x, w, k, mask, bias, res, 2, 0, scheme)[0]))


@pytest.mark.parametrize("T", [129, 999])
@pytest.mark.parametrize("layer", [1, 4])
@pytest.mark.parametrize("scheme", [0, 1])
def test_cpc_conv_clusters_bit_identical(s3b_lib, monkeypatch, scheme, layer, T):
    """Modified CPC's strided conv 1 (k 8, stride 4) and conv 4 (k 4, stride 2) on the padded row layout, N = 256: two
    128-wide tiles, which f16q8 runs as a cluster of 2; then the ChannelNorm."""
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    L = s * (T - 1) + 2 * s - 2 * p + s - 1
    g = torch.Generator(device="cuda").manual_seed(T + layer + scheme)
    x = torch.relu(torch.randn(3, L, 256, device="cuda", generator=g))
    w = torch.randn(256, 256, 2 * s, device="cuda", generator=g) / (512 * s) ** 0.5
    bias, gamma, beta = (0.1 * torch.randn(256, device="cuda", generator=g),
                         0.5 + torch.rand(256, device="cuda", generator=g), 0.2 * torch.randn(256, device="cuda", generator=g))
    _assert_identical(f"cpc conv {layer} s{scheme} T={T}",
                      _runs(monkeypatch, lambda: _cpc_conv(s3b_lib, x, layer, w, bias, gamma, beta, scheme)))
