"""LightHuBERT on the GPU: the four-taps pos_conv at 24 and 40 channels per group and the LayerNorm at 384 / 640
against fp64, whole forwards of the four subnets against the executed reference's goldens and the fp64 oracle in
both operand schemes, hidden state 0's zeroed padding, and bit-identity across batch composition, lanes,
forward_host, repeats and a long-lived model."""
from __future__ import annotations

import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import lighthubert_oracle as LO  # noqa: E402
from test_gemm_layouts_gpu import _check, _pos_inputs, _posconv, _posconv_pipeline, _posconv_refs  # noqa: E402

pytestmark = pytest.mark.gpu

REL_TOL = 2e-4  # relative Frobenius error per hidden state, as tests/test_upstream_gpu.py
ELEM_TOL = 1e-3  # per element, relative to the state's absolute maximum
GOLDENS = ("lighthubert_small", "lighthubert_base", "lighthubert_stage1", "lighthubert_student_small",
           "lighthubert_small_c2", "lighthubert_variant_default", "lighthubert_variant_bias")


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _wavs(lens, seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) * scale for n in lens]


NARROW_POS_DIMS = [384, 640]  # D of 16 groups of 24 / 40 channels: the hubert_pruner subnets
NARROW_LN_DIMS = [384, 640]


@pytest.mark.parametrize("T", [1, 2, 127, 128, 998])
@pytest.mark.parametrize("D", NARROW_POS_DIMS)
@pytest.mark.parametrize("ln", [False, True])
def test_posconv_four_taps_narrow_groups(s3b_lib, D, T, ln):
    """x + GELU(grouped conv(k = 128) + b) (and the encoder LayerNorm) at 16 groups of 24 / 40 channels, four taps per
    k-block (96 / 160 GEMM columns, 2 / 3 k-steps of the 64-wide box), against F.conv1d in fp64 per element."""
    x, w, bias, g = _pos_inputs(2, T, D, 16, 128, D + T + 7 * ln)
    gamma = (1.0 + 0.3 * torch.randn(D, device="cuda", generator=g)) if ln else None
    beta = (0.3 * torch.randn(D, device="cuda", generator=g)) if ln else None
    out = _posconv(x, w, bias, 16, 128, 4, 0, gamma, beta)
    exact, emu, e1, e2 = _posconv_refs(x, w, 16, 128, 4)
    ref1, b1 = _posconv_pipeline(exact, e1, x, bias, 0, gamma, beta)
    ref2, b2 = _posconv_pipeline(emu, e2, x, bias, 0, gamma, beta)
    _check(f"posconv D={D} cpg={D // 16} taps=4 T={T} ln={ln}", out, ref1, b1, ref2, b2, (e1, e2), 0)


def test_posconv_narrow_groups_refuse_one_tap(s3b_lib):
    x = torch.zeros(1, 4, 384, device="cuda")
    w = torch.zeros(384, 24, 128, device="cuda")
    b = torch.zeros(384, device="cuda")
    r = s3b_lib.s3b_posconv_f32(x.data_ptr(), w.data_ptr(), b.data_ptr(), 1, 4, 384, 16, 128, 1, 0, None, None, -1,
                                x.data_ptr(), None)
    assert r != 0 and b"four taps" in s3b_lib.s3b_last_error()
    r = s3b_lib.s3b_posconv_f32(x.data_ptr(), w.data_ptr(), b.data_ptr(), 1, 4, 384, 16, 126, 4, 0, None, None, -1,
                                x.data_ptr(), None)
    assert r != 0 and b"multiple of 4" in s3b_lib.s3b_last_error()


@pytest.mark.parametrize("D", NARROW_LN_DIMS)
@pytest.mark.parametrize("gelu", [0, 1])
def test_layernorm_narrow(s3b_lib, D, gelu):
    from s3prl_b200 import lib

    M = 1000
    g = torch.Generator(device="cuda").manual_seed(D + gelu)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 5
    gm = 1 + 0.3 * torch.randn(D, device="cuda", generator=g)
    bt = 0.3 * torch.randn(D, device="cuda", generator=g)
    out = torch.empty_like(x)
    lib.check(s3b_lib.s3b_layernorm_f32(x.data_ptr(), M, D, gm.data_ptr(), bt.data_ptr(), gelu, out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x.double(), (D,), gm.double(), bt.double(), 1e-5)
    if gelu:
        ref = torch.nn.functional.gelu(ref)
    assert _rel(out, ref) < 2e-6


def _expert(scheme, **kw):
    from s3prl_b200.upstream.lighthubert import LighthubertExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        ex = LighthubertExpert(**kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


def _ckpt(tmp_path, cfg, seed):
    from s3prl_b200.upstream.lighthubert import fabricate_lighthubert_state_dict

    path = tmp_path / "lighthubert.pt"
    torch.save({"cfg": {"model": cfg}, "model": fabricate_lighthubert_state_dict(seed, cfg)}, path)
    return str(path)


def _assert_close(what, h, ref):
    err = _rel(h, ref)
    el = ((h.double() - ref.double()).abs().max() / ref.double().abs().max()).item()
    print(f"{what}: abs max {ref.abs().max().item():.3f}, relative error {err:.3e} (measured/bound "
          f"{err / REL_TOL:.3f}), element {el:.3e} (measured/bound {el / ELEM_TOL:.3f})")
    assert err < REL_TOL and el < ELEM_TOL, what


@pytest.mark.parametrize("scheme", ["f16q8", "bf16x3"])
@pytest.mark.parametrize("fixture", GOLDENS)
def test_matches_reference_golden(s3b_lib, tmp_path, fixture, scheme):
    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ex = _expert(scheme, ckpt=_ckpt(tmp_path, g["config"], g["weight_seed"]))
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        hs = ex([w.cuda() for w in _wavs(case["lens"], case["wav_seed"], case["wav_scale"])])["hidden_states"]
        assert len(hs) == case["num_hidden"] == 13 and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            _assert_close(f"{fixture} lens={case['lens']} {scheme} state {l}",
                          h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu(), case["sub"][l])


@pytest.mark.parametrize("scheme", ["f16q8", "bf16x3"])
@pytest.mark.parametrize("kind,over", [("small", {}), ("base", {}), ("stage1", {}), ("stage1", dict(supernet_type="small"))],
                         ids=["small", "base", "stage1", "student_small"])
def test_matches_oracle_ragged(s3b_lib, tmp_path, kind, over, scheme):
    """Ragged batch with odd T (T = 149 for 48000 samples), a ~400-sample utterance; hidden state 0's padded frames
    are exactly 0."""
    from s3prl_b200.upstream.lighthubert import (cut_subnet, fabricate_lighthubert_state_dict, lighthubert_config,
                                                 select_subnet, supernet_arch)

    cfg = lighthubert_config(kind, **over)
    ex = _expert(scheme, ckpt=_ckpt(tmp_path, cfg, 2))
    lens = [48000, 401, 31234, 16001, 47999, 9000]
    wavs = _wavs(lens, seed=11)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    _, sub = select_subnet(cfg)
    sd = cut_subnet(fabricate_lighthubert_state_dict(2, cfg), supernet_arch(cfg), sub)
    ref = LO.lighthubert_forward(wavs, sd, sub)
    T = hs[0].shape[1]
    assert T % 2 == 1 and len(hs) == len(ref) == 13
    for l, (h, r) in enumerate(zip(hs, ref)):
        _assert_close(f"ragged {kind}{over or ''} {scheme} state {l}", h.cpu(), r)
    chunk = max(lens) // T
    for b, n in enumerate(lens):
        v = -(-n // chunk)
        assert torch.all(hs[0][b, v:] == 0), b
        assert torch.all(hs[0][b, :v].abs().sum(-1) > 0), b


def test_bit_identical_batch_shards_lanes_host_repeats(s3b_lib):
    ex = _expert(None, kind="small")
    lens = [int(v) for v in torch.randint(400, 160000, (32,), generator=torch.Generator().manual_seed(3))]
    lens[5] = 160000
    wavs = [w.cuda() for w in _wavs(lens, seed=21)]
    full = torch.stack(ex(wavs)["hidden_states"]).clone()
    # an utterance alone, padded to the batch's max_len, vs inside the batch of 32
    ex.global_max_len = max(lens)
    for i in (0, 5, 17):
        alone = torch.stack(ex([wavs[i]])["hidden_states"])
        assert torch.equal(alone[:, 0], full[:, i]), i
    halves = [torch.stack(ex(wavs[s])["hidden_states"]) for s in (slice(0, 16), slice(16, 32))]
    assert torch.equal(torch.cat(halves, dim=1), full)
    ex.global_max_len = None
    for lanes in (1, 2):
        ex.lanes = lanes
        assert torch.equal(torch.stack(ex(wavs)["hidden_states"]), full), lanes
    ex.lanes = 0
    host = ex.forward_host([w.cpu() for w in wavs[:8]])
    dev8 = torch.stack(ex(wavs[:8])["hidden_states"]).cpu()
    assert torch.equal(host, dev8)
    # a long-lived model: other shapes in between, then the first batch again
    for n in (3, 17, 32):
        ex(wavs[:n])
    for _ in range(3):
        assert torch.equal(torch.stack(ex(wavs)["hidden_states"]), full)
    print("lighthubert_small: bit-identical across batch composition, lanes, forward_host and repeats")


def test_forward_ex_outputs(s3b_lib):
    """ffn_out is served under proj_hidden0: the fc2 outputs before the residual; the hidden states do not change."""
    ex = _expert(None, kind="base")
    wavs = [w.cuda() for w in _wavs([16000, 9001], seed=5)]
    native, ws, lens, max_len, T = ex._prepare(wavs)
    plain = ex._forward_ex(native, ws, lens, max_len, T)
    ffn = torch.empty((12, 2, T, 640), device="cuda")
    out = ex._forward_ex(native, ws, lens, max_len, T, ffn_out=ffn)
    assert torch.equal(out, plain) and torch.isfinite(ffn).all()
