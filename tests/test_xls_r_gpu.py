"""GPU tests of XLS-R 1B / 2B (80- and 120-wide attention heads, 1920-channel encoders): attention at head widths 64, 80
and 120 and at LightHuBERT's 6, 8 and 10 heads of 64, the QKV scatter epilogue at the same heads, the positional conv
with 80- and 120-channel groups and LayerNorm(1920) at block level against fp64 torch, and the whole model against the
executed-reference goldens (tests/golden/xls_r_*.pt) and the CPU oracle on ragged batches, with determinism across
lanes, shards and a converted checkpoint.
Bounds: blocks 1e-4 relative Frobenius and 2e-4 of the output scale elementwise (the operand planes carry ~16
significant bits), as tests/test_blocks_gpu.py; the model the golden bars of tests/test_upstream_gpu.py (2e-4 per layer,
1e-3 of the layer's abs max). Every check prints measured / bound."""
import ctypes as C
import math
import os
import sys
from dataclasses import replace
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"

pytestmark = pytest.mark.gpu

REL_TOL = 2e-4
ABS_FRAC = 1e-3
BLOCK_REL = 1e-4
BLOCK_ABS = 2e-4
LOG2E = 1.4426950408889634


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _check_block(out, ref, what):
    assert torch.isfinite(out).all(), what
    rel = _rel(out, ref)
    mx = (out.double() - ref.double()).abs().max().item() / ref.abs().max().item()
    print(f"{what}: rel/bound={rel / BLOCK_REL:.3f} maxabs/bound={mx / BLOCK_ABS:.3f}")
    assert rel < BLOCK_REL, (what, rel)
    assert mx < BLOCK_ABS, (what, mx)


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _attention(q, k, v, valid, H, hd, ctx_format):
    from s3prl_b200 import lib

    B, T, _ = q.shape
    out = torch.full_like(q, float("nan"))
    opts = lib.S3BAttentionOpts(ctx_format=ctx_format, head_dim=hd)
    vf = (C.c_int32 * B)(*valid)
    lib.check(lib.load().s3b_attention_ex(_ptr(q), _ptr(k), _ptr(v), vf, B, T, H, C.byref(opts), _ptr(out), _stream()))
    torch.cuda.synchronize()
    return out


# (H, hd); H = 6, 8, 10: the LightHuBERT subnets; 16 heads of 80 / 120: XLS-R 1B / 2B as served
HEADS = [(3, 64), (3, 80), (3, 120), (6, 64), (8, 64), (10, 64), (16, 80), (16, 120)]
HEAD_IDS = ["64", "80", "120", "h6-64", "h8-64", "h10-64", "h16-80", "h16-120"]


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("H,hd", HEADS, ids=HEAD_IDS)
@pytest.mark.parametrize("T", [1, 37, 63, 64, 65, 127, 128, 129, 999])
def test_attention_head_widths(s3b_lib, T, H, hd, fmt):
    """Ragged valid lengths: T, about 2T / 3, T rounded down to a multiple of 64 (a whole number of key blocks), 1."""
    B = 4
    valid = [T, max(1, (2 * T) // 3), max(1, T - T % 64), 1]
    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(T * 10 + hd + fmt + 1000 * H)
    q, k, v = (torch.randn(B, T, D, device="cuda", generator=g) for _ in range(3))
    out = _attention(q, k, v, valid, H, hd, fmt)
    qh, kh, vh = (t.double().view(B, T, H, hd).transpose(1, 2) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) * hd**-0.5
    mask = torch.arange(T, device="cuda")[None, :] >= torch.tensor(valid, device="cuda")[:, None]
    s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    ref = (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, T, D)
    _check_block(out, ref, f"attention H={H} hd={hd} T={T} valid={valid} ctx_format={fmt}")


def test_attention_refusals(s3b_lib):
    from s3prl_b200 import lib

    for hd in (48, 96, 128):
        x = torch.zeros(1, 8, 2 * hd, device="cuda")
        with pytest.raises(lib.S3BError, match="head_dim"):
            _attention(x, x, x, [8], 2, hd, 0)
    emb = torch.zeros(320, 2, device="cuda")
    x = torch.zeros(1, 8, 160, device="cuda")
    opts = lib.S3BAttentionOpts(head_dim=80, num_buckets=320, max_distance=800)
    opts.rel_emb = emb.data_ptr()
    out = torch.empty_like(x)
    r = lib.load().s3b_attention_ex(_ptr(x), _ptr(x), _ptr(x), (C.c_int32 * 1)(8), 1, 8, 2, C.byref(opts), _ptr(out),
                                    _stream())
    assert r != 0 and b"head_dim 64" in lib.load().s3b_last_error()


# ------------------------------------------------------------------------------------------------
# QKV scatter epilogue
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("H,hd", [(16, 80), (16, 120), (6, 64), (8, 64), (10, 64)],
                         ids=["80", "120", "h6-64", "h8-64", "h10-64"])
@pytest.mark.parametrize("T", [1, 37, 130])
def test_qkv_scatter(s3b_lib, T, H, hd, scheme):
    """q, k as [B][H][T][hd] (q scaled by hd^-0.5 * log2(e)) and v^T as [B][H][hd][Tp], Tp = T rounded up to 8; the
    padding columns of v^T stay zero. XLS-R's 16 heads of 80 and 120, LightHuBERT's 6, 8 and 10 heads of 64."""
    from s3prl_b200 import lib

    B = 2
    D, Tp = H * hd, (T + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(T + hd + scheme + 100 * H)
    x = torch.randn(B, T, D, device="cuda", generator=g)
    w = torch.randn(3 * D, D, device="cuda", generator=g) / D**0.5
    b = torch.randn(3 * D, device="cuda", generator=g) * 0.1
    q = torch.full((B, H, T, hd), float("nan"), device="cuda")
    k = torch.full_like(q, float("nan"))
    vt = torch.full((B, H, hd, Tp), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_qkv_hd_f32(_ptr(x), _ptr(w), _ptr(b), B, T, H, hd, scheme, _ptr(q), _ptr(k), _ptr(vt),
                                     _stream()))
    torch.cuda.synchronize()
    y = (x.double() @ w.double().t() + b.double()).view(B, T, 3, H, hd)
    scale = float(torch.tensor(LOG2E / math.sqrt(hd), dtype=torch.float32))
    _check_block(q, y[:, :, 0].transpose(1, 2) * scale, f"qkv q H={H} hd={hd} T={T} scheme={scheme}")
    _check_block(k, y[:, :, 1].transpose(1, 2), f"qkv k H={H} hd={hd} T={T} scheme={scheme}")
    _check_block(vt[..., :T], y[:, :, 2].permute(0, 2, 3, 1), f"qkv v^T H={H} hd={hd} T={T} scheme={scheme}")
    assert torch.equal(vt[..., T:], torch.zeros_like(vt[..., T:]))


# ------------------------------------------------------------------------------------------------
# positional conv and LayerNorm(1920)
# ------------------------------------------------------------------------------------------------
def _posconv(x, w, bias, G, k, gamma=None, beta=None, out_fmt=-1):
    from s3prl_b200 import lib

    B, T, D = x.shape
    out = torch.full((B, T, D), float("nan"), device="cuda")
    lib.check(lib.load().s3b_posconv_f32(_ptr(x), _ptr(w), _ptr(bias), B, T, D, G, k, 1, 0, _ptr(gamma), _ptr(beta),
                                         out_fmt, _ptr(out), _stream()))
    torch.cuda.synchronize()
    return out


WIDE_GROUP_DIMS = [1280, 1920]  # D of 16 groups of 80 / 120 channels: XLS-R 1B / 2B


@pytest.mark.parametrize("T", [1, 37, 63, 130, 999])
@pytest.mark.parametrize("D", WIDE_GROUP_DIMS)
def test_posconv_wide_groups(s3b_lib, D, T):
    """x + GELU(grouped conv(x) + b), 16 groups of 80 / 120 channels, k = 128 (SamePad drops the last frame), with and
    without the LayerNorm, in fp32 and in both operand-plane formats (planes only through the LayerNorm)."""
    G, k, B = 16, 128, 2
    cpg = D // G
    g = torch.Generator(device="cuda").manual_seed(D + T)
    x = torch.randn(B, T, D, device="cuda", generator=g)
    w = torch.randn(D, cpg, k, device="cuda", generator=g) / (cpg * k) ** 0.5
    bias = torch.randn(D, device="cuda", generator=g) * 0.2
    conv = F.conv1d(x.double().transpose(1, 2), w.double(), bias.double(), padding=k // 2, groups=G)[..., :T]
    ref = x.double() + F.gelu(conv.transpose(1, 2))
    _check_block(_posconv(x, w, bias, G, k), ref, f"posconv D={D} T={T}")
    gamma = 1.0 + 0.3 * torch.randn(D, device="cuda", generator=g)
    beta = 0.3 * torch.randn(D, device="cuda", generator=g)
    ref_ln = F.layer_norm(ref, (D,), gamma.double(), beta.double(), 1e-5)
    out = _posconv(x, w, bias, G, k, gamma, beta)
    _check_block(out, ref_ln, f"posconv+LN D={D} T={T}")
    for fmt in (0, 1):
        planes = _posconv(x, w, bias, G, k, gamma, beta, out_fmt=fmt)
        _check_block(planes, ref_ln, f"posconv+LN planes fmt={fmt} D={D} T={T}")


def test_posconv_groups_stay_apart(s3b_lib):
    """Groups 100x apart in magnitude, each checked against its own scale: an output column landing in the neighbouring
    group, or a read of the next group's channels meeting a non-zero weight, shows as an error of the neighbour's size."""
    D, G, k, B, T = 1920, 16, 128, 1, 77
    cpg = D // G
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, T, D, device="cuda", generator=g)
    x.view(B, T, G, cpg).mul_(torch.tensor([100.0 if i % 2 else 0.01 for i in range(G)], device="cuda").view(1, 1, G, 1))
    w = torch.randn(D, cpg, k, device="cuda", generator=g) / (cpg * k) ** 0.5
    bias = torch.zeros(D, device="cuda")
    out = _posconv(x, w, bias, G, k) - x
    conv = F.conv1d(x.double().transpose(1, 2), w.double(), None, padding=k // 2, groups=G)[..., :T]
    ref = F.gelu(conv.transpose(1, 2))
    for gi in range(G):
        sl = slice(gi * cpg, (gi + 1) * cpg)
        _check_block(out[..., sl], ref[..., sl], f"posconv group {gi}")


LAYERNORM_WIDE_D = 1920  # XLS-R 2B's encoder LayerNorms (eps 1e-5)


@pytest.mark.parametrize("gelu", [0, 1])
def test_layernorm_1920(s3b_lib, gelu):
    from s3prl_b200 import lib

    M, D = 333, LAYERNORM_WIDE_D
    g = torch.Generator(device="cuda").manual_seed(gelu)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 1
    gamma = 1.0 + 0.3 * torch.randn(D, device="cuda", generator=g)
    beta = 0.3 * torch.randn(D, device="cuda", generator=g)
    out = torch.full_like(x, float("nan"))
    lib.check(s3b_lib.s3b_layernorm_f32(_ptr(x), M, D, _ptr(gamma), _ptr(beta), gelu, _ptr(out), _stream()))
    torch.cuda.synchronize()
    ref = F.layer_norm(x.double(), (D,), gamma.double(), beta.double(), 1e-5)
    if gelu:
        ref = F.gelu(ref)
    _check_block(out, ref, f"layernorm 1920 gelu={gelu}")


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


_EXPERT = {}


def _expert(name, layers, scheme):
    from s3prl_b200.upstream.configs import XLS_R
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    key = (name, layers, scheme)
    if key not in _EXPERT:
        _EXPERT.clear()
        torch.cuda.empty_cache()
        saved = os.environ.get("S3B_GEMM_SCHEME")
        if scheme is not None:
            os.environ["S3B_GEMM_SCHEME"] = scheme
        try:
            cfg = XLS_R[name] if layers is None else replace(XLS_R[name], encoder_layers=layers)
            ex = UpstreamExpert(name="wav2vec2_local", arch=cfg, state_dict=fabricate_state_dict(cfg, seed=0)).to("cuda")
            ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
            _EXPERT[key] = ex
        finally:
            if scheme is not None:
                if saved is None:
                    os.environ.pop("S3B_GEMM_SCHEME", None)
                else:
                    os.environ["S3B_GEMM_SCHEME"] = saved
    return _EXPERT[key]


def _compare_layers(hs, ref, what):
    assert len(hs) == len(ref)
    worst = 0.0
    for l, (h, r) in enumerate(zip(hs, ref)):
        h = h.cpu()
        assert h.shape == r.shape and torch.isfinite(h).all(), (what, l)
        rel = _rel(h, r)
        mx = (h.double() - r.double()).abs().max().item() / r.abs().max().item()
        assert rel < REL_TOL, (what, l, rel)
        assert mx < ABS_FRAC, (what, l, mx)
        worst = max(worst, rel)
    print(f"{what}: worst per-layer relative error {worst:.3e} (measured/bound {worst / REL_TOL:.3f})")


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("lens", [[40000, 33333, 900], [16000, 50, 399]])
@pytest.mark.parametrize("name", ["xls_r_1b", "xls_r_2b"])
def test_matches_oracle_ragged(s3b_lib, name, lens, scheme):
    """4-layer variants against the CPU oracle (oracle/upstream_oracle.py), in the default scheme and in bf16x3."""
    sys.path.insert(0, str(ROOT / "oracle"))
    import upstream_oracle as O

    from s3prl_b200.upstream.weights import fabricate_state_dict

    ex = _expert(name, 4, scheme)
    wavs = _wavs(lens, seed=1234)
    with torch.no_grad():
        ref, _pad = O.upstream_forward(wavs, fabricate_state_dict(ex.arch, seed=0), ex.arch)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    _compare_layers(hs, ref, f"{name} 4 layers scheme={scheme or 'default'} lens={lens}")


@pytest.mark.parametrize("fixture", ["xls_r_1b", "xls_r_2b", "xls_r_1b_c3", "xls_r_2b_c3"])
def test_matches_reference_golden(s3b_lib, fixture):
    """The full 48-layer models (fabricated checkpoint, default scheme) against the executed reference
    (tools/make_xls_r_golden.py), with the bars of tests/test_upstream_gpu.py's golden test."""
    fx = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ex = _expert(fx["arch"], None, None)
    cs, ts = fx["channel_stride"], fx.get("time_stride", 1)
    worst = 0.0
    for case in fx["cases"]:
        hs = ex([w.cuda() for w in _wavs(case["lens"], case["wav_seed"])])["hidden_states"]
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu()
            ref = case["sub"][l]
            assert torch.isfinite(sub).all()
            rel = _rel(sub, ref)
            assert rel < REL_TOL, (fixture, l, rel)
            assert (sub.double() - ref.double()).abs().max().item() < ABS_FRAC * ref.abs().max().item(), (fixture, l)
            assert abs(h.double().norm().item() - case["norms"][l].item()) < REL_TOL * case["norms"][l].item()
            worst = max(worst, rel)
    print(f"{fixture}: worst per-layer relative error vs reference golden {worst:.3e} "
          f"(measured/bound {worst / REL_TOL:.3f})")


@pytest.mark.parametrize("name", ["xls_r_1b", "xls_r_2b"])
def test_lanes_shards_and_converted_file_are_bit_identical(s3b_lib, name, tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.convert import save_converted_checkpoint
    from s3prl_b200.upstream.weights import fabricate_state_dict

    ex = _expert(name, 4, None)
    lens = [48000, 40000, 33333, 900]
    wavs = [w.cuda() for w in _wavs(lens, seed=99)]
    ex.lanes = 1
    one = torch.stack(ex(wavs)["hidden_states"])
    ex.lanes = 2
    two = torch.stack(ex(wavs)["hidden_states"])
    ex.lanes = 0
    assert torch.equal(one, two)
    ex.global_max_len = max(lens)
    try:
        for idx in ([0, 1], [2, 3], [3]):
            part = torch.stack(ex([wavs[i] for i in idx])["hidden_states"])
            assert torch.equal(part, one[:, idx]), idx
    finally:
        ex.global_max_len = None
    path = tmp_path / f"{name}.pt"
    save_converted_checkpoint(path, ex.arch, fabricate_state_dict(ex.arch, seed=0))
    local = hub.ENTRIES["wav2vec2_local"](str(path)).to("cuda")
    assert local.arch == ex.arch
    assert torch.equal(torch.stack(local(wavs)["hidden_states"]), torch.stack(ex(wavs)["hidden_states"]))
