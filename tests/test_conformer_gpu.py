"""GPU tests of the wav2vec 2.0 Conformer (rotary attention): its two new kernels and the SiLU GEMM epilogue at block
level against fp64 torch, the whole model against the executed-reference goldens (tests/golden/conformer_rope*.pt) and
against the CPU oracle (tests/conformer_oracle.py) on ragged batches (default scheme, bf16x3, a 2-layer post-LN
variant, a k = 15 variant), determinism across lanes and shards, and the refusals of layer-result outputs.
Bounds: single blocks 1e-4 relative Frobenius and 2e-4 of the output scale elementwise (the operand planes carry ~16
significant bits); the model the golden bars of tests/test_upstream_gpu.py (2e-4 per layer, 1e-3 of the abs max)."""
import ctypes as C
import sys
from dataclasses import replace
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
GOLDEN = ROOT / "tests" / "golden"

pytestmark = pytest.mark.gpu

REL_TOL = 2e-4
ABS_FRAC = 1e-3


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _check_block(out, ref, what):
    assert torch.isfinite(out).all(), what
    rel = _rel(out, ref)
    mx = (out.double() - ref).abs().max().item()
    print(f"{what}: rel={rel:.3e} maxabs/scale={mx / ref.abs().max().item():.3e}")
    assert rel < 1e-4, (what, rel)
    assert mx < 2e-4 * ref.abs().max().item(), (what, mx)


def _conv_ref(x, w, gamma, beta, mean, var):
    """GLU -> depthwise conv (zero padding per utterance) -> BatchNorm (eval) -> SiLU in fp64, channels-last."""
    x = x.double()
    D = w.size(0)
    u = F.glu(x, dim=-1).transpose(1, 2)
    u = F.conv1d(u, w.double(), padding=(w.size(2) - 1) // 2, groups=D)
    u = F.batch_norm(u, mean.double(), var.double(), gamma.double(), beta.double(), False, 0.0, 1e-5)
    return F.silu(u).transpose(1, 2)


def _conv_native(s3b_lib, x, w, gamma, beta, mean, var, fmt):
    from s3prl_b200 import lib

    B, T, D2 = x.shape
    out = torch.full((B, T, D2 // 2), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_conformer_conv_f32(_ptr(x), B, T, D2 // 2, w.size(2), _ptr(w), _ptr(gamma), _ptr(beta),
                                             _ptr(mean), _ptr(var), fmt, _ptr(out), _stream()))
    torch.cuda.synchronize()
    return out


def _bn_params(D, g):
    return (torch.randn(D, device="cuda", generator=g) * 0.1 + 1, torch.randn(D, device="cuda", generator=g) * 0.1,
            torch.randn(D, device="cuda", generator=g) * 0.1, torch.rand(D, device="cuda", generator=g) + 0.5)


DEPTHWISE_D = 256
DEPTHWISE_KS = [3, 31]
DEPTHWISE_TS = [1, 2, 15, 16, 31, 32, 129, 499]


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("k", DEPTHWISE_KS)
@pytest.mark.parametrize("T", DEPTHWISE_TS)
def test_depthwise_block(s3b_lib, T, k, fmt):
    g = torch.Generator(device="cuda").manual_seed(T * 100 + k)
    B, D = 2, DEPTHWISE_D
    x = torch.randn(B, T, 2 * D, device="cuda", generator=g)
    w = torch.randn(D, 1, k, device="cuda", generator=g) / k**0.5
    bn = _bn_params(D, g)
    out = _conv_native(s3b_lib, x, w, *bn, fmt)
    _check_block(out, _conv_ref(x, w, *bn), f"depthwise T={T} k={k} fmt={fmt}")


@pytest.mark.parametrize("fmt", [0, 1])
def test_depthwise_reads_no_other_utterance(s3b_lib, fmt):
    """Utterances 100x apart in magnitude, each checked against its own scale: a read across the utterance boundary
    (a halo row of the neighbour instead of the zero padding) would show as an error of the neighbour's size."""
    g = torch.Generator(device="cuda").manual_seed(7)
    B, T, D, k = 3, 77, 1024, 31
    x = torch.randn(B, T, 2 * D, device="cuda", generator=g)
    x[:, :, :D] *= torch.tensor([1.0, 100.0, 0.01], device="cuda").view(B, 1, 1)
    w = torch.randn(D, 1, k, device="cuda", generator=g) / k**0.5
    bn = _bn_params(D, g)
    bn = (bn[0], torch.zeros_like(bn[1]), torch.zeros_like(bn[2]), bn[3])  # no bias: the output scales with the input
    out = _conv_native(s3b_lib, x, w, *bn, fmt)
    ref = _conv_ref(x, w, *bn)
    for b in range(B):
        _check_block(out[b], ref[b], f"depthwise utterance {b} fmt={fmt}")


def test_depthwise_refusals(s3b_lib):
    x = torch.zeros(1, 4, 128, device="cuda")
    w = torch.zeros(64, 1, 4, device="cuda")
    v = torch.ones(64, device="cuda")
    out = torch.zeros(1, 4, 64, device="cuda")
    assert s3b_lib.s3b_conformer_conv_f32(_ptr(x), 1, 4, 64, 4, _ptr(w), _ptr(v), _ptr(v), _ptr(v), _ptr(v), 0, _ptr(out),
                                          _stream()) != 0
    assert b"odd" in s3b_lib.s3b_last_error()
    assert s3b_lib.s3b_conformer_conv_f32(_ptr(x), 1, 4, 96, 3, _ptr(w), _ptr(v), _ptr(v), _ptr(v), _ptr(v), 0, _ptr(out),
                                          _stream()) != 0


def _rope_ref(y, T, inv_freq):
    M, D = y.shape
    t = torch.arange(M, device=y.device) % T
    ang = (t.float()[:, None] * inv_freq[None, :]).double()  # the reference's fp32 angle
    cos, sin = torch.cat((ang.cos(), ang.cos()), -1), torch.cat((ang.sin(), ang.sin()), -1)
    yh = y.view(M, D // 64, 64)
    rot = torch.cat((-yh[..., 32:], yh[..., :32]), -1)
    return (yh * cos[:, None, :] + rot * sin[:, None, :]).view(M, D)


ROPE_CASES = [(3, 1, 1024), (2, 999, 1024), (1, 4096, 1024), (2, 130, 768)]  # (B, T, D)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("B,T,D", ROPE_CASES)
def test_layernorm_rope_block(s3b_lib, B, T, D, fmt):
    from s3prl_b200 import lib

    g = torch.Generator(device="cuda").manual_seed(T + D)
    M = B * T
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 0.5
    gamma = torch.randn(D, device="cuda", generator=g) * 0.1 + 1
    beta = torch.randn(D, device="cuda", generator=g) * 0.1
    inv_freq = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    y, yr = torch.empty_like(x), torch.empty_like(x)
    f = (C.c_float * 32)(*inv_freq.tolist())
    lib.check(s3b_lib.s3b_layernorm_rope_f32(_ptr(x), M, T, D, _ptr(gamma), _ptr(beta), f, fmt, _ptr(y), _ptr(yr),
                                             _stream()))
    torch.cuda.synchronize()
    ref = F.layer_norm(x.double(), (D,), gamma.double(), beta.double(), 1e-5)
    _check_block(y, ref, f"layernorm B={B} T={T} D={D} fmt={fmt}")
    _check_block(yr, _rope_ref(ref, T, inv_freq.cuda()), f"layernorm+rope B={B} T={T} D={D} fmt={fmt}")
    # NULL inv_freq: the library's own 1 / 10000^(2j / 64), rounded from double (torch's fp32 power can differ from it by
    # an ulp, which is why the model passes the checkpoint's or torch's buffer)
    yr2 = torch.empty_like(x)
    lib.check(s3b_lib.s3b_layernorm_rope_f32(_ptr(x), M, T, D, _ptr(gamma), _ptr(beta), None, fmt, _ptr(y), _ptr(yr2),
                                             _stream()))
    torch.cuda.synchronize()
    f64 = (1.0 / (10000.0 ** (torch.arange(0, 64, 2, dtype=torch.float64) / 64))).float()
    _check_block(yr2, _rope_ref(ref, T, f64.cuda()), f"layernorm+rope default inv_freq B={B} T={T} D={D} fmt={fmt}")


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("M,N,K,out_fmt", [(1000, 1024, 1024, -1), (300, 4096, 1024, 1), (257, 1024, 4096, 0)])
def test_linear_silu(s3b_lib, scheme, M, N, K, out_fmt):
    from s3prl_b200 import lib

    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K**0.5
    b = torch.randn(N, device="cuda", generator=g)
    out = torch.full((M, N), float("nan"), device="cuda")
    opts = lib.S3BLinearOpts(scheme=scheme, out_fmt=out_fmt)
    lib.check(s3b_lib.s3b_linear_ex(_ptr(a), _ptr(w), _ptr(b), None, M, N, K, 2, C.byref(opts), _ptr(out), _stream()))
    torch.cuda.synchronize()
    assert opts.scheme_used == scheme
    ref = F.silu(a.double() @ w.double().t() + b.double())
    _check_block(out, ref, f"linear+silu scheme={scheme} M={M} N={N} K={K} out_fmt={out_fmt}")
    assert s3b_lib.s3b_linear_ex(_ptr(a), _ptr(w), _ptr(b), None, M, N, K, 3, C.byref(opts), _ptr(out), _stream()) != 0


def _wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


def _arch(variant):
    from s3prl_b200.upstream.configs import ARCHS

    a = ARCHS["wav2vec2_conformer_rope"]
    if variant == "post_ln_2l":  # post-LN encoder, GroupNorm extractor, no waveform normalisation
        return replace(a, encoder_layers=2, layer_norm_first=False, extractor_mode="default", conv_bias=False,
                       normalize=False)
    if variant == "k15":
        return replace(a, encoder_layers=4, depthwise_conv_kernel_size=15)
    return a


_EXPERT = {}


def _expert(variant, scheme):
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    key = (variant, scheme)
    if key not in _EXPERT:
        _EXPERT.clear()
        import os

        saved = os.environ.get("S3B_GEMM_SCHEME")
        if scheme is not None:
            os.environ["S3B_GEMM_SCHEME"] = scheme
        try:
            cfg = _arch(variant)
            _EXPERT[key] = UpstreamExpert(name="wav2vec2_conformer_rope", arch=cfg,
                                          state_dict=fabricate_state_dict(cfg, seed=0)).to("cuda")
            _EXPERT[key]._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        finally:
            if scheme is not None:
                if saved is None:
                    os.environ.pop("S3B_GEMM_SCHEME", None)
                else:
                    os.environ["S3B_GEMM_SCHEME"] = saved
    return _EXPERT[key]


@pytest.mark.parametrize(
    "variant,scheme,lens",
    [
        ("large", None, [40000, 33333, 900]),
        ("large", None, [16000, 50, 399]),  # shorter than the receptive field: the wav2vec2 mask index wraps around
        ("large", "bf16x3", [40000, 33333, 900]),
        ("post_ln_2l", None, [40000, 33333, 900]),
        ("k15", None, [40000, 33333, 900]),
        ("k15", "bf16x3", [16000, 50, 399]),
    ],
)
def test_matches_oracle_ragged(s3b_lib, variant, scheme, lens):
    import conformer_oracle

    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = _arch(variant)
    wavs = _wavs(lens, seed=1234)
    with torch.no_grad():
        ref, _pad = conformer_oracle.conformer_forward(wavs, fabricate_state_dict(cfg, seed=0), cfg)
    hs = _expert(variant, scheme)([w.cuda() for w in wavs])["hidden_states"]
    assert len(hs) == len(ref) == cfg.encoder_layers + 1
    worst = 0.0
    for l, (h, r) in enumerate(zip(hs, ref)):
        assert h.shape == r.shape
        h = h.cpu()
        assert torch.isfinite(h).all()
        rel = _rel(h, r)
        mx = (h.double() - r.double()).abs().max().item()
        assert rel < REL_TOL, (variant, scheme, lens, l, rel)
        assert mx < ABS_FRAC * r.abs().max().item(), (variant, scheme, lens, l, mx)
        worst = max(worst, rel)
    print(f"conformer {variant} scheme={scheme or 'default'} lens={lens}: worst per-layer relative error {worst:.3e}")


@pytest.mark.parametrize("fixture", ["conformer_rope", "conformer_rope_c3"])
def test_matches_reference_golden(s3b_lib, fixture):
    """The hub entry's model (fabricated checkpoint, default scheme) against the executed reference
    (tools/make_conformer_golden.py), with the bars of tests/test_upstream_gpu.py's golden test."""
    from s3prl_b200.upstream.expert import UpstreamExpert

    fx = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    _EXPERT.clear()
    expert = UpstreamExpert(name=fx["arch"], seed=0).to("cuda")
    cs, ts = fx["channel_stride"], fx.get("time_stride", 1)
    worst = 0.0
    for case in fx["cases"]:
        res = expert([w.cuda() for w in _wavs(case["lens"], case["wav_seed"])])
        hs = res["hidden_states"]
        assert len(hs) == case["num_hidden"]
        assert tuple(hs[0].shape) == tuple(case["shape"])
        assert res["last_hidden_state"] is hs[-1]
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu()
            ref = case["sub"][l]
            assert torch.isfinite(sub).all()
            rel = _rel(sub, ref)
            assert rel < REL_TOL, (fixture, l, rel)
            assert (sub.double() - ref.double()).abs().max().item() < ABS_FRAC * ref.abs().max().item(), (fixture, l)
            nrm = h.double().norm().item()
            assert abs(nrm - case["norms"][l].item()) < REL_TOL * case["norms"][l].item()
            worst = max(worst, rel)
    print(f"{fixture}: worst per-layer relative error vs reference golden = {worst:.3e}")


def test_lanes_and_shards_are_bit_identical(s3b_lib):
    ex = _expert("k15", None)
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


def test_layer_results_are_refused(s3b_lib):
    from s3prl_b200 import lib
    from s3prl_b200.upstream.expert import UpstreamExpert

    with pytest.raises(TypeError, match="Conformer"):
        UpstreamExpert(name="wav2vec2_conformer_rope", state_dict={}, feature_selection="fairseq_layers")
    ex = _expert("post_ln_2l", None)
    native = ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))
    wavs = [w.cuda() for w in _wavs([16000, 9000], seed=5)]
    T = ex.num_frames(16000)
    out = torch.empty(3, 2, T, 1024, device="cuda")
    ffn = torch.empty(2, 2, T, 1024, device="cuda")
    ptrs = (C.c_void_p * 2)(*[w.data_ptr() for w in wavs])
    lens = (C.c_int64 * 2)(16000, 9000)
    for field in ("ffn_out", "last_residual"):
        opts = lib.S3BForwardOpts(**{field: ffn.data_ptr()})
        r = native.lib.s3b_forward_ex(native.handle, ptrs, lens, 2, 16000, _ptr(out), _stream(), C.byref(opts))
        assert r != 0 and b"Conformer" in native.lib.s3b_last_error(), field
    opts = lib.S3BForwardOpts()
    lib.check(native.lib.s3b_forward_ex(native.handle, ptrs, lens, 2, 16000, _ptr(out), _stream(), C.byref(opts)))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
