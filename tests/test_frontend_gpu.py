"""Block-level GPU tests of the feature extractor's front end (frontend.cu) through s3b_frontend_f32, which launches it
with the model's own code (model.cu: launch_frontend, shared with the forward): waveform packing with the optional
per-utterance normalisation, conv 0 (Conv1d(1, 512, 10, stride 5)) with GroupNorm(512, 512) over all L0 frames of the
padded batch or per-frame LayerNorm(512), GELU, and the operand planes of both formats decoded back to fp32.

Every case is compared with fp64 torch on the same fp32 inputs (pack, F.layer_norm, F.conv1d, F.group_norm or
F.layer_norm, F.gelu), within a per-element bound derived from the inputs and stated next to the test, and prints
measured/bound.

The GroupNorm statistics are formed from the second-order moments of the conv windows (frontend.cu:
conv0_moments_kernel), var = w^T R w / L0 - mean^2. That form cancels by a channel's conditioning
(sum_j |w_j| |x|)^2 / var(z), which is large where a filter rejects most of the signal: a high-pass filter on
band-limited or DC-offset audio. White noise, the kind of input of the end-to-end tests, never produces it. The bound
here is linear in the conditioning, the accuracy of an fp32 two-pass GroupNorm, so the inputs below include such
channels."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from test_gemm_layouts_gpu import _call, _epilogue, _ln, _ln_bound, _ptr, _stream

pytestmark = pytest.mark.gpu

EPS = 1e-5
U = 2.0**-24  # fp32 unit roundoff
C1 = 12  # conv 0 in fp32: a 10-term fmaf chain loses <= 10 U S_t; the z * scale + shift fold 2 U |mu| more
DELTA_R = 16 * U  # relative rstd accuracy of an fp32 two-pass GroupNorm (~log2(L0) U of its summed variance)


def _lib():
    from s3prl_b200 import lib

    return lib


def _frontend(wavs, max_len, w, bias, gamma, beta, layer_norm, fmt, normalize=False):
    """s3b_frontend_f32 -> (out [B][L0][512], packed waveform [B][max_len])."""
    B = len(wavs)
    L0 = (max_len - 10) // 5 + 1
    ptrs = (C.c_void_p * B)(*[t.data_ptr() for t in wavs])
    lens = (C.c_int64 * B)(*[t.numel() for t in wavs])
    out = torch.full((B, L0, 512), float("nan"), device="cuda")
    wav_out = torch.full((B, max_len), float("nan"), device="cuda")
    _call(_lib().load().s3b_frontend_f32, ptrs, lens, B, max_len, int(normalize), _ptr(w), _ptr(bias), _ptr(gamma),
          _ptr(beta), layer_norm, fmt, _ptr(wav_out), _ptr(out), _stream())
    return out, wav_out


def _rep(y, fmt):
    """Representation error of the operand planes of fmt for a value y: bf16 hi/lo keeps 16 bits; f16q8 keeps fp16's 11
    plus 4 bits of the e4m3 residual, with the e4m3 subnormal floor 2^-20."""
    return 2.0**-16 * y.abs() if fmt == 0 else 2.0**-15 * y.abs() + 2.0**-20


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def _noise(n, rms, g):
    return torch.randn(n, generator=g, dtype=torch.float64) * rms


def _band_limited(n, frac, g):
    """Unit-rms noise keeping only the bottom `frac` of the band."""
    x = torch.randn(n, generator=g, dtype=torch.float64)
    s = torch.fft.rfft(x)
    s[max(1, int(frac * s.numel())):] = 0
    y = torch.fft.irfft(s, n)
    return y / y.pow(2).mean().sqrt().clamp_min(1e-30)


def _signal(kind, n, g):
    if kind == "white1":
        x = _noise(n, 1.0, g)
    elif kind == "white1e-4":  # var(z) << eps: the normalisation is eps-dominated
        x = _noise(n, 1e-4, g)
    elif kind == "white30":
        x = _noise(n, 30.0, g)
    elif kind == "band10":  # bottom 10 % of the band
        x = _band_limited(n, 0.10, g)
    elif kind == "band25":
        x = _band_limited(n, 0.25, g)
    elif kind == "dc":  # 0.9 DC + 0.003 white noise
        x = 0.9 + _noise(n, 0.003, g)
    elif kind == "const":
        x = torch.full((n,), 0.7, dtype=torch.float64)
    elif kind == "zero":
        x = torch.zeros(n, dtype=torch.float64)
    else:
        raise ValueError(kind)
    return x.float().cuda()


def _filters(kind, g):
    """Conv-0 weights [512][10]: kaiming random (fan_in 10), or a bank of four filter families: the alternating-sign
    high-pass (sum |w| ~ 3.6 at c = 0), Hann-windowed band-passes with centres across the band, an all-equal (DC)
    filter, and kaiming random."""
    kaiming = torch.randn(512, 10, generator=g, dtype=torch.float64) * math.sqrt(2.0 / 10)
    if kind == "kaiming":
        return kaiming.float().cuda()
    j = torch.arange(10, dtype=torch.float64)
    c = torch.arange(512, dtype=torch.float64)[:, None]
    k = torch.div(c, 4, rounding_mode="floor")
    high = (-1.0) ** j * 0.36 * (1.0 + k / 128)
    hann = torch.sin(math.pi * (j + 0.5) / 10) ** 2
    band = hann * torch.cos(2 * math.pi * (0.5 * (k % 64) / 63) * (j - 4.5)) * 0.5
    dc = 0.1 * (1.0 + k % 3) * torch.ones_like(j)
    fam = (c % 4).expand(512, 10)
    w = torch.where(fam == 0, high, torch.where(fam == 1, band, torch.where(fam == 2, dc, kaiming)))
    return w.float().cuda()


def _affine(g, bias):
    gamma = (1.0 + 0.2 * torch.randn(512, generator=g)).cuda()
    beta = (0.2 * torch.randn(512, generator=g)).cuda()
    b = (0.5 * torch.randn(512, generator=g)).cuda() if bias else None
    return gamma, beta, b


def _pack_ref(wavs, max_len):
    x = torch.zeros(len(wavs), max_len, dtype=torch.float64, device="cuda")
    for b, t in enumerate(wavs):
        x[b, : t.numel()] = t.double()
    return x


def _conv(x, w):
    """fp64 conv 0 of [B][max_len] -> [B][L0][512]."""
    return F.conv1d(x[:, None, :], w.double()[:, None, :], stride=5).transpose(1, 2)


# ------------------------------------------------------------------------------------------------
# references and bounds
# ------------------------------------------------------------------------------------------------
def _groupnorm_ref(x, w, bias, gamma, beta, fmt):
    """GroupNorm(512, 512) over all L0 frames + GELU in fp64 on the packed waveform x, with the conv bias added (the
    kernel drops it: it cancels in z - mean(z)). Bound per element, linear in the conditioning:
      |v - v_ref| <= |gamma| r [C1 U (S_t + mean_t S_t + |mu|) + |z - mu| DELTA_R] + U (|v| + |beta|)
    with S_t = sum_j |w_j| |x[5t + j]|, mu and r = 1 / sqrt(var + eps) of the kernel's bias-free z: the fp32 conv's
    rounding, the rstd of an fp32 two-pass, the z * scale + shift fold; then GELU (_epilogue) and the planes' _rep."""
    z0 = _conv(x, w)
    S = _conv(x.abs(), w.abs())
    mu = z0.mean(1, keepdim=True)
    r = (z0.var(1, unbiased=False, keepdim=True) + EPS).rsqrt()
    z = z0 if bias is None else z0 + bias.double()
    v = F.group_norm(z.transpose(1, 2), 512, gamma.double(), beta.double(), EPS).transpose(1, 2)
    g, be = gamma.double().abs(), beta.double().abs()
    ev = g * r * (C1 * U * (S + S.mean(1, keepdim=True) + mu.abs()) + (z0 - mu).abs() * DELTA_R) + U * (v.abs() + be)
    out, e = _epilogue(v, ev, gelu=True)
    cond = (S.pow(2).mean(1) * r.squeeze(1).pow(2))  # (rms_t S_t)^2 / (var + eps): the channels' conditioning
    return out, e + _rep(out, fmt), cond


def _layernorm_ref(x, w, bias, gamma, beta, fmt):
    """Per-frame LayerNorm(512) of z (+ bias) + GELU in fp64. The fp32 conv (+ bias) loses
    e_z = C1 U (S_t + |b|); the LayerNorm's bound is _ln_bound(e_z, y, rs) (test_gemm_layouts_gpu), the fmaf with
    gamma, beta another U |v|, then GELU (_epilogue) and the planes' _rep."""
    z = _conv(x, w)
    S = _conv(x.abs(), w.abs())
    if bias is not None:
        z = z + bias.double()
        S = S + bias.double().abs()
    y, rs = _ln(z)
    v = y * gamma.double() + beta.double()
    ev = gamma.double().abs() * _ln_bound(C1 * U * S, y, rs) + U * v.abs()
    out, e = _epilogue(v, ev, gelu=True)
    return out, e + _rep(out, fmt)


def _ratio(what, out, ref, bound):
    assert torch.isfinite(out).all(), what
    return (out.double() - ref).abs() / bound


def _report(what, rat, names=None):
    worst = rat.max().item()
    per = ""
    if names is not None:
        per = " (" + ", ".join(f"{n} {rat[b].max().item():.3f}" for b, n in enumerate(names)) + ")"
    print(f"{what}: measured/bound {worst:.3f}{per}")
    assert worst < 1.0, (what, worst)


# ------------------------------------------------------------------------------------------------
# packing
# ------------------------------------------------------------------------------------------------
PACK_LENS = [1, 9, 10, 11, 14, 15]


@pytest.mark.parametrize("sharded", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
def test_pack(s3b_lib, normalize, sharded):
    """Ragged lengths 1, 9, 10, 11, 14, 15, a large-DC small-signal utterance, a near-constant one (var << eps) and one of
    max_len samples (sharded: max_len above every length). Padding is exactly 0; without normalisation the copy is
    bit-exact. With it, each utterance is F.layer_norm over its own length, within
      |y - y_ref| <= 2 [r (e_m + U |x - m|) + |y_ref| (d_r + U)],   d_r = (e_m^2 + 2 U var) / (2 (var + eps)) + 4 U
    where e_m = U |m| is the fp32 rounding of the mean (summed in fp64), which also biases the fp32 centred variance by
    e_m^2; d_r bounds the relative error of rstd (float variance, + eps, rsqrtf). GroupNorm conv 0 on the packed
    waveform is checked as in test_groupnorm."""
    g = torch.Generator().manual_seed(11 + 2 * normalize + sharded)
    max_len = 4000 + (97 if sharded else 0)
    wavs = [_signal("white1", n, g) * (1 + n) for n in PACK_LENS]
    wavs.append((1000.0 + _noise(3001, 1e-3, g)).float().cuda())  # |m| / sigma = 1e6
    wavs.append((0.5 + _noise(2222, 1e-5, g)).float().cuda())  # var = 1e-10 << eps
    wavs.append(_signal("band25", 4000, g))
    wg = torch.Generator().manual_seed(5)
    w = _filters("bank", wg)
    gamma, beta, _ = _affine(wg, False)
    out, packed = _frontend(wavs, max_len, w, None, gamma, beta, 0, 0, normalize=normalize)
    worst = 0.0
    for b, t in enumerate(wavs):
        n = t.numel()
        assert torch.equal(packed[b, n:], torch.zeros_like(packed[b, n:])), ("padding", b)
        if not normalize:
            assert torch.equal(packed[b, :n], t), ("copy", b)
            continue
        x = t.double()
        m = x.mean()
        var = x.var(unbiased=False)
        r = (var + EPS).rsqrt()
        ref = F.layer_norm(x, (n,), eps=EPS)
        em = U * m.abs()
        dr = (em * em + 2 * U * var) / (2 * (var + EPS)) + 4 * U
        bound = 2 * (r * (em + U * (x - m).abs()) + ref.abs() * (dr + U))
        rat = ((packed[b, :n].double() - ref).abs() / bound).max().item()
        worst = max(worst, rat)
        assert rat < 1.0, ("normalize", b, n, rat)
    if normalize:
        print(f"pack normalize sharded={sharded}: measured/bound {worst:.3f}")
    ref, bound, _ = _groupnorm_ref(packed.double(), w, None, gamma, beta, 0)
    _report(f"pack normalize={normalize} sharded={sharded} conv0+GN", _ratio("pack", out, ref, bound))


# ------------------------------------------------------------------------------------------------
# conv 0 + GroupNorm
# ------------------------------------------------------------------------------------------------
L0S = [1, 2, 3, 4, 5, 255, 256, 257, 513, 31999]
# two ragged batches per case: the first reaches max_len, the second does not (the sharded case); each has an
# utterance shorter than 10 samples or a silent one
SETS = [
    (("white1", 1.0), ("band10", 0.8), ("dc", 0.55), ("const", 7)),
    (("white1e-4", 0.97), ("white30", 0.7), ("const", 0.9), ("zero", 0.4), ("band25", 0.6)),
]


def _batch(L0, sid, g):
    max_len = 5 * (L0 - 1) + 10 + L0 % 5  # L0 % 5 samples beyond the last frame
    names, wavs = [], []
    for kind, f in SETS[sid]:
        n = f if isinstance(f, int) else max(1, int(f * max_len))
        names.append(kind)
        wavs.append(_signal(kind, min(n, max_len), g))
    return max_len, names, wavs


CONV0_BIAS = [False, True]  # conv_bias, in both extractor modes


@pytest.mark.parametrize("L0", L0S)
@pytest.mark.parametrize("bias", CONV0_BIAS)
@pytest.mark.parametrize("filters", ["kaiming", "bank"])
@pytest.mark.parametrize("fmt", [0, 1])
def test_groupnorm(s3b_lib, fmt, filters, bias, L0):
    """extractor_mode "default": GroupNorm(512, 512) over all L0 frames of the padded batch, padding included,
    against F.group_norm of the fp64 conv WITH the conv bias (which the kernel drops); bound: _groupnorm_ref. The
    worst conditioning of the batch is printed beside the ratio."""
    g = torch.Generator().manual_seed(L0 * 8 + 4 * fmt + 2 * (filters == "bank") + bias)
    w = _filters(filters, g)
    gamma, beta, b = _affine(g, bias)
    for sid in range(len(SETS)):
        max_len, names, wavs = _batch(L0, sid, g)
        out, packed = _frontend(wavs, max_len, w, b, gamma, beta, 0, fmt)
        ref, bound, cond = _groupnorm_ref(_pack_ref(wavs, max_len), w, b, gamma, beta, fmt)
        rat = _ratio("gn", out, ref, bound)
        _report(f"GN fmt={fmt} {filters} bias={bias} L0={L0} set {sid} (conditioning <= {cond.max().item():.1e})",
                rat, names)


# ------------------------------------------------------------------------------------------------
# conv 0 + per-frame LayerNorm
# ------------------------------------------------------------------------------------------------
def _near_equal_filters(g):
    """512 filters within 1e-3 of one another: on a DC-offset input a frame's channel spread is ~1e-3 of its mean."""
    base = torch.randn(10, generator=g, dtype=torch.float64).abs() * 0.3 + 0.05
    return (base + 1e-3 * torch.randn(512, 10, generator=g, dtype=torch.float64)).float().cuda()


@pytest.mark.parametrize("L0", [1, 4, 5, 256, 257, 513, 3001])
@pytest.mark.parametrize("bias", CONV0_BIAS)
@pytest.mark.parametrize("filters", ["kaiming", "bank", "near_equal"])
@pytest.mark.parametrize("fmt", [0, 1])
def test_layernorm(s3b_lib, fmt, filters, bias, L0):
    """extractor_mode "layer_norm": LayerNorm over the 512 channels of each frame, conv bias included; padded frames
    (z = bias, or 0 without one: output gelu(beta)) and, with near-equal filters on DC-offset audio, frames whose
    channel spread is ~1e-3 of their mean. Bound: _layernorm_ref."""
    g = torch.Generator().manual_seed(L0 * 16 + 8 * fmt + bias + 3 * len(filters))
    w = _near_equal_filters(g) if filters == "near_equal" else _filters(filters, g)
    gamma, beta, b = _affine(g, bias)
    for sid in range(len(SETS)):
        max_len, names, wavs = _batch(L0, sid, g)
        out, _ = _frontend(wavs, max_len, w, b, gamma, beta, 1, fmt)
        ref, bound = _layernorm_ref(_pack_ref(wavs, max_len), w, b, gamma, beta, fmt)
        _report(f"LN fmt={fmt} {filters} bias={bias} L0={L0} set {sid}", _ratio("ln", out, ref, bound), names)


# ------------------------------------------------------------------------------------------------
# cross-format and bit-exact properties
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer_norm", [0, 1])
def test_formats_agree(s3b_lib, layer_norm):
    """The fmt-0 and fmt-1 decodes of one launch configuration are the same fp32 value through two plane formats: they
    agree within the sum of the formats' representation bounds, which a swapped pair or a misplaced plane breaks."""
    g = torch.Generator().manual_seed(77 + layer_norm)
    w = _filters("bank", g)
    gamma, beta, b = _affine(g, True)
    max_len, names, wavs = _batch(513, 0, g)
    o0, _ = _frontend(wavs, max_len, w, b, gamma, beta, layer_norm, 0)
    o1, _ = _frontend(wavs, max_len, w, b, gamma, beta, layer_norm, 1)
    y = torch.maximum(o0.double().abs(), o1.double().abs())
    rat = (o0.double() - o1.double()).abs() / (_rep(y, 0) + _rep(y, 1))
    _report(f"formats agree layer_norm={layer_norm}", rat, names)


@pytest.mark.parametrize("layer_norm", [0, 1])
def test_batch_independence_and_determinism(s3b_lib, layer_norm):
    """An utterance's output for a given max_len does not depend on the other utterances of the batch (the
    block-level form of the shard-equivalence property), and two identical calls agree, bit for bit."""
    g = torch.Generator().manual_seed(5 + layer_norm)
    w = _filters("bank", g)
    gamma, beta, b = _affine(g, True)
    max_len, _, wavs = _batch(1000, 1, g)
    for normalize in (False, True):
        full, packed = _frontend(wavs, max_len, w, b, gamma, beta, layer_norm, 1, normalize)
        again, packed2 = _frontend(wavs, max_len, w, b, gamma, beta, layer_norm, 1, normalize)
        assert torch.equal(full, again) and torch.equal(packed, packed2)
        for i, t in enumerate(wavs):
            alone, p1 = _frontend([t], max_len, w, b, gamma, beta, layer_norm, 1, normalize)
            assert torch.equal(alone[0], full[i]), (i, normalize)
            assert torch.equal(p1[0], packed[i]), (i, normalize)


def test_validation(s3b_lib):
    """Impossible requests are errors, not fall-backs."""
    lib = _lib()
    L = lib.load()
    g = torch.Generator().manual_seed(1)
    w = _filters("kaiming", g)
    gamma, beta, b = _affine(g, True)
    wav = torch.randn(100, device="cuda")
    out = torch.empty(4 * 100 * 512, device="cuda")

    def call(lens, max_len, layer_norm=0, fmt=0, wv=w, ga=gamma, ptr=None, normalize=0):
        ptrs = (C.c_void_p * len(lens))(*([wav.data_ptr()] * len(lens) if ptr is None else ptr))
        ln = (C.c_int64 * len(lens))(*lens)
        _call(L.s3b_frontend_f32, ptrs, ln, len(lens), max_len, normalize, _ptr(wv), _ptr(b), _ptr(ga), _ptr(beta),
              layer_norm, fmt, None, _ptr(out), _stream())

    call([100, 10], 100)  # valid
    cases = [
        (dict(lens=[5], max_len=9), "max_len"),
        (dict(lens=[50, 101], max_len=100), "lens"),
        (dict(lens=[50, 0], max_len=100), "lens"),
        (dict(lens=[50], max_len=100, fmt=2), "out_fmt"),
        (dict(lens=[50], max_len=100, fmt=-1), "out_fmt"),
        (dict(lens=[50], max_len=100, layer_norm=2), "layer_norm"),
        (dict(lens=[50], max_len=100, normalize=2), "normalize"),
        (dict(lens=[50], max_len=100, wv=None), "null"),
        (dict(lens=[50], max_len=100, ga=None), "null"),
        (dict(lens=[50, 50], max_len=100, ptr=[wav.data_ptr(), None]), "null"),
    ]
    for kw, msg in cases:
        with pytest.raises(lib.S3BError, match=msg):
            call(**kw)


# ------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------
def test_hubert_highpass_band_limited(s3b_lib):
    """hubert_base through the model (fabricated weights, conv 0 replaced by the filter bank of _filters) on band-limited
    and DC-offset audio, against the oracle at the parity tolerance of test_upstream_gpu: whether the front end's error
    on ill-conditioned channels reaches the hidden states."""
    from test_upstream_gpu import _EXPERTS, _compare  # (puts oracle/ on sys.path)

    import upstream_oracle as O
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = ARCHS["hubert_base"]
    sd = fabricate_state_dict(cfg, seed=0)
    g = torch.Generator().manual_seed(3)
    sd["feature_extractor.conv_layers.0.0.weight"] = _filters("bank", g).cpu().view(512, 1, 10)
    wavs = [_signal("band10", 48000, g).cpu(), _signal("dc", 31999, g).cpu(), _signal("band25", 16000, g).cpu()]
    with torch.no_grad():
        ref, _ = O.upstream_forward(wavs, sd, cfg)
    _EXPERTS.clear()
    expert = UpstreamExpert(arch=cfg, state_dict=sd, name="hubert_highpass").to("cuda")
    hs = expert([w.cuda() for w in wavs])["hidden_states"]
    assert len(hs) == len(ref)
    worst = max(_compare(h.cpu(), r, f"hubert high-pass layer {l}") for l, (h, r) in enumerate(zip(hs, ref)))
    print(f"hubert_base high-pass bank, band-limited input: worst per-layer relative error vs oracle = {worst:.3e}")
