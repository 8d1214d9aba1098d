"""GPU tests of modified CPC (``modified_cpc``): one conv + ChannelNorm + ReLU at block level (``s3b_cpc_conv_f32``)
per element in both GEMM operand schemes at every residue of the input length mod the stride (conv 0 against fp64,
conv 1..4 against fp64 and the emulated operand decomposition of tests/test_gemm_layouts_gpu.py), the norm's edges
(common offsets, spreads below sqrt(eps), constant frames, NaN inputs), the neighbouring utterances of a batch never
read, the LSTM recurrence at block level (``s3b_cpc_lstm_f32``) against fp64, the whole model against the
executed-reference goldens (tests/golden/cpc_ref*.pt) and the fp64 CPU oracle (tests/cpc_oracle.py), bit-identical
results across batch order and composition, padded length (frames before an utterance's last), shards, lanes,
``forward_host``, repeated calls and a long-lived model after a poisoned call, and the launch counts.
Bounds: convs per element, derived from the operands (_cn_bound, _plane_err); recurrence 1e-4 relative Frobenius and
2e-4 of the largest output per element; model 2e-4 relative per hidden state. Every check prints measured / bound."""
import ctypes as C
import os
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import cpc_oracle as CO  # noqa: E402
from test_gemm_layouts_gpu import _check, _epilogue, _gemm_refs, _through_planes  # noqa: E402
from test_npc_gpu import _separation  # noqa: E402

pytestmark = pytest.mark.gpu

BLOCK_REL = 1e-4
BLOCK_ELEM = 2e-4
REL_TOL = 2e-4
U = 2.0**-24  # fp32 unit roundoff
NORM_DEPTH = 9  # norm.cu: a channel's value passes 3 adds in its lane's sum, 5 in warp_sum: log2(256) + 1 rounded up
CONV0_DEPTH = 12  # frontend.cu cpc_conv0_kernel: 7 serial adds of a lane's 8 channels, 5 in warp_sum


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _wavs(lens, seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) * scale for n in lens]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------------
# block level
# ------------------------------------------------------------------------------------------------
def _cpc_conv(s3b_lib, x, layer, w, bias, gamma, beta, scheme):
    from s3prl_b200 import lib

    B, L = x.shape[0], x.shape[1]
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    T = (L + 2 * p - 2 * s) // s + 1
    out = torch.full((B, T, 256), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_cpc_conv_f32(_ptr(x), B, L, layer, _ptr(w), _ptr(bias), _ptr(gamma), _ptr(beta), scheme,
                                       _ptr(out), _stream()))
    torch.cuda.synchronize()
    return out


def _cn(v):
    """fp64 ChannelNorm without the affine, per row: y = (v - mean) rstd, rstd = 1 / sqrt(unbiased variance + 1e-5)."""
    mu = v.mean(-1, keepdim=True)
    rs = (v.var(-1, unbiased=True, keepdim=True) + 1e-5).rsqrt()
    return (v - mu) * rs, rs


def _cn_bound(e, v, y, rs, depth):
    """|dy| of y = ChannelNorm(v) for an input error e, the _ln_bound analogue with the unbiased variance over D
    channels. First order: dy = rstd (dv - mean(dv)) + (v - mean) d(rstd) with d(rstd) = -rstd^3 d(var) / 2 and
    d(var) = 2 / (D - 1) sum (v - mean) dv, so |d(var)| <= 2 sqrt(D / (D - 1)) sqrt(var) rms(dv) (Cauchy-Schwarz), and
    as rstd sqrt(var) <= 1: |dy| <= rstd (|dv| + mean|dv| + sqrt(D / (D - 1)) |y| rms(dv)).
    Plus the kernel's fp32 arithmetic:
    - 2^-20 |y| for the subtraction, the variance (squares, a sum of 256, the 1 / 255 scaling), rsqrtf, the scaling by
      rstd and gamma (about 10 roundings of the unit 2^-24, each relative to |y|);
    - the mean's rounding: depth U mean|v| rstd, with depth the adds a value passes through on its way into the sum
      (a first-order bound on any summation order of that depth). With no common offset it is below 2^-20; on frames
      whose channels share an offset of many spreads it is what a correct two-pass fp32 kernel achieves, as the
      variance is then taken around a mean whose error is this small."""
    D = v.shape[-1]
    rms = e.pow(2).mean(-1, keepdim=True).sqrt()
    return (rs * (e + e.mean(-1, keepdim=True) + (D / (D - 1)) ** 0.5 * y.abs() * rms) + 2.0**-20 * y.abs()
            + depth * U * v.abs().mean(-1, keepdim=True) * rs)


def _cn_relu(v, e, gamma, beta, depth):
    """relu(ChannelNorm(v) gamma + beta) in fp64 and its bound for an error e of v: the norm (_cn_bound), gamma, the
    fp32 add of beta; ReLU is 1-Lipschitz."""
    y, rs = _cn(v)
    z = y * gamma.double() + beta.double()
    return torch.relu(z), gamma.double().abs() * _cn_bound(e, v, y, rs, depth) + U * z.abs()


def _cpc_im2col(x, layer):
    """conv 1..4 as the GEMM the kernel runs: row (b, t) of A is x[b, s t + j - p] for j < 2 s, zero outside [0, L),
    tap-major; interior: the rows with every tap inside [0, L)."""
    B, L, _ = x.shape
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    T = (L + 2 * p - 2 * s) // s + 1
    idx = s * torch.arange(T, device=x.device)[:, None] + torch.arange(2 * s, device=x.device)[None, :]  # padded
    a = F.pad(x, (0, 0, p, p))[:, idx, :].reshape(B * T, 2 * s * 256)
    return a, ((idx >= p) & (idx < L + p)).all(1).repeat(B)


def _conv_case(s3b_lib, what, x, layer, w, bias, gamma, beta, scheme, frob=True):
    """conv 1..4 + ChannelNorm + ReLU of x against both references per element: the GEMM's (_gemm_refs on the im2col
    view, which must equal F.conv1d in fp64) through the fp32 bias add (_epilogue) and the norm (_cn_relu). Returns
    the output [B * T][256] and which rows' receptive fields are all zeros (their pre-norm frame is exactly bias)."""
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    out = _cpc_conv(s3b_lib, x, layer, w, bias, gamma, beta, scheme).view(-1, 256)
    a, interior = _cpc_im2col(x, layer)
    wk = w.permute(0, 2, 1).reshape(256, 2 * s * 256)
    exact, emu, e1, e2 = _gemm_refs(a, wk, scheme)
    conv = F.conv1d(x.double().transpose(1, 2), w.double(), stride=s, padding=p).transpose(1, 2).reshape(-1, 256)
    assert ((conv - exact).abs() <= 1e-6 * e1).all()  # the im2col view is the convolution (to fp64 rounding)
    gemm, apart_check = _separation(what, a, wk, e1, e2, interior, scheme)
    ref1, b1 = _cn_relu(*_epilogue(conv, e1, bias), gamma, beta, NORM_DEPTH)
    ref2, b2 = _cn_relu(*_epilogue(emu, e2, bias), gamma, beta, NORM_DEPTH)
    _check(what, out, ref1, b1, ref2, b2, gemm, scheme, frob=frob, apart_check=apart_check)
    return out, (a == 0).all(1)


def _conv0_case(s3b_lib, what, x, w, cbias, gamma, beta, scheme):
    """conv 0 + ChannelNorm + ReLU of the waveforms x [B][L] per element against fp64, read back from the scheme's
    operand planes: the fp32 FMA chain of 10 taps (10 U sum|w x|) and the bias add (U |z|), the norm (_cn_relu, with
    the conv 0 kernel's summation depth) and the planes' representation error (_plane_err). Returns the output
    [B * T][256] and which rows' receptive fields are all zeros (their pre-norm frame is exactly cbias)."""
    s, p = CO.STRIDES[0], CO.PADDINGS[0]
    out = _cpc_conv(s3b_lib, x, 0, w, cbias, gamma, beta, scheme).view(-1, 256)
    xd, wd = x.double().unsqueeze(1), w.double()
    z = F.conv1d(xd, wd, cbias.double(), stride=s, padding=p).transpose(1, 2).reshape(-1, 256)
    mag = F.conv1d(xd.abs(), wd.abs(), stride=s, padding=p).transpose(1, 2).reshape(-1, 256)
    ref, bound = _cn_relu(z, 10 * U * mag + U * z.abs(), gamma, beta, CONV0_DEPTH)
    bound = bound + _plane_err(ref, scheme)
    assert torch.isfinite(out).all(), what
    r = ((out.double() - ref).abs() / bound).max().item()
    print(f"{what}: measured/bound fp64 {r:.3f}")
    assert r < 1.0, (what, r)
    zeros = (F.pad(x, (p, p)).unfold(1, 2 * s, s)[:, : out.shape[0] // x.shape[0]] == 0).all(-1).reshape(-1)
    return out, zeros


def _plane_err(y, fmt):
    """|read back - y| for operand planes of format fmt written from fp32 y (_through_planes), |y| < 448:
    bf16 hi / lo: 2^-9 of 2^-9 |y| left after the hi plane, and the fp32 add of the two: 2^-17 |y| covers both.
    f16q8: fp16 keeps r = y - fp16(y) within 2^-11 |y| (2^-25 below fp16's normals); e4m3 keeps r 2048 within 2^-4 of
    itself, or 2^-10 in its subnormals: 2^-15 |y| + 2^-21, and U |y| for the fp32 add."""
    if fmt == 0:
        return 2.0**-17 * y.abs()
    return (2.0**-15 + U) * y.abs() + 2.0**-21


_T = [1, 2, 127, 128, 129, 1000]
_UTT_SCALES = (1.0, 0.25, 0.5)  # per utterance of a batch of 3: a row read from the wrong utterance shows


def _norm_params(g):
    return (0.1 * torch.randn(256, device="cuda", generator=g), 0.5 + torch.rand(256, device="cuda", generator=g),
            0.2 * torch.randn(256, device="cuda", generator=g))


def _conv_weights(layer, g, scale=1.0):
    s = CO.STRIDES[layer]
    cin = 1 if layer == 0 else 256
    return torch.randn(256, cin, 2 * s, device="cuda", generator=g) * (scale / (cin * 2 * s) ** 0.5)


def _lengths(layer):
    """(T, L): every T of _T at every residue of the input length mod the stride."""
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    return [(T, s * (T - 1) + 2 * s - 2 * p + r) for T in _T for r in range(s)]


def _input(layer, L, g, scale=1.0):
    """Three utterances at different scales: waveforms (randn 0.1; utterance 2 with a DC offset and utterance 1 with a
    stretch of exact zeros, where conv 0's frames are cbias alone) or conv outputs (relu(randn))."""
    sc = torch.tensor(_UTT_SCALES, device="cuda")
    if layer == 0:
        x = torch.randn(3, L, device="cuda", generator=g) * 0.1 * scale * sc[:, None]
        x[2] += 0.3 * scale
        x[1, L // 3 : L // 3 + 40] = 0
        return x
    return torch.relu(torch.randn(3, L, 256, device="cuda", generator=g)) * scale * sc[:, None, None]


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("layer", [0, 1, 2, 3, 4])
def test_cpc_conv_block_matches_fp64(s3b_lib, scheme, layer):
    """Each conv + ChannelNorm + ReLU per element at every T of _T and every residue of the input length mod the
    stride: conv 0 against fp64 (_conv0_case), conv 1..4 against fp64 and the emulated operand decomposition
    (_conv_case)."""
    for T, L in _lengths(layer):
        g = torch.Generator(device="cuda").manual_seed(1000 * layer + 10 * T + L + 7 * scheme)
        x = _input(layer, L, g)
        w = _conv_weights(layer, g)
        bias, gamma, beta = _norm_params(g)
        what = f"cpc conv {layer} s{scheme} T={T} L={L}"
        if layer == 0:
            out, _ = _conv0_case(s3b_lib, what, x, w, bias, gamma, beta, scheme)
        else:
            out, _ = _conv_case(s3b_lib, what, x, layer, w, bias, gamma, beta, scheme)
        assert out.shape[0] == 3 * T, (out.shape, T)


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("layer", [0, 1, 2, 3, 4])
def test_cpc_channelnorm_edges(s3b_lib, scheme, layer):
    """The ChannelNorm of both CPC norm paths (conv 0's kernel, and the norm kernel after conv 1..4) per element on
    frames that tell a correct fp32 norm from a subtly wrong one, built from weights, bias and input:
    - offset: every channel of a frame shares an offset of about 100x the frame's spread (conv 1..4: a constant bias
      of 70 over outputs of spread ~0.7; conv 0: taps summing to 1 on each channel, over a waveform with a DC offset
      of 100x its noise). A one-pass E[x^2] - mean^2 variance loses the spread there.
    - tiny: the spread (~1e-3) is below sqrt(eps) = 3.2e-3, which tells eps inside the rsqrt from eps outside it.
    - constant: frames whose receptive field is all zeros are the constant bias alone; the output is exactly
      relu(beta) (conv 0: through its operand planes).
    - NaN: one NaN input sample (conv 0) or row (conv 1..4) makes every output frame whose receptive field holds it NaN
      in all channels, kept through the ReLU; every other frame is bit-identical to the run without it."""
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    T = 300
    L = s * (T - 1) + 2 * s - 2 * p + s - 1
    g = torch.Generator(device="cuda").manual_seed(50 + layer + 10 * scheme)
    _, gamma, beta = _norm_params(g)
    relu_beta = torch.relu(beta) if layer else _through_planes(torch.relu(beta), scheme)
    for kind in ("offset", "tiny"):
        what = f"cpc conv {layer} s{scheme} {kind}"
        if layer == 0:
            w = _conv_weights(0, g)
            if kind == "offset":
                w = w - w.mean(-1, keepdim=True) + 0.1  # each channel's taps sum to 1: the DC is a common offset
                x = 10.0 + 0.1 * torch.randn(3, L, device="cuda", generator=g)
            else:
                x = 1e-3 * torch.randn(3, L, device="cuda", generator=g)
            x[:, 100:140] = 0
            cbias = torch.full((256,), 1.5 if kind == "offset" else 0.25, device="cuda")
            out, zeros = _conv0_case(s3b_lib, what, x, w, cbias, gamma, beta, scheme)
        else:
            x = _input(layer, L, g) / torch.tensor(_UTT_SCALES, device="cuda")[:, None, None]
            x[:, 100:140] = 0
            w = _conv_weights(layer, g, 1.0 if kind == "offset" else 1.4e-3)
            bias = torch.full((256,), 70.0 if kind == "offset" else 0.25, device="cuda")
            out, zeros = _conv_case(s3b_lib, what, x, layer, w, bias, gamma, beta, scheme, frob=False)
        assert zeros.sum() >= 3, what
        assert torch.equal(out[zeros], relu_beta.expand(int(zeros.sum()), 256)), (what, "constant frames")
        print(f"{what}: {int(zeros.sum())} constant frames exactly relu(beta)")

    x = _input(layer, L, g)
    w = _conv_weights(layer, g)
    bias, _, _ = _norm_params(g)
    clean = _cpc_conv(s3b_lib, x, layer, w, bias, gamma, beta, scheme)
    n0 = L // 2
    x[1, n0] = float("nan")
    out = _cpc_conv(s3b_lib, x, layer, w, bias, gamma, beta, scheme)
    t = torch.arange(T, device="cuda")
    hit = (s * t - p <= n0) & (n0 < s * t - p + 2 * s)
    assert hit.sum() == 2, hit.sum()
    assert torch.isnan(out[1, hit]).all(), "frames reading the NaN"
    keep = torch.ones(3, T, dtype=torch.bool, device="cuda")
    keep[1, hit] = False
    assert torch.equal(out[keep], clean[keep]), "frames not reading the NaN"
    print(f"cpc conv {layer} s{scheme}: NaN at input {n0} -> frames {t[hit].tolist()} NaN, the rest bit-identical")


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("layer", [0, 1, 2, 3, 4])
def test_neighbours_are_never_read(s3b_lib, scheme, layer):
    """Utterance 1 of a batch of 3 whose utterances 0 and 2 are all NaN is bit-identical to utterance 1 run alone, at
    lengths where the first frame reads the front padding and the last one the padded rows (or samples) at the end."""
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    for T, r in ((1, 0), (129, s - 1), (200, 0)):
        L = s * (T - 1) + 2 * s - 2 * p + r
        g = torch.Generator(device="cuda").manual_seed(T + layer + r + 10 * scheme)
        x = _input(layer, L, g)
        w = _conv_weights(layer, g)
        bias, gamma, beta = _norm_params(g)
        alone = _cpc_conv(s3b_lib, x[1:2].contiguous(), layer, w, bias, gamma, beta, scheme)
        x[0], x[2] = float("nan"), float("nan")
        out = _cpc_conv(s3b_lib, x, layer, w, bias, gamma, beta, scheme)
        assert torch.isfinite(alone).all()
        assert torch.equal(out[1], alone[0]), (T, L)
    print(f"cpc conv {layer} s{scheme}: utterance 1 between NaN neighbours bit-identical")


def test_cpc_conv_refusals(s3b_lib):
    x = torch.zeros(1, 400, 256, device="cuda")
    w = torch.zeros(256, 256, 8, device="cuda")
    v = torch.zeros(256, device="cuda")
    out = torch.zeros(1, 400, 256, device="cuda")
    for B, L, layer, want in ((1, 400, 5, b"layer"), (1, 400, -1, b"layer"), (0, 400, 1, b"batch"),
                              (1, 3, 1, b"too short"), (1, 3, 0, b"too short")):
        r = s3b_lib.s3b_cpc_conv_f32(_ptr(x), B, L, layer, _ptr(w), _ptr(v), _ptr(v), _ptr(v), -1, _ptr(out), None)
        assert r != 0 and want in s3b_lib.s3b_last_error(), (B, L, layer)


def _lstm_ref(x, sd, k):
    return CO.lstm_layer(x, *(sd[f"gAR.baseNet.{n}_l{k}"].double() for n in ("weight_ih", "weight_hh", "bias_ih",
                                                                             "bias_hh")))


def _cpc_lstm(s3b_lib, xg, whh, out_fmt=-1):
    from s3prl_b200 import lib

    B, T = xg.shape[0], xg.shape[1]
    out = torch.full((B, T, 256), float("nan"), device="cuda")
    planes = torch.full((B, T, 256), float("nan"), device="cuda") if out_fmt >= 0 else None
    lib.check(s3b_lib.s3b_cpc_lstm_f32(_ptr(xg), _ptr(whh), B, T, out_fmt, _ptr(out), _ptr(planes), _stream()))
    torch.cuda.synchronize()
    return out, planes


@pytest.mark.parametrize("B,T", [(1, 1), (4, 37), (5, 2000), (70, 300)])
def test_cpc_lstm_matches_fp64(s3b_lib, B, T):
    """One and two layers from xg = W_ih x + b_ih + b_hh, against the fp64 cell in relative Frobenius norm and per
    element (the largest error over the largest output); B = 5 and 70 leave the last cluster's group of four partly
    filled. Layer 0 writes bf16 hi / lo planes, layer 1 f16q8 ones: the kernel stores them from the same registers as
    the fp32 output, so they are bit for bit the planes of that output."""
    from s3prl_b200.upstream.cpc import fabricate_cpc_state_dict

    n_active = C.c_int32()
    s3b_lib.s3b_cpc_lstm_max_active_clusters(C.byref(n_active))
    sd = fabricate_cpc_state_dict(4, 2)
    g = torch.Generator().manual_seed(B * 7 + T)
    x = torch.relu(torch.randn(B, T, 256, generator=g, dtype=torch.float64))
    worst = worst_elem = 0.0
    inp = x
    for k in range(2):
        xg = (inp.float() @ sd[f"gAR.baseNet.weight_ih_l{k}"].T + sd[f"gAR.baseNet.bias_ih_l{k}"]
              + sd[f"gAR.baseNet.bias_hh_l{k}"])
        out, planes = _cpc_lstm(s3b_lib, xg.cuda().contiguous(), sd[f"gAR.baseNet.weight_hh_l{k}"].cuda(), k)
        ref = _lstm_ref(inp, sd, k)
        e = _rel(out.cpu(), ref)
        elem = ((out.cpu().double() - ref).abs().max() / ref.abs().max()).item()
        worst, worst_elem = max(worst, e), max(worst_elem, elem)
        assert e < BLOCK_REL and elem < BLOCK_ELEM, (k, e, elem)
        assert torch.equal(planes, _through_planes(out, k)), k  # out_fmt k
        inp = out.cpu().double()
    print(f"cpc lstm B={B} T={T}: worst relative error over 2 layers {worst:.3e} (measured/bound "
          f"{worst / BLOCK_REL:.3f}), elementwise {worst_elem:.3e} ({worst_elem / BLOCK_ELEM:.3f}); planes bit for bit; "
          f"{n_active.value} clusters of 8 CTAs co-resident, {(B + 3) // 4} needed")


def test_cpc_lstm_bit_identical_in_any_slot(s3b_lib):
    from s3prl_b200.upstream.cpc import fabricate_cpc_state_dict

    sd = fabricate_cpc_state_dict(4)
    whh = sd["gAR.baseNet.weight_hh_l0"].cuda()
    g = torch.Generator().manual_seed(5)
    xg = torch.randn(11, 50, 1024, generator=g).cuda()
    full, _ = _cpc_lstm(s3b_lib, xg, whh)
    for i in (0, 3, 6, 10):
        alone, _ = _cpc_lstm(s3b_lib, xg[i : i + 1].contiguous(), whh)
        assert torch.equal(alone[0], full[i]), i
    perm = torch.randperm(11, generator=g)
    shuffled, _ = _cpc_lstm(s3b_lib, xg[perm].contiguous(), whh)
    assert torch.equal(shuffled, full[perm])


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _expert(scheme, **kw):
    from s3prl_b200.upstream.cpc import CpcExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        ex = CpcExpert(**kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


def _ckpt(tmp_path, over, seed):
    from s3prl_b200.upstream.cpc import cpc_config, fabricate_cpc_state_dict

    config = cpc_config(**over)
    sd = fabricate_cpc_state_dict(seed, config["nLevelsGRU"])
    path = tmp_path / "cpc.pt"
    torch.save({"config": config, "weights": sd}, path)
    return str(path), sd


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("fixture", ["cpc_ref", "cpc_ref_c2", "cpc_ref_variant"])
def test_matches_reference_golden(s3b_lib, tmp_path, fixture, scheme):
    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    path, _ = _ckpt(tmp_path, g["config"], g["weight_seed"])
    ex = _expert(scheme, ckpt=path)
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        wavs = [w.cuda() for w in _wavs(case["lens"], case["wav_seed"], case["wav_scale"])]
        res = ex(wavs)
        assert tuple(res["_hidden_states_info"]) == tuple(case["names"])
        hs = res["hidden_states"]
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            err = _rel(h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu(), case["sub"][l])
            print(f"cpc {fixture} lens={case['lens']} scheme={scheme or 'default'} state {l}: abs max "
                  f"{h.abs().max().item():.3f}, relative error {err:.3e} (measured/bound {err / REL_TOL:.3f})")
            assert err < REL_TOL


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("levels", [1, 2])
def test_matches_oracle_ragged(s3b_lib, tmp_path, scheme, levels):
    path, sd = _ckpt(tmp_path, {"nLevelsGRU": levels}, 2)
    ex = _expert(scheme, ckpt=path)
    lens = [48000, 159, 31234, 16001, 47999, 90, 9000]
    wavs = _wavs(lens, seed=11)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    ref = CO.forward(wavs, sd, levels)
    assert len(hs) == len(ref) == 2
    for l, (h, r) in enumerate(zip(hs, ref)):
        err = _rel(h.cpu(), r)
        print(f"cpc ragged levels={levels} scheme={scheme or 'default'} state {l}: abs max {r.abs().max().item():.3f}"
              f", relative error {err:.3e} (measured/bound {err / REL_TOL:.3f})")
        assert err < REL_TOL


def test_bit_identical_batch_shards_lanes_host_repeats(s3b_lib):
    from s3prl_b200.upstream.cpc import num_frames

    ex = _expert(None)
    lens = [int(v) for v in torch.randint(100, 160000, (32,), generator=torch.Generator().manual_seed(3))]
    lens[5] = 160000
    wavs = [w.cuda() for w in _wavs(lens, seed=21)]
    full = torch.stack(ex(wavs)["hidden_states"]).clone()
    # batch order at the same max_len
    perm = torch.randperm(32, generator=torch.Generator().manual_seed(4)).tolist()
    assert torch.equal(torch.stack(ex([wavs[i] for i in perm])["hidden_states"]), full[:, perm])
    # an utterance alone, padded to the batch's max_len, vs inside the batch of 32; shards of the batch
    ex.global_max_len = max(lens)
    for i in (0, 5, 17):
        alone = torch.stack(ex([wavs[i]])["hidden_states"])
        assert torch.equal(alone[:, 0], full[:, i]), i
    halves = [torch.stack(ex(wavs[s])["hidden_states"]) for s in (slice(0, 16), slice(16, 32))]
    assert torch.equal(torch.cat(halves, dim=1), full)
    ex.global_max_len = None
    # a different max_len: frames before an utterance's last one are unchanged
    for i in (0, 17, 30):
        alone = torch.stack(ex([wavs[i]])["hidden_states"])
        t = num_frames(lens[i]) - 1
        assert torch.equal(alone[:, 0, :t], full[:, i, :t]), i
    for lanes in (1, 2):
        ex.lanes = lanes
        assert torch.equal(torch.stack(ex(wavs)["hidden_states"]), full), lanes
    ex.lanes = 0
    host = ex.forward_host([w.cpu() for w in wavs[:8]])
    dev8 = torch.stack(ex(wavs[:8])["hidden_states"]).cpu()
    assert torch.equal(host, dev8)
    native = ex._native
    counts = []
    for i in range(10):
        c0 = native.lib.s3b_launch_count(native.handle)
        res = torch.stack(ex(wavs)["hidden_states"])
        counts.append(native.lib.s3b_launch_count(native.handle) - c0)
        assert torch.equal(res, full), f"call {i + 1} changed the result"
    assert len(set(counts)) == 1, counts
    # a long-lived model after a poisoned call larger than every probe (NaN, inf, 1e30 samples) and calls of other
    # shapes gives what a fresh one gives: no pad row of a reused workspace leaks into a result
    g = torch.Generator().manual_seed(8)
    poison = []
    for n in (170000, 165000, 150000, 170000):
        p = torch.randn(n, generator=g) * 1e30
        p[::7] = float("nan")
        p[3::11] = float("inf")
        poison.append(p.cuda())
    ex.lanes = 2
    bad = torch.stack(ex(poison)["hidden_states"])
    assert not torch.isfinite(bad[1]).all()
    ex.lanes = 0
    fresh = _expert(None)
    for probe in (wavs[3:9], wavs[:1], wavs):
        assert torch.equal(torch.stack(ex(probe)["hidden_states"]), torch.stack(fresh(probe)["hidden_states"]))
    print(f"cpc bit-identity: batch order and composition, max_len (frames before the last), shards, lanes 1/2, "
          f"forward_host, 10 repeats ({counts[0]} launches each), long-lived model after a poisoned call vs fresh")


@pytest.mark.parametrize("levels", [1, 3])
def test_launch_counts_profile_and_refusals(s3b_lib, tmp_path, levels):
    from s3prl_b200 import lib

    path, _ = _ckpt(tmp_path, {"nLevelsGRU": levels}, 1)
    ex = _expert(None, ckpt=path)
    ex.lanes = 1
    native = ex._native
    wavs = [w.cuda() for w in _wavs([16000, 8000], seed=1)]
    T = ex.num_frames(16000)
    out = torch.empty(2, 2, T, 256, device="cuda")
    ptrs = (C.c_void_p * 2)(*[w.data_ptr() for w in wavs])
    for field in ("ffn_out", "last_residual"):
        opts = lib.S3BForwardOpts(**{field: out.data_ptr()})
        r = native.lib.s3b_forward_ex(native.handle, ptrs, (C.c_int64 * 2)(16000, 8000), 2, 16000,
                                      C.c_void_p(out.data_ptr()), _stream(), C.byref(opts))
        assert r != 0 and field.encode() in native.lib.s3b_last_error()
    with pytest.raises(ValueError, match="159"):
        ex([torch.zeros(158, device="cuda"), torch.zeros(20, device="cuda")])
    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    c0 = native.lib.s3b_launch_count(native.handle)
    ex(wavs)
    total = native.lib.s3b_launch_count(native.handle) - c0
    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
    lib.check(native.lib.s3b_profile_read_ex(native.handle, 6, ms, fl, n, 1))
    lib.check(native.lib.s3b_profile_enable(native.handle, 0))
    # 4 conv GEMMs + 1 input GEMM per layer; conv 0; 4 norms; the wave pack; 1 recurrence per layer
    assert list(n) == [4 + levels, 0, 1, 4, 1, levels], list(n)
    assert total == 10 + 2 * levels, total
    # FLOPs with the real channels: conv i has 2 s_i taps of 256 channels
    L = [16000]
    for s, p in zip(CO.STRIDES, CO.PADDINGS):
        L.append((L[-1] + 2 * p - 2 * s) // s + 1)
    want = sum(2.0 * 2 * L[i + 1] * 256 * 256 * 2 * CO.STRIDES[i] for i in range(1, 5)) + levels * 2.0 * 2 * T * 1024 * 256
    assert abs(fl[0] / want - 1) < 1e-12, (fl[0], want)
    print(f"cpc profile ms (levels={levels}): gemm {ms[0]:.3f} conv0 {ms[2]:.3f} norm {ms[3]:.3f} "
          f"recurrence {ms[5]:.3f}")


def test_finalize_names_a_missing_tensor(s3b_lib):
    from s3prl_b200 import lib
    from s3prl_b200.upstream.cpc import CpcExpert

    ex = CpcExpert()
    ex._state_dict_host["gEncoder.batchNorm2.weight"] = torch.ones(256)  # not [1, 256, 1]
    with pytest.raises(lib.S3BError, match=r"gEncoder\.batchNorm2\.weight"):
        ex.to("cuda")([torch.randn(16000, device="cuda")])
