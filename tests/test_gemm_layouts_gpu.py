"""Block-level GPU tests of the GEMM's layouts in both operand schemes, through the entry points that build their launches
with the model's own code: the flat linears (tile widths 128 / 256, operand-plane output, post_extract_proj's row mask,
fc2's pre-residual output, the distiller's and DeCoAR's column slices), the QKV epilogue, conv 1..6 and the positional
conv in both formulations with its combine kernel.

Every case is checked against two references, both in fp64 on the GPU:
1. the exact operation on the fp32 inputs, within a per-element bound derived from the inputs (_gemm_refs: the
   scheme's representation error c * 2^-16 * (|A| |W|^T), the f16q8 floors and saturation terms, accumulation), and
   within the 1e-4 relative Frobenius bar of the block tests where the operands are N(0, 1)-scaled;
2. the scheme's own operand decomposition emulated in torch (bf16x3: hi hi + hi lo + lo hi; f16q8: A16 W16 +
   2^-15 (A_l8 W_h8 + A_h8 W_l8), satfinite as a clamp to +-448), within an accumulation-only bound much tighter than
   reference 1 (50x or more for f16q8, 4x or more for bf16x3: see below), so that a dropped k-step or a misread operand
   plane shows.
Outputs written as operand planes are compared bit for bit with the planes of the fp32 output of the same launch
configuration (_through_planes).

The accumulation bound lets every accumulating MMA of an output element lose up to C_ACC / 2 ulps of a running sum of
size sqrt(sum_k (a_k w_k)^2) (the partial sums' scale): C_ACC * 2^-24 * n * sqrt(sum_k (a_k w_k)^2) over the n MMAs
that read non-zero operands. The error grows with n, not sqrt(n): on an H100 the kernel's distance to the emulation
grew like sqrt(K) relative to a random-walk model (bf16x3, K 512 -> 4096: 2.4x -> 6.1x of 8 * 2^-24 * sqrt(n Q)),
the mark of an accumulator that truncates. The e4m3 correction MMAs are taken to keep about 13 bits of the correction
sum (2^-13 in place of 2^-24: Hopper's FP8 MMAs are reported to keep around 14 bits; not measured separately here).
Against fp64 the f16q8 bounds are 50x or more wider than the accumulation bound; for bf16x3, whose operands keep 16
bits, they are 4x - 20x wider (the accumulation error is the larger part of its total), which still leaves a dropped
16-wide k-step of any of its three products several times over the accumulation bound. Each case prints both ratios."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

C_ACC = 4.0
GELU_SLOPE = 1.13  # max |GELU'(x)|
GELU_ERR = 3e-7  # relative error of the kernels' erfc-polynomial GELU (common.cuh: gelu_erf)
Q_SCALE = torch.tensor(1.4426950408889634, dtype=torch.float32).item() * 0.125  # kQScale: 1/8 * log2(e), in fp32


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lib():
    from s3prl_b200 import lib

    return lib


def _call(fn, *args):
    _lib().check(fn(*args))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# operand formats and references
# ------------------------------------------------------------------------------------------------
def _e4m3(x):
    """cvt.rn.satfinite to e4m3 (fp32 in), as fp64."""
    return x.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).double()


def _planes(x, scheme, weight):
    """The operand planes of fp32 x, as fp64 values scaled back: bf16x3 (hi, lo); f16q8 (x16, x_h8, x_l8) with
    activations x_h8 = e4m3(fp16(x)), x_l8 = e4m3((x - x16) 2^11) 2^-11 and weights x_h8 = e4m3(x 2^4) 2^-4,
    x_l8 = e4m3((x - x16) 2^15) 2^-15 (frontend.cu: split_q8_kernel)."""
    if scheme == 0:
        hi = x.bfloat16().float()
        return hi.double(), (x - hi).bfloat16().double()
    x16 = x.half().float()
    r = x - x16  # exact in fp32
    if weight:
        return x16.double(), _e4m3(x * 16.0) / 16.0, _e4m3(r * 2.0**15) * 2.0**-15
    return x16.double(), _e4m3(x16), _e4m3(r * 2.0**11) * 2.0**-11


def _through_planes(y, fmt):
    """What a consumer reads back from operand planes of format fmt written from fp32 y (split_pack2 /
    split_q8_pack2, then load_planes2), bit for bit."""
    if fmt == 0:
        hi = y.bfloat16().float()
        return hi + (y - hi).bfloat16().float()
    h = y.half().float()
    return h + ((y - h) * 2048.0).clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float() * 2.0**-11


def _gemm_refs(a, w, scheme):
    """a [M][K], w [N][K] fp32 -> (exact, emulated, e1, e2) in fp64 for a @ w^T.
    e1 (vs exact): bf16x3 2 * 2^-16 P (hi + lo keeps 16 bits of each operand, lo lo dropped); f16q8 8 * 2^-16 P
    (e4m3 keeps 4 bits of the 2^-11 residuals, on both correction products) + the e4m3 subnormal floors (A_l8, A_h8:
    2^-21 |w|; W_l8, W_h8: 2^-25 |a|; summed generously as 2^-20 sum|w| + 2^-24 sum|a|) + saturation (A_h8 clamps
    |a16| > 448, W_h8 |w| > 28: 2^-11 (|A| relu(|W| - 28)^T + relu(|A| - 448) |W|^T)); plus e2.
    e2 (vs emulated): accumulation only (module docstring)."""
    K = a.shape[1]
    ad, wd = a.double(), w.double()
    exact = ad @ wd.t()
    P = ad.abs() @ wd.abs().t()
    Q = (ad * ad) @ (wd * wd).t()
    ks = K // 16  # 16-wide k-steps (bf16 / fp16 MMAs); the e4m3 corrections: 2 MMAs per 32 = K / 16 as well
    if scheme == 0:
        ah, al = _planes(a, 0, False)
        wh, wl = _planes(w, 0, True)
        emu = ah @ wh.t() + ah @ wl.t() + al @ wh.t()
        e2 = C_ACC * 2.0**-24 * 3 * ks * Q.sqrt()
        e1 = 2 * 2.0**-16 * P + e2
    else:
        a16, ah8, al8 = _planes(a, 1, False)
        w16, wh8, wl8 = _planes(w, 1, True)
        emu = a16 @ w16.t() + al8 @ wh8.t() + ah8 @ wl8.t()
        qc = (al8 * al8) @ (wh8 * wh8).t() + (ah8 * ah8) @ (wl8 * wl8).t()
        e2 = C_ACC * ks * (2.0**-24 * Q.sqrt() + 2.0**-13 * qc.sqrt())
        floor = 2.0**-20 * wd.abs().sum(1)[None, :] + 2.0**-24 * ad.abs().sum(1)[:, None]
        sat = 2.0**-11 * (ad.abs() @ (wd.abs() - 28).clamp_min(0).t() + (ad.abs() - 448).clamp_min(0) @ wd.abs().t())
        e1 = 8 * 2.0**-16 * P + floor + sat + e2
    return exact, emu, e1, e2


def _epilogue(pre, e, bias=None, gelu=False, res=None):
    """fp64 epilogue v = pre (+ bias); GELU?; (+ residual) and the propagated bound of a pre-activation error e plus
    the kernel's fp32 roundings and GELU approximation."""
    v = pre if bias is None else pre + bias.double()
    out = F.gelu(v) if gelu else v
    eo = e + 2.0**-24 * v.abs()
    if gelu:
        eo = GELU_SLOPE * eo + GELU_ERR * v.abs()
    if res is not None:
        out = out + res.double()
    return out, eo + 2.0**-24 * out.abs()


def _check(what, out, ref1, b1, ref2, b2, gemm, scheme, frob=True, apart_check=True):
    """out within b1 of ref1 and b2 of ref2 everywhere; the GEMM's bounds gemm = (e1, e2) apart by the factor the
    module docstring states (median), unless the caller checks the property that factor stands for itself
    (apart_check=False: tests/test_port_shapes_gpu.py at K >= 5120); 1e-4 relative Frobenius vs ref1 where the
    operands are N(0, 1)-scaled (frob)."""
    assert torch.isfinite(out).all(), what
    o = out.double()
    r1 = ((o - ref1).abs() / b1).max().item()
    r2 = ((o - ref2).abs() / b2).max().item()
    apart = (gemm[0] / gemm[1]).median().item()
    rel = ((o - ref1).norm() / ref1.norm()).item()
    print(f"{what}: measured/bound fp64 {r1:.3f}, emulated {r2:.3f} (bounds {apart:.0f}x apart); rel {rel:.2e}")
    assert r1 < 1.0, (what, "fp64", r1)
    assert r2 < 1.0, (what, "emulated", r2)
    if apart_check:
        assert apart >= (50.0 if scheme == 1 else 4.0), (what, apart)
    if frob:
        assert rel < 1e-4, (what, rel)


def _linear(a, w, bias=None, res=None, gelu=False, M=None, N=None, K=None, **opts):
    lib = _lib()
    M = a.shape[0] if M is None else M
    N = w.shape[0] if N is None else N
    K = w.shape[1] if K is None else K
    o = lib.S3BLinearOpts(**opts)
    out = torch.full((M, N), float("nan"), device="cuda")
    _call(lib.load().s3b_linear_ex, _ptr(a), _ptr(w), _ptr(bias), _ptr(res), M, N, K, int(gelu), C.byref(o), _ptr(out),
          _stream())
    return out, o


# ------------------------------------------------------------------------------------------------
# flat linears
# ------------------------------------------------------------------------------------------------
LINEAR_SHAPES = [(512, 768), (512, 1024), (768, 2304), (1024, 3072), (768, 768), (1024, 1024), (768, 3072), (3072, 768),
                 (1024, 4096), (4096, 1024)]  # (K, N): post_extract_proj, QKV, out_proj, fc1 / fc2 of base and large


def _operands(M, N, K, mag, g):
    if mag == "large":  # |a| up to 3000 (A_h8 saturates above 448), |w| up to 40 (W_h8 above 28)
        a = (torch.randn(M, K, device="cuda", generator=g) * 700).clamp(-3000, 3000)
        w = (torch.randn(N, K, device="cuda", generator=g) * 10).clamp(-40, 40)
    else:
        s = 1.0 if mag == "unit" else 1e-3  # 1e-3: the f16q8 residuals fall into e4m3's subnormals
        a = torch.randn(M, K, device="cuda", generator=g) * s
        w = torch.randn(N, K, device="cuda", generator=g) * (s / K**0.5)
    return a, w


@pytest.mark.parametrize("M", [1, 127, 128, 129, 1000, 4099])
@pytest.mark.parametrize("K,N", LINEAR_SHAPES)
@pytest.mark.parametrize("scheme", [0, 1])
def test_linear_layouts(s3b_lib, scheme, K, N, M):
    """out_proj / fc2 style (bias + residual, fp32) at both tile widths, which must agree bit for bit; fc1 style (bias +
    GELU) as fp32 and as operand planes of the scheme's format."""
    g = torch.Generator(device="cuda").manual_seed(M * 131 + K * 7 + N + scheme)
    a, w = _operands(M, N, K, "unit", g)
    b = torch.randn(N, device="cuda", generator=g) * 0.5
    r = torch.randn(M, N, device="cuda", generator=g)
    exact, emu, e1, e2 = _gemm_refs(a, w, scheme)
    outs = {}
    for tile in (256, 128) if N % 256 == 0 else (128,):
        outs[tile], o = _linear(a, w, b, r, scheme=scheme, tile_n=tile)
        assert (o.scheme_used, o.tile_n_used) == (scheme, tile)
    ref1, b1 = _epilogue(exact, e1, b, res=r)
    ref2, b2 = _epilogue(emu, e2, b, res=r)
    _check(f"linear s{scheme} M={M} K={K} N={N} residual", outs[128], ref1, b1, ref2, b2, (e1, e2), scheme)
    if 256 in outs:
        assert torch.equal(outs[256], outs[128]), "tile widths 128 and 256 differ"

    h32, o = _linear(a, w, b, gelu=True, scheme=scheme)
    ref1, b1 = _epilogue(exact, e1, b, gelu=True)
    ref2, b2 = _epilogue(emu, e2, b, gelu=True)
    _check(f"linear s{scheme} M={M} K={K} N={N} gelu (tile {o.tile_n_used})", h32, ref1, b1, ref2, b2, (e1, e2), scheme)
    hp, _ = _linear(a, w, b, gelu=True, scheme=scheme, out_fmt=scheme)
    assert torch.equal(hp, _through_planes(h32, scheme)), "GELU operand planes != planes of the fp32 output"


@pytest.mark.parametrize("mag", ["small", "large"])
@pytest.mark.parametrize("K,N", LINEAR_SHAPES)
@pytest.mark.parametrize("scheme", [0, 1])
def test_linear_magnitudes(s3b_lib, scheme, K, N, mag):
    """x1e-3 (f16q8 residuals in e4m3 subnormals: the floors of _gemm_refs) and |a| ~ 3000, |w| ~ 40 (A_h8 and W_h8
    saturate: the emulation clamps, the fp64 bound has the saturation term). Planes only where fp16 holds the output."""
    M = 1000
    g = torch.Generator(device="cuda").manual_seed(K * 3 + N + scheme + len(mag))
    a, w = _operands(M, N, K, mag, g)
    exact, emu, e1, e2 = _gemm_refs(a, w, scheme)
    out, o = _linear(a, w, scheme=scheme)
    assert o.scheme_used == scheme
    ref1, b1 = _epilogue(exact, e1)
    ref2, b2 = _epilogue(emu, e2)
    _check(f"linear s{scheme} K={K} N={N} {mag}", out, ref1, b1, ref2, b2, (e1, e2), scheme, frob=False)
    if mag == "small":
        for fmt in (0, 1):
            planes, _ = _linear(a, w, scheme=scheme, out_fmt=fmt)
            assert torch.equal(planes, _through_planes(out, fmt)), fmt


@pytest.mark.parametrize("scheme", [0, 1])
def test_linear_row_mask(s3b_lib, scheme):
    """post_extract_proj: padded frames (row_mask != 0) come out exactly zero, as fp32 and as bf16 hi/lo planes; the
    other rows are bit-identical to an unmasked launch."""
    M, K, N = 1000, 512, 768
    g = torch.Generator(device="cuda").manual_seed(99 + scheme)
    a, w = _operands(M, N, K, "unit", g)
    b = torch.randn(N, device="cuda", generator=g)
    mask = (torch.rand(M, device="cuda", generator=g) < 0.3).to(torch.uint8)
    mask[-129:] = 1  # a whole padded tail tile
    keep = mask == 0
    free, _ = _linear(a, w, b, scheme=scheme)
    exact, emu, e1, e2 = _gemm_refs(a, w, scheme)
    ref1, b1 = _epilogue(exact, e1, b)
    ref2, b2 = _epilogue(emu, e2, b)
    _check(f"proj s{scheme}", free, ref1, b1, ref2, b2, (e1, e2), scheme)
    for fmt in (-1, 0):
        out, _ = _linear(a, w, b, scheme=scheme, out_fmt=fmt, row_mask=mask.data_ptr())
        assert torch.equal(out[~keep], torch.zeros_like(out[~keep])), fmt
        want = free if fmt < 0 else _through_planes(free, 0)
        assert torch.equal(out[keep], want[keep]), fmt


@pytest.mark.parametrize("scheme", [0, 1])
def test_linear_out_pre(s3b_lib, scheme):
    """fc2's out_pre: the value before the residual add, so that out == out_pre + residual bit for bit, and out_pre is
    the launch without residual."""
    M, K, N = 1000, 3072, 768
    g = torch.Generator(device="cuda").manual_seed(7 + scheme)
    a, w = _operands(M, N, K, "unit", g)
    b = torch.randn(N, device="cuda", generator=g)
    r = torch.randn(M, N, device="cuda", generator=g) * 3
    pre = torch.full((M, N), float("nan"), device="cuda")
    out, _ = _linear(a, w, b, r, scheme=scheme, out_pre=pre.data_ptr())
    alone, _ = _linear(a, w, b, scheme=scheme)
    assert torch.equal(pre, alone)
    assert torch.equal(out, pre + r)
    exact, emu, e1, e2 = _gemm_refs(a, w, scheme)
    ref1, b1 = _epilogue(exact, e1, b, res=r)
    ref2, b2 = _epilogue(emu, e2, b, res=r)
    _check(f"fc2 s{scheme}", out, ref1, b1, ref2, b2, (e1, e2), scheme)


SPLIT_SLICES = [  # (N, K, lda, a_off): A is the K-column slice at a_off of rows lda apart
    (768, 768, 3 * 768, 0),  # the distiller's SplitLinear, tasks 0, 1, 2
    (768, 768, 3 * 768, 768),
    (768, 768, 3 * 768, 2 * 768),
    (4096, 1024, 2048, 0),  # DeCoAR's LSTM input GEMM above layer 0: the forward direction's half of [2048]
    (4096, 1024, 2048, 1024),  # the backward direction's half
]


@pytest.mark.parametrize("N,K,lda,a_off", SPLIT_SLICES, ids=["0", "1", "2", "decoar_fwd", "decoar_bwd"])
@pytest.mark.parametrize("scheme", [0, 1])
def test_linear_split_slice(s3b_lib, scheme, N, K, lda, a_off):
    """A strided column slice of A (the distiller's SplitLinear, DeCoAR's bidirectional layer input): bit-identical to
    the dense slice. The columns outside the slice are NaN, so reading any of them shows."""
    M = 499
    g = torch.Generator(device="cuda").manual_seed(11 + a_off + N + 5 * scheme)
    h = torch.full((M, lda), float("nan"), device="cuda")
    h[:, a_off : a_off + K] = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K**0.5
    b = torch.randn(N, device="cuda", generator=g)
    out, _ = _linear(h, w, b, M=M, N=N, K=K, scheme=scheme, lda=lda, a_off=a_off)
    a = h[:, a_off : a_off + K].contiguous()
    dense, _ = _linear(a, w, b, scheme=scheme)
    assert torch.equal(out, dense)
    exact, emu, e1, e2 = _gemm_refs(a, w, scheme)
    ref1, b1 = _epilogue(exact, e1, b)
    ref2, b2 = _epilogue(emu, e2, b)
    _check(f"split linear s{scheme} N={N} K={K} lda={lda} a_off={a_off}", out, ref1, b1, ref2, b2, (e1, e2), scheme)


# ------------------------------------------------------------------------------------------------
# QKV epilogue
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T,H", [(2, 499, 12), (3, 1, 12), (2, 129, 16), (1, 1000, 16), (2, 37, 12)])
@pytest.mark.parametrize("scheme", [0, 1])
def test_qkv(s3b_lib, scheme, B, T, H):
    """The QKV epilogue: q = q_scale (x W_q^T + b_q) and k as [B][H][T][64], v^T as [B][H][64][Tp] (Tp = T rounded up to
    8; the epilogue never writes columns T..), all bf16 hi/lo. Bit for bit the planes of the fp32 linear on the same
    operands (scaled in fp32 for q), which is itself checked against both references; q, k, v^T also directly against
    fp64."""
    D, Tp, M = H * 64, (T + 7) & ~7, B * T
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T * 10 + H + scheme)
    x = torch.randn(B, T, D, device="cuda", generator=g)
    w = torch.randn(3 * D, D, device="cuda", generator=g) / D**0.5
    b = torch.randn(3 * D, device="cuda", generator=g) * 0.5
    q = torch.full((B, H, T, 64), float("nan"), device="cuda")
    k = torch.full_like(q, float("nan"))
    vt = torch.full((B, H, 64, Tp), float("nan"), device="cuda")
    _call(_lib().load().s3b_qkv_f32, _ptr(x), _ptr(w), _ptr(b), B, T, H, scheme, _ptr(q), _ptr(k), _ptr(vt), _stream())

    y, o = _linear(x.view(M, D), w, b, scheme=scheme)
    assert o.scheme_used == scheme
    exact, emu, e1, e2 = _gemm_refs(x.view(M, D), w, scheme)
    ref1, b1 = _epilogue(exact, e1, b)
    ref2, b2 = _epilogue(emu, e2, b)
    _check(f"qkv s{scheme} B={B} T={T} H={H} linear", y, ref1, b1, ref2, b2, (e1, e2), scheme)

    def heads(t):  # [M][D] -> [B][H][T][64]
        return t.reshape(B, T, H, 64).transpose(1, 2)

    assert torch.equal(q, heads(_through_planes(y[:, :D] * Q_SCALE, 0))), "q"
    assert torch.equal(k, heads(_through_planes(y[:, D : 2 * D], 0))), "k"
    assert torch.equal(vt[..., :T], heads(_through_planes(y[:, 2 * D :], 0)).transpose(2, 3)), "v^T"
    plane = 2.0**-16 * ref1.abs()  # the bf16 hi/lo planes keep 16 bits
    for name, got, sl, s in (("q", q, slice(0, D), Q_SCALE), ("k", k, slice(D, 2 * D), 1.0)):
        err = (got.double() - heads(ref1[:, sl]) * s).abs() / (heads(b1[:, sl] + plane[:, sl]) * s)
        assert err.max().item() < 1.0, name
    err = (vt[..., :T].double() - heads(ref1[:, 2 * D :]).transpose(2, 3)).abs()
    assert (err / heads(b1[:, 2 * D :] + plane[:, 2 * D :]).transpose(2, 3)).max().item() < 1.0, "v^T"


# ------------------------------------------------------------------------------------------------
# conv 1..6
# ------------------------------------------------------------------------------------------------
def _conv(x, w, bias, Lin, kw, gelu, scheme, out_fmt):
    B = x.shape[0]
    Lout = (Lin - kw) // 2 + 1
    out = torch.full((B, Lout, 512), float("nan"), device="cuda")
    _call(_lib().load().s3b_conv_gemm_f32, _ptr(x), _ptr(w), _ptr(bias), B, Lin, kw, int(gelu), scheme, out_fmt,
          _ptr(out), _stream())
    return out


@pytest.mark.parametrize("odd", [False, True])
@pytest.mark.parametrize("Lout", [1, 2, 127, 128, 129, 799])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("kw", [3, 2])
@pytest.mark.parametrize("scheme", [0, 1])
def test_conv(s3b_lib, scheme, kw, bias, Lout, odd):
    """Conv1d(512, 512, kw, stride 2) on channels-last [3][Lin][512] (different content per utterance) in the model's
    epilogue modes: GELU + operand planes (conv 1..5), GELU + fp32 (conv 6), fp32 without GELU (layer_norm mode).
    Reference 1: F.conv1d in fp64; reference 2 and the bounds: the same product as the [B*Lout][kw*512] im2col GEMM."""
    B = 3
    Lin = 2 * (Lout - 1) + kw
    if (Lin % 2 == 1) != odd:
        Lin += 1  # same Lout: the extra sample is never read by an output frame
    g = torch.Generator(device="cuda").manual_seed(kw * 1000 + Lout * 2 + odd + 17 * scheme + 3 * bias)
    x = torch.randn(B, Lin, 512, device="cuda", generator=g) * (1.0 + torch.arange(B, device="cuda")[:, None, None])
    w = torch.randn(512, 512, kw, device="cuda", generator=g) / (512 * kw) ** 0.5
    bv = torch.randn(512, device="cuda", generator=g) if bias else None
    idx = 2 * torch.arange(Lout, device="cuda")[:, None] + torch.arange(kw, device="cuda")[None, :]
    a = x[:, idx, :].reshape(B * Lout, kw * 512)  # row (b, t) = [x[b, 2t + j, :] for j < kw]
    wk = w.permute(0, 2, 1).reshape(512, kw * 512)
    exact, emu, e1, e2 = _gemm_refs(a, wk, scheme)
    conv = F.conv1d(x.double().transpose(1, 2), w.double(), stride=2).transpose(1, 2).reshape(B * Lout, 512)
    assert ((conv - exact).abs() <= 1e-9 * (1 + exact.abs())).all()  # the im2col view is the convolution
    for gelu, fmt in ((True, -1), (False, -1)):
        out = _conv(x, w, bv, Lin, kw, gelu, scheme, fmt)
        ref1, b1 = _epilogue(conv, e1, bv, gelu=gelu)
        ref2, b2 = _epilogue(emu, e2, bv, gelu=gelu)
        _check(f"conv s{scheme} kw={kw} Lin={Lin} bias={bias} gelu={gelu}", out.view(B * Lout, 512), ref1, b1, ref2, b2,
               (e1, e2), scheme)
        if gelu:
            planes = _conv(x, w, bv, Lin, kw, True, scheme, scheme)
            assert torch.equal(planes, _through_planes(out, scheme)), "GELU operand planes"


# ------------------------------------------------------------------------------------------------
# positional conv
# ------------------------------------------------------------------------------------------------
def _ln(v):
    mu = v.mean(-1, keepdim=True)
    rs = (v.var(-1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
    return (v - mu) * rs, rs


def _ln_bound(e, y, rs):
    """|dy| of y = LayerNorm(v) for an input error e: (|dv| + mean|dv| + |y| rms(dv)) / sigma, plus 2^-20 (1 + |y|) for
    the kernel's fp32 mean, variance and rsqrt."""
    rms = e.pow(2).mean(-1, keepdim=True).sqrt()
    return rs * (e + e.mean(-1, keepdim=True) + y.abs() * rms) + 2.0**-20 * (1 + y.abs())


def _posconv_pipeline(conv, e, x, bias, mode, gamma, beta):
    v = conv + bias.double()
    if mode == 0:  # x + GELU(conv + bias)
        out = x.double() + F.gelu(v)
        eo = GELU_SLOPE * (e + 2.0**-24 * v.abs()) + GELU_ERR * v.abs() + 2.0**-24 * out.abs()
    else:  # GELU(LayerNorm_noaffine(conv + bias)) (+ x)
        y, rs = _ln(v)
        out = F.gelu(y)
        eo = GELU_SLOPE * _ln_bound(e + 2.0**-24 * v.abs(), y, rs) + GELU_ERR * y.abs()
        if mode == 2:
            out = out + x.double()
            eo = eo + 2.0**-24 * out.abs()
    if gamma is not None:
        y, rs = _ln(out)
        out = y * gamma.double() + beta.double()
        eo = gamma.double().abs() * _ln_bound(eo, y, rs) + 2.0**-24 * out.abs()
    return out, eo


def _posconv(x, w, bias, G, k, taps, mode, gamma=None, beta=None, out_fmt=-1):
    B, T, D = x.shape
    out = torch.full_like(x, float("nan"))
    _call(_lib().load().s3b_posconv_f32, _ptr(x), _ptr(w), _ptr(bias), B, T, D, G, k, taps, mode, _ptr(gamma),
          _ptr(beta), out_fmt, _ptr(out), _stream())
    return out


def _posconv_refs(x, w, G, k, taps):
    """Grouped conv (padding k // 2, first T outputs: SamePad for even k) -> exact, emulated bf16x3, e1, e2 per element.
    Accumulating MMAs per output frame: 3 per 16-channel k-step (48 channels: 3 k-steps of the 64-wide box) and tap
    that reads a frame inside [0, T) (the zero-filled ones add exact zeros), + 4 fp32 adds of the combine."""
    B, T, D = x.shape
    cpg = D // G

    def conv(xx, ww):
        return F.conv1d(xx.transpose(1, 2), ww, padding=k // 2, groups=G)[..., :T].transpose(1, 2)

    xd, wd = x.double(), w.double()
    exact = conv(xd, wd)
    P = conv(xd.abs(), wd.abs())
    Q = conv(xd * xd, wd * wd)
    xh, xl = _planes(x, 0, False)
    wh, wl = _planes(w, 0, True)
    emu = conv(xh, wh) + conv(xh, wl) + conv(xl, wh)
    t = torch.arange(T, device=x.device)
    taps_in = (torch.clamp(t - k // 2 + k, max=T) - torch.clamp(t - k // 2, min=0)).double()
    n = 3 * ((cpg + 15) // 16) * taps_in[None, :, None] + 4
    e2 = C_ACC * 2.0**-24 * n * Q.sqrt()
    return exact, emu, 2 * 2.0**-16 * P + e2, e2


POS_CONFIGS = [  # (D, groups, k, taps per k-block, mode)
    (768, 16, 128, 4, 0),  # base: 48 channels per group, k_steps = 3
    (768, 16, 128, 1, 0),
    (1024, 16, 128, 4, 0),  # large: 64 channels per group
    (1024, 16, 128, 1, 0),
    (512, 16, 128, 1, 0),  # LightHuBERT student small: 32 channels per group, one tap per k-block (32-column tiles)
    (768, 16, 19, 4, 1),  # data2vec blocks: 19 taps -> 20 (one zero tap)
    (768, 16, 19, 4, 2),
    (1024, 16, 19, 4, 1),  # data2vec large: five k-blocks of 64-channel groups
    (1024, 16, 19, 4, 2),
    (1024, 16, 24, 4, 1),  # even k: SamePad drops the last frame
    (1024, 16, 24, 4, 2),
    (768, 16, 3, 4, 1),
    (768, 16, 3, 4, 2),
]


def _pos_inputs(B, T, D, G, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, T, D, device="cuda", generator=g)
    w = torch.randn(D, D // G, k, device="cuda", generator=g) / (D // G * k) ** 0.5
    bias = torch.randn(D, device="cuda", generator=g) * 0.2
    return x, w, bias, g


@pytest.mark.parametrize("T", [1, 2, 3, 64, 65, 128, 129, 499])
@pytest.mark.parametrize("D,G,k,taps,mode", POS_CONFIGS)
def test_posconv(s3b_lib, D, G, k, taps, mode, T):
    """Positional conv as the model's add_pos_conv runs it, B = 2: x + GELU(conv + b) (mode 0), the data2vec blocks (mode 1, and
    mode 2 with the residual), against F.conv1d(padding k // 2, groups) truncated to T and the mode's arithmetic in
    fp64; the bounds propagate through GELU and the LayerNorms (_ln_bound)."""
    x, w, bias, _ = _pos_inputs(2, T, D, G, k, D + k * 3 + taps + 10 * mode + T * 100)
    out = _posconv(x, w, bias, G, k, taps, mode)
    exact, emu, e1, e2 = _posconv_refs(x, w, G, k, taps)
    ref1, b1 = _posconv_pipeline(exact, e1, x, bias, mode, None, None)
    ref2, b2 = _posconv_pipeline(emu, e2, x, bias, mode, None, None)
    _check(f"posconv D={D} k={k} taps={taps} mode={mode} T={T}", out, ref1, b1, ref2, b2, (e1, e2), 0)


@pytest.mark.parametrize("T", [3, 129, 499])
@pytest.mark.parametrize("D,G,k,taps,mode", [c for c in POS_CONFIGS if c[4] != 1])
def test_posconv_post_ln(s3b_lib, D, G, k, taps, mode, T):
    """Post-LN models: the encoder LayerNorm (gamma, beta) on the result, as fp32 and as operand planes of both formats
    (bit for bit the planes of the fp32 output)."""
    x, w, bias, g = _pos_inputs(2, T, D, G, k, D + k + taps + mode + T)
    gamma = 1.0 + 0.3 * torch.randn(D, device="cuda", generator=g)
    beta = 0.3 * torch.randn(D, device="cuda", generator=g)
    out = _posconv(x, w, bias, G, k, taps, mode, gamma, beta)
    exact, emu, e1, e2 = _posconv_refs(x, w, G, k, taps)
    ref1, b1 = _posconv_pipeline(exact, e1, x, bias, mode, gamma, beta)
    ref2, b2 = _posconv_pipeline(emu, e2, x, bias, mode, gamma, beta)
    _check(f"posconv+LN D={D} k={k} taps={taps} mode={mode} T={T}", out, ref1, b1, ref2, b2, (e1, e2), 0)
    for fmt in (0, 1):
        planes = _posconv(x, w, bias, G, k, taps, mode, gamma, beta, out_fmt=fmt)
        assert torch.equal(planes, _through_planes(out, fmt)), fmt


# ------------------------------------------------------------------------------------------------
# validation
# ------------------------------------------------------------------------------------------------
def test_entry_points_validate(s3b_lib):
    """Impossible requests are errors, not silent fall-backs."""
    lib = _lib()
    L = lib.load()
    a = torch.randn(256, 4096, device="cuda")
    w = torch.randn(4096, 4096, device="cuda")
    with pytest.raises(lib.S3BError, match="f16q8"):  # K % 128 != 0
        _linear(a, w, M=256, N=256, K=192, scheme=1)
    with pytest.raises(lib.S3BError, match="tile_n"):  # 256 does not divide 384
        _linear(a, w, M=256, N=384, K=256, tile_n=256)
    for bad in ({"scheme": 2}, {"out_fmt": 2}, {"tile_n": 64}, {"lda": 100, "a_off": 0}):
        with pytest.raises(lib.S3BError):
            _linear(a, w, M=256, N=256, K=256, **bad)
    out = torch.empty(4096 * 16, device="cuda")
    with pytest.raises(lib.S3BError, match="f16q8"):  # QKV of 3 heads: K = 192
        _call(L.s3b_qkv_f32, _ptr(a), _ptr(w), _ptr(w), 1, 10, 3, 1, _ptr(out), _ptr(out), _ptr(out), _stream())
    x = torch.randn(1, 16, 1024, device="cuda")
    with pytest.raises(lib.S3BError, match="channels per group"):  # 8 groups of 128 channels
        _posconv(x, torch.randn(1024, 128, 4, device="cuda"), torch.zeros(1024, device="cuda"), 8, 4, 4, 0)
    w1 = torch.randn(1024, 64, 4, device="cuda")
    with pytest.raises(lib.S3BError, match="LayerNorm"):  # one tap: planes only through the LayerNorm, as in the model
        _posconv(x, w1, torch.zeros(1024, device="cuda"), 16, 4, 1, 0, out_fmt=0)
    with pytest.raises(lib.S3BError):  # the data2vec blocks have no one-tap formulation
        _posconv(x, torch.randn(1024, 64, 3, device="cuda"), torch.zeros(1024, device="cuda"), 16, 3, 1, 1)
    with pytest.raises(lib.S3BError):  # kw 4
        _call(L.s3b_conv_gemm_f32, _ptr(a), _ptr(w), None, 1, 100, 4, 0, 0, -1, _ptr(out), _stream())
    with pytest.raises(lib.S3BError):  # conv output format 2
        _call(L.s3b_conv_gemm_f32, _ptr(a), _ptr(w), None, 1, 100, 3, 0, 0, 2, _ptr(out), _stream())
    with pytest.raises(lib.S3BError, match="struct_size"):
        o = lib.S3BLinearOpts()
        o.struct_size = 8
        _call(L.s3b_linear_ex, _ptr(a), _ptr(w), None, None, 16, 256, 256, 0, C.byref(o), _ptr(out), _stream())
