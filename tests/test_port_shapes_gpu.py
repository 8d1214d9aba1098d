"""Block-level GPU tests of the existing GEMM, LayerNorm and Featurizer kernels at the shapes the ports run them at,
where otherwise only whole-model parity (2e-4 per layer) would look:
- the flat linears of XLS-R 1B / 2B (QKV, out_proj, fc1, fc2, post_extract_proj: K up to 7680, N = 1920 on 128-wide
  tiles only), DeCoAR 2.0's post_extract_proj and APC's gate GEMMs (K = 128: the 80 fbank bins zero-padded, two
  k-blocks per tile, so the ring's stage / phase wraps mid-tile), the encoder linears and post_extract_proj of the
  384-, 512- and 640-wide LightHuBERT subnets, DeCoAR's proj, modified CPC's LSTM input GEMM (K = 256) and the
  Conformer's [q | k] / pointwise_conv1 (N = 2048), in both operand schemes, with the two references of
  tests/test_gemm_layouts_gpu.py; tests/test_port_coverage_cpu.py checks that every served shape has a row here or in
  another block table;
- pick_bn's choice between 128- and 256-wide tiles by the fill of the last round, at XLS-R 1B's and LightHuBERT's fc2;
- LayerNorm at D = 1280 (XLS-R 1B, pre-LN) with partial 8-row blocks, LayerNorm + RoPE at D = 512 and 1280;
- the Featurizer weighted sum and its backward against fp64 at every served layer count, up to kMaxLayers = 64, and at
  a size whose grid-stride loops wrap (forward: more float4 than the 132 x 8 x 256 capped grid; backward: past its
  132-block cap).

Separation of the GEMM bounds at long K. test_gemm_layouts_gpu._check asks the fp64 bound to be 50x the
accumulation-only bound for f16q8, a proxy for "a dropped k-step shows against the emulation". The ratio falls like
1 / sqrt(K) (accumulation ~ K^1.5, representation ~ K): with N(0, 1)-scaled operands it is ~49x at K = 5120 and ~41x
at K = 7680 (the floors and saturation terms keep the other magnitudes far above 50x). For f16q8 at K >= 5120, where
it is under 50x, the proxy is replaced by what it stands for, computed from the case's own operands (_dropped_steps):
- the emulation without the middle 16-wide k-step of the fp16 product must be over the accumulation bound on most
  elements;
- the emulation without either e4m3 correction product must be over it on a good share of elements (the check is a
  maximum over all of them).
A single 16-wide k-step of a correction product is ~2^-11 of an fp16 k-step; it sits at a few hundredths of the
accumulation bound here (and under a tenth at K = 4096), so no per-element bound of this kind can see it. It is printed,
not asserted.

Every case prints measured / bound."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from test_conformer_gpu import _rope_ref
from test_gemm_layouts_gpu import (_call, _check, _epilogue, _gemm_refs, _lib, _linear, _operands, _planes, _ptr,
                                   _stream, _through_planes)
from test_xls_r_gpu import _check_block

pytestmark = pytest.mark.gpu

U = 2.0**-24  # fp32 unit roundoff


# ------------------------------------------------------------------------------------------------
# GEMMs at the ports' production shapes
# ------------------------------------------------------------------------------------------------
PORT_LINEARS = [  # (layer, N, K, epilogue)
    ("xls_r_1b.qkv", 3840, 1280, "bias"),
    ("xls_r_1b.out_proj", 1280, 1280, "residual"),
    ("xls_r_1b.fc1", 5120, 1280, "gelu"),
    ("xls_r_1b.fc2", 1280, 5120, "out_pre"),
    ("xls_r_1b.post_extract_proj", 1280, 512, "row_mask"),
    ("xls_r_2b.qkv", 5760, 1920, "bias"),  # 45 tiles of 128: no clusters
    ("xls_r_2b.out_proj", 1920, 1920, "residual"),  # 1920 % 256 != 0: 128-wide tiles only
    ("xls_r_2b.fc1", 7680, 1920, "gelu"),
    ("xls_r_2b.fc2", 1920, 7680, "out_pre"),  # the project's longest contraction
    ("xls_r_2b.post_extract_proj", 1920, 512, "row_mask"),
    ("decoar2.post_extract_proj", 768, 128, "row_mask"),
    ("apc.gate_l0", 1536, 128, "bias"),
    ("apc.gate_l12", 1536, 512, "bias"),  # also the QKV of LightHuBERT's 512-wide subnet
    # LightHuBERT subnets: 384 wide (6 heads, FFN 1536), 512 (8 heads, FFN 2048), 640 (10 heads, FFN 2560); under f16q8
    # N = 384, 640, 1152 and 1920 are an odd number of 128-wide tiles, which run without clusters
    ("lighthubert_small.qkv", 1152, 384, "bias"),
    ("lighthubert_small.out_proj", 384, 384, "residual"),
    ("lighthubert_small.fc1", 1536, 384, "gelu"),
    ("lighthubert_small.fc2", 384, 1536, "out_pre"),
    ("lighthubert_small.post_extract_proj", 384, 512, "row_mask"),
    ("lighthubert_stage1_small.out_proj", 512, 512, "residual"),
    ("lighthubert_stage1_small.fc1", 2048, 512, "gelu"),
    ("lighthubert_stage1_small.fc2", 512, 2048, "out_pre"),  # tile width by M: test_lighthubert_fc2_tile_picker
    ("lighthubert_stage1_small.post_extract_proj", 512, 512, "row_mask"),
    ("lighthubert_base.qkv", 1920, 640, "bias"),
    ("lighthubert_base.out_proj", 640, 640, "residual"),
    ("lighthubert_base.fc1", 2560, 640, "gelu"),
    ("lighthubert_base.fc2", 640, 2560, "out_pre"),
    ("lighthubert_base.post_extract_proj", 640, 512, "row_mask"),
    ("decoar.proj", 1024, 128, "bias_planes"),  # into the LSTM's operand planes
    ("cpc.lstm_input", 1024, 256, "bias"),
    ("conformer.qk_pw1", 2048, 1024, "bias"),  # [q | k] and pointwise_conv1 of wav2vec2_conformer_rope
]
FBANK_BINS = 80  # K = 128 layers: columns 80.. of A (the CMVN kernel's planes) and W (the finalized weights) are zero
LONG_K = 5120  # f16q8 from here on: _dropped_steps in place of the 50x proxy


def _port_operands(M, N, K, mag, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, w = _operands(M, N, K, mag, g)
    if K == 128:
        a[:, FBANK_BINS:] = 0
        w[:, FBANK_BINS:] = 0
    return a, w, g


def _dropped_steps(what, a, w, e2):
    """f16q8 at long K: emulations that lost one k-step or one product, measured against the accumulation bound e2."""
    K = a.shape[1]
    a16, ah8, al8 = _planes(a, 1, False)
    w16, wh8, wl8 = _planes(w, 1, True)
    k = K // 32 * 16  # the middle 16-wide k-step

    def over(d):  # share of elements the loss moves by more than e2
        return (d.abs() > e2).double().mean().item()

    fp16_step = over(a16[:, k : k + 16] @ w16[:, k : k + 16].t())
    corr = min(over(al8 @ wh8.t()), over(ah8 @ wl8.t()))
    corr_step = ((al8[:, -16:] @ wh8[:, -16:].t()).abs() / e2).median().item()
    print(f"{what}: dropped fp16 k-step over the accumulation bound on {fp16_step:.3f} of elements, dropped correction "
          f"product on {corr:.3f}; a dropped correction k-step is {corr_step:.3f} of the bound (median)")
    assert fp16_step > 0.9, (what, "fp16 k-step", fp16_step)
    assert corr > 0.1, (what, "correction product", corr)


def _refs_and_separation(what, a, w, scheme):
    """_gemm_refs, and for f16q8 at K >= 5120 where the bounds are less than 50x apart, _dropped_steps in place of
    that proxy; returns (exact, emu, e1, e2, apart_check for _check)."""
    exact, emu, e1, e2 = _gemm_refs(a, w, scheme)
    replaced = scheme == 1 and a.shape[1] >= LONG_K and (e1 / e2).median().item() < 50.0
    if replaced:
        _dropped_steps(what, a, w, e2)
    return exact, emu, e1, e2, not replaced


def _tiles(N):
    return (128, 256) if N % 256 == 0 else (128,)


def _per_tile(N, scheme, launch):
    """launch(tile_n) -> (out, opts) at every tile width N allows; the outputs must agree bit for bit."""
    outs = {}
    for tile in _tiles(N):
        outs[tile], o = launch(tile)
        assert (o.scheme_used, o.tile_n_used) == (scheme, tile)
    for tile in outs:
        assert torch.equal(outs[tile], outs[128]), f"tile widths 128 and {tile} differ"
    return outs[128]


@pytest.mark.parametrize("M", [1, 127, 129, 1000, 4099])
@pytest.mark.parametrize("layer,N,K,epi", PORT_LINEARS, ids=[c[0] for c in PORT_LINEARS])
@pytest.mark.parametrize("scheme", [0, 1])
def test_port_linear(s3b_lib, scheme, layer, N, K, epi, M):
    """The layer's epilogue at both tile widths where N allows (bit-identical), against fp64 and against the scheme's
    emulated operand decomposition: residual (out_proj), GELU as fp32 and as the scheme's operand planes (fc1), out_pre
    before the residual (fc2), the row mask as fp32 and bf16 planes (post_extract_proj), bias only (QKV's GEMM, the
    recurrent models' input GEMMs), bias as fp32 and as the scheme's operand planes (DeCoAR's proj)."""
    what = f"{layer} s{scheme} M={M} N={N} K={K}"
    a, w, g = _port_operands(M, N, K, "unit", M * 131 + K * 7 + N + scheme)
    b = torch.randn(N, device="cuda", generator=g) * 0.5
    exact, emu, e1, e2, apart_check = _refs_and_separation(what, a, w, scheme)

    def check(tag, out, bias=b, gelu=False, res=None):
        ref1, b1 = _epilogue(exact, e1, bias, gelu=gelu, res=res)
        ref2, b2 = _epilogue(emu, e2, bias, gelu=gelu, res=res)
        _check(f"{what} {tag}", out, ref1, b1, ref2, b2, (e1, e2), scheme, apart_check=apart_check)

    if epi == "residual":
        r = torch.randn(M, N, device="cuda", generator=g)
        check("residual", _per_tile(N, scheme, lambda t: _linear(a, w, b, r, scheme=scheme, tile_n=t)), res=r)
    elif epi in ("bias", "bias_planes"):
        free = _per_tile(N, scheme, lambda t: _linear(a, w, b, scheme=scheme, tile_n=t))
        check("bias", free)
        if epi == "bias_planes":
            planes = _per_tile(N, scheme, lambda t: _linear(a, w, b, scheme=scheme, out_fmt=scheme, tile_n=t))
            assert torch.equal(planes, _through_planes(free, scheme)), "operand planes != planes of the fp32 output"
    elif epi == "gelu":
        h32 = _per_tile(N, scheme, lambda t: _linear(a, w, b, gelu=True, scheme=scheme, tile_n=t))
        check("gelu", h32, gelu=True)
        hp = _per_tile(N, scheme, lambda t: _linear(a, w, b, gelu=True, scheme=scheme, out_fmt=scheme, tile_n=t))
        assert torch.equal(hp, _through_planes(h32, scheme)), "GELU operand planes != planes of the fp32 output"
    elif epi == "out_pre":
        r = torch.randn(M, N, device="cuda", generator=g) * 3
        alone = _per_tile(N, scheme, lambda t: _linear(a, w, b, scheme=scheme, tile_n=t))
        for tile in _tiles(N):
            pre = torch.full((M, N), float("nan"), device="cuda")
            out, _ = _linear(a, w, b, r, scheme=scheme, tile_n=tile, out_pre=pre.data_ptr())
            assert torch.equal(pre, alone), tile
            assert torch.equal(out, pre + r), tile
        check("residual + out_pre", out, res=r)
    else:  # row_mask
        mask = (torch.rand(M, device="cuda", generator=g) < 0.3).to(torch.uint8)
        mask[-129:] = 1  # a whole padded tail tile
        keep = mask == 0
        free = _per_tile(N, scheme, lambda t: _linear(a, w, b, scheme=scheme, tile_n=t))
        check("bias", free)
        for fmt in (-1, 0):
            want = free if fmt < 0 else _through_planes(free, 0)
            out = _per_tile(N, scheme, lambda t: _linear(a, w, b, scheme=scheme, out_fmt=fmt, row_mask=mask.data_ptr(),
                                                          tile_n=t))
            assert torch.equal(out[~keep], torch.zeros_like(out[~keep])), fmt
            assert torch.equal(out[keep], want[keep]), fmt


PORT_SHAPES = list(dict.fromkeys((N, K) for _, N, K, _ in PORT_LINEARS))


@pytest.mark.parametrize("mag", ["small", "large"])
@pytest.mark.parametrize("N,K", PORT_SHAPES)
@pytest.mark.parametrize("scheme", [0, 1])
def test_port_linear_magnitudes(s3b_lib, scheme, N, K, mag):
    """x1e-3 (f16q8 residuals in e4m3's subnormals) and |a| ~ 3000, |w| ~ 40 (A_h8 and W_h8 saturate), M = 1000, as
    test_gemm_layouts_gpu.test_linear_magnitudes; planes only where fp16 holds the output."""
    M = 1000
    what = f"linear s{scheme} N={N} K={K} {mag}"
    a, w, _ = _port_operands(M, N, K, mag, K * 3 + N + scheme + len(mag))
    exact, emu, e1, e2, apart_check = _refs_and_separation(what, a, w, scheme)
    out, o = _linear(a, w, scheme=scheme)
    assert o.scheme_used == scheme
    ref1, b1 = _epilogue(exact, e1)
    ref2, b2 = _epilogue(emu, e2)
    _check(what, out, ref1, b1, ref2, b2, (e1, e2), scheme, frob=False, apart_check=apart_check)
    if mag == "small":
        for fmt in (0, 1):
            planes, _ = _linear(a, w, scheme=scheme, out_fmt=fmt)
            assert torch.equal(planes, _through_planes(out, fmt)), fmt


def test_xls_r_fc2_tile_picker(s3b_lib):
    """XLS-R 1B fc2 in f16q8 at a production batch (16 x 999 frames): the only layer whose tile width depends on M and
    the SM count. The picked width's result is bit for bit both forced widths'."""
    M, N, K = 16 * 999, 1280, 5120
    a, w, g = _port_operands(M, N, K, "unit", 5)
    b = torch.randn(N, device="cuda", generator=g)
    r = torch.randn(M, N, device="cuda", generator=g)
    auto, o = _linear(a, w, b, r, scheme=1)
    assert o.scheme_used == 1 and o.tile_n_used in (128, 256)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"fc2 M={M}: tile_n {o.tile_n_used} picked on {sms} SMs")
    for tile in (128, 256):
        forced, of = _linear(a, w, b, r, scheme=1, tile_n=tile)
        assert of.tile_n_used == tile
        assert torch.equal(forced, auto), tile


def _picked_bn(M, N, K, sms):
    """pick_bn's width (model.cu) for an f16q8 linear whose N is a multiple of 256: 256 columns at K >= 2048 when the
    last round of 256-wide tiles is empty or fills at least half of the SMs, 128 columns otherwise."""
    if K < 2048:
        return 128
    last = -(-M // 128) * (N // 256) % sms
    return 256 if last == 0 or last >= sms // 2 else 128


def test_lighthubert_fc2_tile_picker(s3b_lib):
    """fc2 of LightHuBERT's 512-wide subnet in f16q8 (N = 512, K = 2048), where the tile width depends on M and the SM
    count: at 128 * (SMs // 2) rows (8448 on 132 SMs) the last round of 256-wide tiles is empty or at least half full,
    at 1280 rows (20 tiles) it is under half full. The picked width is the rule's for this device, and forcing the
    other width gives the same bits."""
    N, K = 512, 2048
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    Ms = (128 * (sms // 2), 1280)
    assert [_picked_bn(M, N, K, sms) for M in Ms] == [256, 128], sms
    for M in Ms:
        a, w, g = _port_operands(M, N, K, "unit", M + 3)
        b = torch.randn(N, device="cuda", generator=g)
        r = torch.randn(M, N, device="cuda", generator=g)
        auto, o = _linear(a, w, b, r, scheme=1)
        want = _picked_bn(M, N, K, sms)
        print(f"lighthubert fc2 M={M}: tile_n {o.tile_n_used} picked on {sms} SMs, rule {want}")
        assert (o.scheme_used, o.tile_n_used) == (1, want), M
        forced, of = _linear(a, w, b, r, scheme=1, tile_n=384 - want)
        assert of.tile_n_used == 384 - want
        assert torch.equal(forced, auto), M


# ------------------------------------------------------------------------------------------------
# LayerNorm widths
# ------------------------------------------------------------------------------------------------
def _ln_params(D, g):
    return 1.0 + 0.3 * torch.randn(D, device="cuda", generator=g), 0.3 * torch.randn(D, device="cuda", generator=g)


LAYERNORM_WIDE_D = 1280  # XLS-R 1B's encoder LayerNorms (eps 1e-5)
ROPE_WIDTHS = [512, 1280]


@pytest.mark.parametrize("M", [1, 7, 8, 9, 1037])
@pytest.mark.parametrize("gelu", [0, 1])
def test_layernorm_1280(s3b_lib, gelu, M):
    """XLS-R 1B's pre-LN LayerNorm(1280): 8 rows per 256-thread block, so M % 8 != 0 leaves a partial last block whose
    idle warps must return without writing; the 8 rows after the output stay untouched."""
    D = LAYERNORM_WIDE_D
    g = torch.Generator(device="cuda").manual_seed(M * 2 + gelu)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 1
    gamma, beta = _ln_params(D, g)
    out = torch.full((M + 8, D), float("nan"), device="cuda")
    _call(s3b_lib.s3b_layernorm_f32, _ptr(x), M, D, _ptr(gamma), _ptr(beta), gelu, _ptr(out), _stream())
    ref = F.layer_norm(x.double(), (D,), gamma.double(), beta.double(), 1e-5)
    if gelu:
        ref = F.gelu(ref)
    _check_block(out[:M], ref, f"layernorm 1280 gelu={gelu} M={M}")
    assert torch.isnan(out[M:]).all(), "rows past M written"


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("B,T", [(3, 1), (2, 130)])
@pytest.mark.parametrize("D", ROPE_WIDTHS)
def test_layernorm_rope_widths(s3b_lib, D, B, T, fmt):
    """LayerNorm + RoPE at the two widths the kernel accepts besides 768 and 1024 (8 and 20 heads of 64), in both
    operand-plane formats."""
    M = B * T
    g = torch.Generator(device="cuda").manual_seed(D + T + fmt)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 0.5
    gamma, beta = _ln_params(D, g)
    inv_freq = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    y = torch.full_like(x, float("nan"))
    yr = torch.full_like(x, float("nan"))
    _call(s3b_lib.s3b_layernorm_rope_f32, _ptr(x), M, T, D, _ptr(gamma), _ptr(beta),
          (C.c_float * 32)(*inv_freq.tolist()), fmt, _ptr(y), _ptr(yr), _stream())
    ref = F.layer_norm(x.double(), (D,), gamma.double(), beta.double(), 1e-5)
    _check_block(y, ref, f"layernorm D={D} B={B} T={T} fmt={fmt}")
    _check_block(yr, _rope_ref(ref, T, inv_freq.cuda()), f"layernorm+rope D={D} B={B} T={T} fmt={fmt}")


# ------------------------------------------------------------------------------------------------
# Featurizer weighted sum
# ------------------------------------------------------------------------------------------------
WS_SHAPES = [  # (NL, B, T, D): hidden states per upstream and width
    (1, 2, 37, 1024),
    (3, 3, 37, 512),  # APC
    (3, 3, 37, 768),  # distilhubert
    (13, 3, 37, 768),  # base models, DeCoAR 2.0
    (13, 3, 37, 384),  # LightHuBERT subnets
    (13, 3, 37, 512),
    (13, 3, 37, 640),
    (25, 2, 49, 1024),  # large models
    (49, 2, 49, 1280),  # XLS-R 1B
    (49, 2, 49, 1920),  # XLS-R 2B
    (64, 2, 33, 512),  # kMaxLayers
    (49, 4, 999, 1920),  # 7.7 M floats per layer: both grid-stride loops wrap (1.5 GB)
]
FWD_THREADS = 132 * 8 * 256  # norm.cu: launch_weighted_sum's grid cap
BWD_BLOCKS, BWD_CHUNK = 132, 256 * 8  # launch_weighted_sum_bwd: float4 per block before the cap, the cap


def _ws_inputs(NL, B, T, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    hs = torch.randn(NL, B, T, D, device="cuda", generator=g)
    hs *= torch.linspace(0.5, 4.0, NL, device="cuda").view(NL, 1, 1, 1)  # layers of different scale
    w = torch.randn(NL, device="cuda", generator=g)  # signed: cancellation across layers
    gout = torch.randn(B, T, D, device="cuda", generator=g)
    return hs, w, gout


def _ws(hs, w):
    out = torch.full(hs.shape[1:], float("nan"), device="cuda")
    _call(_lib().load().s3b_weighted_sum, _ptr(hs), hs.shape[0], hs[0].numel(), _ptr(w), _ptr(out), _stream())
    return out


def _ws_bwd(hs, gout):
    grad = torch.full((hs.shape[0],), float("nan"), device="cuda")
    _call(_lib().load().s3b_weighted_sum_backward, _ptr(hs), hs.shape[0], hs[0].numel(), _ptr(gout), _ptr(grad),
          _stream())
    return grad


@pytest.mark.parametrize("NL,B,T,D", WS_SHAPES)
def test_weighted_sum(s3b_lib, NL, B, T, D):
    """Forward against the fp64 sum_l w_l h_l within NL u sum_l |w_l h_l| (an fp32 FMA chain in layer order), and bit
    for bit across two calls; backward against fp64 <h_l, g> within (4 + per-thread iterations + 5 + 8 + blocks) u
    sum |h_l g| (the float4 dot and the serial loop, the warp butterfly, the block's 8 partials, the atomics)."""
    hs, w, gout = _ws_inputs(NL, B, T, D, NL * 7 + T + D)
    n4 = hs[0].numel() // 4
    bwd_blocks = min(-(-n4 // BWD_CHUNK), BWD_BLOCKS)
    iters = -(-n4 // (bwd_blocks * 256))
    if T == 999:  # the case exists to run the loops past their grids
        assert n4 > FWD_THREADS and -(-n4 // BWD_CHUNK) > BWD_BLOCKS

    out = _ws(hs, w)
    assert torch.equal(_ws(hs, w), out), "forward differs between two calls"
    grad = _ws_bwd(hs, gout)

    ref = torch.zeros(hs.shape[1:], dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(ref)
    gd = gout.double()
    gref = torch.zeros(NL, dtype=torch.float64, device="cuda")
    gmag = torch.zeros_like(gref)
    for l in range(NL):
        h = hs[l].double()
        t = w[l].double() * h
        ref += t
        mag += t.abs()
        p = h * gd
        gref[l] = p.sum()
        gmag[l] = p.abs().sum()
    assert torch.isfinite(out).all() and torch.isfinite(grad).all()
    err = (out.double() - ref).abs()
    r_fwd = (err / (NL * U * mag)).max().item()
    r_bwd = ((grad.double() - gref).abs() / ((4 + iters + 5 + 8 + bwd_blocks) * U * gmag)).max().item()
    print(f"weighted sum NL={NL} B={B} T={T} D={D} (backward: {bwd_blocks} blocks x {iters} iterations): "
          f"measured/bound forward {r_fwd:.3f}, backward {r_bwd:.3f}")
    assert r_fwd <= 1.0, r_fwd
    assert r_bwd <= 1.0, r_bwd


def test_weighted_sum_refusals(s3b_lib):
    """More layers than the kernel's shared table (65 > kMaxLayers), and a layer size that is not whole float4. Then,
    forward and backward alike, with the argument named in the message: num < 1 (a negative num passed the old
    `NL > 64` check and let all 256 threads index the 64-entry table), negative layer sizes (a negative multiple of 4
    passed as a huge size_t), and hs / out / grad_out off the 16-byte alignment of their float4 accesses. Nothing is
    written by a refused call."""
    L = _lib().load()
    hs = torch.zeros(65 * 8, device="cuda")
    w = torch.zeros(65, device="cuda")
    out = torch.zeros(8, device="cuda")
    grad = torch.zeros(65, device="cuda")
    assert L.s3b_weighted_sum(_ptr(hs), 65, 8, _ptr(w), _ptr(out), _stream()) != 0
    assert L.s3b_weighted_sum(_ptr(hs), 64, 8, _ptr(w), _ptr(out), _stream()) == 0  # the edge itself runs
    assert L.s3b_weighted_sum(_ptr(hs), 3, 6, _ptr(w), _ptr(out), _stream()) != 0
    assert L.s3b_weighted_sum_backward(_ptr(hs), 3, 6, _ptr(out), _ptr(grad), _stream()) != 0
    torch.cuda.synchronize()

    def refused(fn, args, what):
        rc = fn(*args, _stream())
        msg = L.s3b_last_error().decode()
        assert rc != 0 and msg.startswith(what + " = "), (fn, what, msg)

    hs.fill_(float("nan"))
    out_nan = torch.full((12,), float("nan"), device="cuda")
    grad.fill_(float("nan"))
    fwd, bwd = L.s3b_weighted_sum, L.s3b_weighted_sum_backward
    # first the cases a library without these checks would still run harmlessly (empty layers launch nothing), so that
    # such a library fails here before any of the out-of-bounds launches below
    refused(fwd, (_ptr(hs), 0, 0, _ptr(w), _ptr(out_nan)), "num")
    refused(bwd, (_ptr(hs), 0, 0, _ptr(out_nan), _ptr(grad)), "num")
    for num in (-1, -(2**31), 65):
        refused(fwd, (_ptr(hs), num, 8, _ptr(w), _ptr(out_nan)), "num")
        refused(bwd, (_ptr(hs), num, 8, _ptr(out_nan), _ptr(grad)), "num")
    for n in (-4, -(2**62), 6):
        refused(fwd, (_ptr(hs), 3, n, _ptr(w), _ptr(out_nan)), "n_per_layer")
        refused(bwd, (_ptr(hs), 3, n, _ptr(out_nan), _ptr(grad)), "n_per_layer")
    for off in (1, 2, 3):
        hs_off, out_off = C.c_void_p(hs.data_ptr() + 4 * off), C.c_void_p(out_nan.data_ptr() + 4 * off)
        refused(fwd, (hs_off, 3, 8, _ptr(w), _ptr(out_nan)), "hs")
        refused(bwd, (hs_off, 3, 8, _ptr(out_nan), _ptr(grad)), "hs")
        refused(fwd, (_ptr(hs), 3, 8, _ptr(w), out_off), "out")
        refused(bwd, (_ptr(hs), 3, 8, out_off, _ptr(grad)), "grad_out")
    torch.cuda.synchronize()
    assert torch.isnan(out_nan).all() and torch.isnan(grad).all()


@pytest.mark.parametrize("NL,D", [(13, 768), (49, 1280)])
def test_featurizer_paths_agree(s3b_lib, NL, D):
    """upstream.featurizer.weighted_sum on slices of one [NL, B, T, D] buffer (read in place) and on separately
    allocated layers (torch.stack first): bit-identical, and bit for bit the direct call on the buffer."""
    from s3prl_b200.upstream.featurizer import _stacked_view, weighted_sum

    hs, _, _ = _ws_inputs(NL, 3, 57, D, NL + D)
    views = [hs[l] for l in range(NL)]
    copies = [hs[l].clone() for l in range(NL)]
    assert _stacked_view(views).data_ptr() == hs.data_ptr()
    assert _stacked_view(copies).data_ptr() not in [c.data_ptr() for c in copies]
    w = torch.randn(NL, device="cuda").softmax(-1)
    in_place = weighted_sum(views, w)
    stacked = weighted_sum(copies, w)
    torch.cuda.synchronize()
    assert torch.equal(in_place, stacked)
    assert torch.equal(in_place, _ws(hs, w))
