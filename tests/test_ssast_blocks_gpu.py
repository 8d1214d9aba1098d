"""SSAST's kernels per element at every window geometry the model serves (SSAST_WINDOWS): the smallest windows, 1 s,
2.5 s and 10 s, windows whose rows per window sit on each side of one and two 128-row GEMM tiles, a window whose
sample count is not a multiple of the 160-sample hop, and the windows around the positional table's crop /
interpolate boundary (the pretrained t_dim - 1, t_dim, t_dim + 1).

- The patch GEMM (s3b_ssast_embed_f32, N = 768, K = 256; model.cu ssast_patch_params): its output block per window is
  2 + P rows, two more than the GEMM's valid rows, and starts two rows in. Frame model: an implicit 2-tap convolution,
  row t of a window reads feature rows t and t + 1; patch model: [P][256] x [768][256]^T per window. Checked per
  element against fp64 and against the scheme's operand-split emulation, with the bounds of
  tests/test_gemm_layouts_gpu.py (_gemm_refs) plus the bias and positional-row adds; the class rows bit for bit.
- No window reads another's rows: window 1 between all-NaN windows 0 and 2 gives the bits of window 1 alone.
- Attention over window token blocks (SB sequences of ST = P + 2 tokens, every key valid) and the QKV scatter at the
  same token counts, against fp64.
- LayerNorm at eps 1e-6 written as operand planes, as a pre-LN layer's LN1 / LN2 write them.
- The output fold bit for bit and the windowed fbank per element against tests/ssast_oracle.py.
- Whole forwards of both models at the new windows against the fp64 oracle, every element of every hidden state.
Every per-element check prints measured / bound."""
from __future__ import annotations

import ctypes as C
import functools
import math
import sys
from collections import namedtuple
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))

import ssast_oracle as SO  # noqa: E402
from s3prl_b200.upstream.ssast import KINDS, geometry  # noqa: E402
from test_gemm_layouts_gpu import _check, _epilogue, _gemm_refs, _through_planes  # noqa: E402
from test_ssast_gpu import _assert_close, _embed, _expert, _structured, _wavs  # noqa: E402
from test_xls_r_gpu import LOG2E, _attention, _check_block, _ptr, _stream  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0**-24  # fp32 unit roundoff
D, H, HD = 768, 12, 64

# ------------------------------------------------------------------------------------------------
# the window geometries
# ------------------------------------------------------------------------------------------------
# the pretrained positional table's time patches ((1024 - ts) // ts + 1 of the released checkpoints' 1024 frames):
# a window with fewer is cropped from it, one with as many or more is interpolated (regrid_pos_embed)
PRETRAINED_T_DIM = {kind: (1024 - ts) // ts + 1 for kind, ((_, ts), _) in KINDS.items()}


def _frame_secs(t_dim):
    """The frame model's window of t_dim time patches: TL = t_dim + 1 feature rows of 160 samples."""
    return (t_dim + 1) * 160 / 16000


def _patch_secs(t_dim):
    """The patch model's window of t_dim time patches: TL = 16 + 10 (t_dim - 1) feature rows of 160 samples."""
    return (16 + 10 * (t_dim - 1)) * 160 / 16000


Window = namedtuple("Window", "kind secs what want")  # want: the geometry() values the row is there for
_PF, _PP = PRETRAINED_T_DIM["frame"], PRETRAINED_T_DIM["patch"]
SSAST_WINDOWS = [
    Window("frame", 0.025, "smallest", {"S": 400, "TL": 2, "t_dim": 1}),
    Window("frame", 1.0, "1 s", {"S": 16000, "t_dim": 99}),
    Window("frame", 2.5, "2.5 s", {"S": 40000, "t_dim": 249}),
    Window("frame", 10.0, "largest", {"S": 160000, "t_dim": 999}),
    Window("frame", _frame_secs(127), "tile edge", {"t_dim": 127}),
    Window("frame", _frame_secs(128), "tile edge", {"t_dim": 128}),
    Window("frame", _frame_secs(129), "tile edge", {"t_dim": 129}),
    Window("frame", 1.001, "off the hop", {"S": 16015, "t_dim": 99}),
    Window("frame", _frame_secs(_PF - 1), "regrid", {"t_dim": _PF - 1}),
    Window("frame", _frame_secs(_PF), "regrid", {"t_dim": _PF}),
    Window("frame", _frame_secs(_PF + 1), "regrid", {"t_dim": _PF + 1}),
    Window("patch", 0.16, "smallest", {"S": 2560, "t_dim": 1, "P": 12}),
    Window("patch", 1.0, "1 s", {"S": 16000, "P": 108}),
    Window("patch", 2.5, "2.5 s", {"S": 40000, "P": 288}),
    Window("patch", 10.0, "largest", {"S": 160000, "P": 1188}),
    Window("patch", _patch_secs(10), "tile edge", {"P": 120}),
    Window("patch", _patch_secs(11), "tile edge", {"P": 132}),
    Window("patch", _patch_secs(21), "tile edge", {"P": 252}),
    Window("patch", _patch_secs(22), "tile edge", {"P": 264}),
    Window("patch", 1.001, "off the hop", {"S": 16015, "P": 108}),
    Window("patch", _patch_secs(_PP - 1), "regrid", {"t_dim": _PP - 1}),
    Window("patch", _patch_secs(_PP), "regrid", {"t_dim": _PP}),
    Window("patch", _patch_secs(_PP + 1), "regrid", {"t_dim": _PP + 1}),
]
WINDOW_IDS = [f"{w.kind}-{w.secs:g}" for w in SSAST_WINDOWS]
# the patch GEMM's rows: (layer, N, K, kind, window_secs); tests/test_port_coverage_cpu.py counts (N, K) as covered
PATCH_GEMMS = [(f"ssast_{w.kind}.patch_embed", D, 256, w.kind, w.secs) for w in SSAST_WINDOWS]
# token counts ST = P + 2 of a window's sequence, each with the window count the attention test runs: 320 (32 x 10 s
# in 1 s windows) where ST <= 131, 8 at the long ones
TOKENS = sorted({geometry(w.kind, w.secs)["P"] + 2 for w in SSAST_WINDOWS})
SHORT_ST = 131


def _windows_for(ST):
    return 320 if ST <= SHORT_ST else 8


# ------------------------------------------------------------------------------------------------
# the patch GEMM
# ------------------------------------------------------------------------------------------------
def _embed_inputs(kind, P, mag, seed):
    """Weights in the checkpoint's layout and a [1, 2 + P, 768] positional table, at the scale of the GEMM output:
    unit (normalised-fbank features, weights of fan-in variance) or 1e-3 of both operands (the f16q8 residuals in
    e4m3's subnormals), bias, tokens and table 1e-6 of unit there."""
    (fs, ts), _ = KINDS[kind]
    g = torch.Generator().manual_seed(seed)
    s = 1.0 if mag == "unit" else 1e-3
    y = s * s
    return {
        "patch_embed.proj.weight": torch.randn(D, 1, fs, ts, generator=g) / math.sqrt(fs * ts) * s,
        "patch_embed.proj.bias": torch.randn(D, generator=g) * 0.02 * y,
        "cls_token": torch.randn(1, 1, D, generator=g) * 0.02 * y,
        "dist_token": torch.randn(1, 1, D, generator=g) * 0.02 * y,
        "pos_embed": torch.randn(1, 2 + P, D, generator=g) * 0.02 * y,
    }


def _gemm_view(kind, feat, sd):
    """The GEMM the kernel runs, as fp32 matrices: A [SB * rows][256] from the features the call received (frame
    model: rows t and t + 1 of a window concatenated; patch model: ssast_oracle.patch_operand) and W [768][256] with
    column dt * 128 + f (frame model, as finalize_ssast lays it out) or kf * 16 + kt (patch model)."""
    w = sd["patch_embed.proj.weight"]
    if kind == "frame":
        a = torch.cat([feat[:, :-1], feat[:, 1:]], dim=-1)
        wk = w[:, 0].permute(0, 2, 1).reshape(D, 256)
    else:
        a = SO.patch_operand(feat, "patch")
        wk = w.reshape(D, 256)
    return a.reshape(-1, 256).contiguous(), wk.contiguous()


def _features(SB, TL, mag, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(SB, TL, 128, generator=g) * 0.4 - 0.2) * (1.0 if mag == "unit" else 1e-3)


@pytest.mark.parametrize("mag", ["unit", "small"])
@pytest.mark.parametrize("scheme", [0, 1], ids=["bf16x3", "f16q8"])
@pytest.mark.parametrize("win", SSAST_WINDOWS, ids=WINDOW_IDS)
def test_patch_gemm_matches_fp64_and_emulation(s3b_lib, win, scheme, mag):
    """Rows 2.. of every window: fp32(GEMM + bias) + pos[2 + p] against fp64 and the emulation (the bias add's and the
    table add's roundings in the bounds); rows 0 and 1 exactly fp32(cls + pos[0]) and fp32(dist + pos[1])."""
    geo = geometry(win.kind, win.secs)
    TL, P = geo["TL"], geo["P"]
    SB = 3
    what = f"ssast {win.kind} patch GEMM {win.secs:g} s (TL={TL}, P={P}) s{scheme} {mag}"
    sd = _embed_inputs(win.kind, P, mag, TL + 7 * scheme + len(mag))
    feat = _features(SB, TL, mag, TL * 3 + scheme + len(mag))
    _, out = _embed(s3b_lib, win.kind, feat, sd, scheme)
    a, wk = _gemm_view(win.kind, feat, sd)
    exact, emu, e1, e2 = _gemm_refs(a.cuda(), wk.cuda(), scheme)
    pos = sd["pos_embed"][0].double().cuda()
    rows = pos[2:].repeat(SB, 1)  # [SB * P][768]

    def ref(pre, e):
        v, b = _epilogue(pre, e, sd["patch_embed.proj.bias"].cuda())
        v = v + rows
        return v, b + U * v.abs()

    ref1, b1 = ref(exact, e1)
    ref2, b2 = ref(emu, e2)
    got = out[:, 2:].reshape(-1, D)
    _check(what, got, ref1, b1, ref2, b2, (e1, e2), scheme, frob=mag == "unit")
    cls = (sd["cls_token"][0, 0] + sd["pos_embed"][0, 0]).expand(SB, -1)
    dist = (sd["dist_token"][0, 0] + sd["pos_embed"][0, 1]).expand(SB, -1)
    assert torch.equal(out[:, 0].cpu(), cls) and torch.equal(out[:, 1].cpu(), dist), what


@pytest.mark.parametrize("scheme", [0, 1], ids=["bf16x3", "f16q8"])
@pytest.mark.parametrize("win", SSAST_WINDOWS, ids=WINDOW_IDS)
def test_patch_gemm_reads_only_its_window(s3b_lib, win, scheme):
    """Window 1 of three whose windows 0 and 2 are all NaN gives the 2 + P rows of window 1 run alone, bit for bit: the
    frame model's last row reads feature row TL - 1 and the patch model's last time patch rows up to TL - 1, and an M
    tile that straddles a window edge must not mix the windows' rows."""
    geo = geometry(win.kind, win.secs)
    TL, P = geo["TL"], geo["P"]
    sd = _embed_inputs(win.kind, P, "unit", TL + 11 * scheme)
    feat = _features(3, TL, "unit", TL + scheme)
    _, alone = _embed(s3b_lib, win.kind, feat[1:2].contiguous(), sd, scheme)
    feat[0], feat[2] = float("nan"), float("nan")
    _, out = _embed(s3b_lib, win.kind, feat, sd, scheme)
    assert torch.isfinite(alone).all()
    assert torch.equal(out[1], alone[0])
    print(f"ssast {win.kind} {win.secs:g} s s{scheme}: window 1 between NaN windows bit-identical ({P + 2} rows)")


# ------------------------------------------------------------------------------------------------
# attention and the QKV scatter over window token blocks
# ------------------------------------------------------------------------------------------------
def _attention_ref(q, k, v):
    """fp64 softmax(q k^T / 8) v per head, in chunks of windows so that the scores stay under ~1 GB."""
    SB, ST, _ = q.shape
    out = torch.empty(q.shape, dtype=torch.float64, device=q.device)
    chunk = max(1, 2**30 // (H * ST * ST * 8))
    for s in range(0, SB, chunk):
        qh, kh, vh = (t[s:s + chunk].double().view(-1, ST, H, HD).transpose(1, 2) for t in (q, k, v))
        a = (qh @ kh.transpose(-1, -2) * HD**-0.5).softmax(-1)
        out[s:s + chunk] = (a @ vh).transpose(1, 2).reshape(-1, ST, D)
    return out


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("ST", TOKENS)
def test_window_attention(s3b_lib, ST, fmt):
    """SB windows of ST tokens, 12 heads of 64, every key valid, as the encoder runs SSAST (no key mask)."""
    SB = _windows_for(ST)
    g = torch.Generator(device="cuda").manual_seed(ST * 2 + fmt)
    q, k, v = (torch.randn(SB, ST, D, device="cuda", generator=g) for _ in range(3))
    out = _attention(q, k, v, [ST] * SB, H, HD, fmt)
    _check_block(out, _attention_ref(q, k, v), f"ssast attention SB={SB} ST={ST} ctx_format={fmt}")


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("ST", TOKENS)
def test_window_attention_uniform_keys(s3b_lib, ST, fmt):
    """Keys identical within each window, as a silent window's patches are before the positional table: the softmax
    is uniform over all ST keys and the context is the mean of the window's values."""
    SB = _windows_for(ST)
    g = torch.Generator(device="cuda").manual_seed(ST * 3 + fmt)
    q, v = (torch.randn(SB, ST, D, device="cuda", generator=g) for _ in range(2))
    k = torch.randn(SB, 1, D, device="cuda", generator=g).expand(SB, ST, D).contiguous()
    out = _attention(q, k, v, [ST] * SB, H, HD, fmt)
    ref = v.double().mean(1, keepdim=True).expand(SB, ST, D)
    _check_block(out, ref, f"ssast attention uniform keys SB={SB} ST={ST} ctx_format={fmt}")


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("ST", TOKENS)
def test_window_qkv_scatter(s3b_lib, ST, scheme):
    """q, k as [SB][12][ST][64] (q scaled by 1/8 * log2(e)) and v^T as [SB][12][64][STp], STp = ST rounded up to 8,
    against fp64; most ST here are not multiples of 8, and the padding columns of v^T stay zero."""
    from s3prl_b200 import lib

    B = 8 if ST <= SHORT_ST else 2
    Tp = (ST + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(ST + scheme)
    x = torch.randn(B, ST, D, device="cuda", generator=g)
    w = torch.randn(3 * D, D, device="cuda", generator=g) / D**0.5
    b = torch.randn(3 * D, device="cuda", generator=g) * 0.1
    q = torch.full((B, H, ST, HD), float("nan"), device="cuda")
    k = torch.full_like(q, float("nan"))
    vt = torch.full((B, H, HD, Tp), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_qkv_hd_f32(_ptr(x), _ptr(w), _ptr(b), B, ST, H, HD, scheme, _ptr(q), _ptr(k), _ptr(vt),
                                     _stream()))
    torch.cuda.synchronize()
    y = (x.double() @ w.double().t() + b.double()).view(B, ST, 3, H, HD)
    scale = float(torch.tensor(LOG2E / math.sqrt(HD), dtype=torch.float32))
    _check_block(q, y[:, :, 0].transpose(1, 2) * scale, f"ssast qkv q B={B} ST={ST} scheme={scheme}")
    _check_block(k, y[:, :, 1].transpose(1, 2), f"ssast qkv k B={B} ST={ST} scheme={scheme}")
    _check_block(vt[..., :ST], y[:, :, 2].permute(0, 2, 3, 1), f"ssast qkv v^T B={B} ST={ST} scheme={scheme}")
    assert torch.equal(vt[..., ST:], torch.zeros_like(vt[..., ST:]))


# ------------------------------------------------------------------------------------------------
# LayerNorm at eps 1e-6 into operand planes
# ------------------------------------------------------------------------------------------------
def _ln_eps(s3b_lib, x, gm, bt, eps, fmt=None):
    """s3b_layernorm_eps_f32 (fmt None: fp32) or s3b_layernorm_eps_planes_f32 (planes of fmt, decoded)."""
    from s3prl_b200 import lib

    M = x.shape[0]
    out = torch.full_like(x, float("nan"))
    s = torch.cuda.current_stream().cuda_stream
    if fmt is None:
        lib.check(s3b_lib.s3b_layernorm_eps_f32(x.data_ptr(), M, D, gm.data_ptr(), bt.data_ptr(), 0, eps,
                                                out.data_ptr(), s))
    else:
        lib.check(s3b_lib.s3b_layernorm_eps_planes_f32(x.data_ptr(), M, D, gm.data_ptr(), bt.data_ptr(), eps, fmt,
                                                       out.data_ptr(), s))
    torch.cuda.synchronize()
    return out


LN_EPS = 1e-6  # the DeiT blocks' LayerNorm eps
# (windows SB, tokens ST): the smallest windows of both models, the longest short one and both models' 10 s windows
LN_GEOMETRIES = [(_windows_for(st), st) for st in (3, 14, SHORT_ST, 1001, 1190)]


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("SB,ST", LN_GEOMETRIES)
def test_layernorm_eps_1e6_planes(s3b_lib, SB, ST, fmt):
    """LN1 / LN2 of SSAST's blocks as the forward writes them (operand planes only), at M = SB * ST rows: bit for bit
    the planes of the same kernel's fp32 output, and per element against fp64 layer_norm(eps=1e-6) within the fp32
    kernel's 2e-6 of the row's largest output plus the planes' representation error (bf16 hi/lo: 2^-16 |y|; f16q8:
    the fp16 plane's residual in e4m3, 2^-15 |y| + 2^-21). The first rows have a variance near eps, where eps 1e-5
    would be over the bound."""
    M = SB * ST
    g = torch.Generator(device="cuda").manual_seed(M + fmt)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 5
    small = min(500, M // 2)
    x[:small] = 1e-3 * torch.randn(small, D, device="cuda", generator=g)  # variance ~ eps: eps decides the scale
    gm = 1 + 0.3 * torch.randn(D, device="cuda", generator=g)
    bt = 0.3 * torch.randn(D, device="cuda", generator=g)
    f32 = _ln_eps(s3b_lib, x, gm, bt, LN_EPS)
    planes = _ln_eps(s3b_lib, x, gm, bt, LN_EPS, fmt)
    assert torch.equal(planes, _through_planes(f32, fmt)), "planes != planes of the fp32 output"
    ref = F.layer_norm(x.double(), (D,), gm.double(), bt.double(), LN_EPS)
    rep = 2.0**-16 * ref.abs() if fmt == 0 else 2.0**-15 * ref.abs() + 2.0**-21
    bound = 2e-6 * ref.abs().amax(-1, keepdim=True) + rep
    r = ((planes.double() - ref).abs() / bound).max().item()
    other = F.layer_norm(x[:small].double(), (D,), gm.double(), bt.double(), 1e-5)
    r5 = ((planes[:small].double() - other).abs() / bound[:small]).max().item()
    print(f"layernorm eps 1e-6 planes fmt={fmt} M={M}: measured/bound {r:.3f}; against eps 1e-5 {r5:.1f}")
    assert r < 1.0
    assert r5 > 10.0  # the small-variance rows tell the two eps apart


# ------------------------------------------------------------------------------------------------
# the output fold and the windowed fbank
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("win", SSAST_WINDOWS, ids=WINDOW_IDS)
def test_fold_at_every_window(s3b_lib, win):
    """s3b_ssast_fold_f32 bit for bit against ssast_oracle.fold, for T = 1, one window and one frame, and all
    nseg * t_dim frames."""
    from s3prl_b200 import lib

    geo = geometry(win.kind, win.secs)
    B, nseg, f_dim, tdim = 2, 3, geo["f_dim"], geo["t_dim"]
    x = torch.randn(B * nseg, 2 + geo["P"], D, device="cuda")
    for T in sorted({1, min(tdim + 1, nseg * tdim), nseg * tdim}):
        out = torch.full((B, T, f_dim * D), float("nan"), device="cuda")
        lib.check(s3b_lib.s3b_ssast_fold_f32(x.data_ptr(), B, nseg, geo["TL"], int(win.kind == "patch"), T,
                                             out.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), SO.fold(x.cpu(), B, f_dim, T)), T


@pytest.mark.parametrize("secs", [0.025, 0.16, 10.0, 1.001])
def test_fbank_at_new_windows(s3b_lib, secs):
    """s3b_ssast_fbank_f32 against ssast_oracle.fbank_windows on structured audio: the smallest windows of both
    models (one and 14 fbank frames), the largest, and a window of 16015 samples, whose windows start off the
    160-sample hop. Windows that start past an utterance's end are silent: exactly the floor.
    Bound per element: spectral_ref.ssast_bounds' interval on each zero-padded window (the fp64 log-mel's stage-by-
    stage interval through (f + 4.2677393) / 9.1379948 with its roundings). Its FFT bound is absolute per frame, so a
    bin far below its frame's peak (past 4.3 s the chirp of _structured aliases, and its frames' lowest mel bins sit
    1e-10 under their peak) gets the wide interval its fp32 spectrum needs."""
    import spectral_ref as R

    from s3prl_b200 import lib

    S = geometry("frame", secs)["S"]
    lens = [40000, 16000, 1, 23457, 15999] if S < 160000 else [170001, 16000, 1, 160000, 159999]
    wavs = [_structured(n, i) for i, n in enumerate(lens)]
    L = max(lens)
    nseg, TL = -(-L // S), S // 160
    dev = [w.cuda() for w in wavs]
    out = torch.full((len(lens) * nseg, TL, 128), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_ssast_fbank_f32((C.c_void_p * len(lens))(*[w.data_ptr() for w in dev]),
                                          (C.c_int64 * len(lens))(*lens), len(lens), L, S, out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    ref = SO.fbank_windows(wavs, S, L)
    got = out.cpu().double()
    m = 1 + (S - 400) // 160
    assert torch.all(got[:, m:] == 0)  # the appended rows
    floor = (math.log(SO.FLOOR) + 4.2677393) / (4.5689974 * 2)
    silent = torch.tensor([s * S >= n for n in lens for s in range(nseg)])
    assert silent.any() and ref[silent][:, :m].eq(floor).all()
    assert (got[silent][:, :m] - floor).abs().max().item() < 1e-6
    eps_w = R.bank_eps("kaldi", 128)
    r = 0.0
    for b, w in enumerate(wavs):
        x = torch.zeros(nseg * S)
        x[:len(w)] = w
        for s in range(nseg):
            if s * S < len(w):
                sb = R.ssast_bounds(x[s * S:(s + 1) * S], eps_w)
                assert (sb["y"] - ref[b * nseg + s, :m]).abs().max() <= 1e-12
                r = max(r, R.interval_ratio(got[b * nseg + s, :m], sb["y"], sb["ylo"], sb["yhi"]).max().item())
    d = (got[:, :m] - ref[:, :m]).abs()
    print(f"ssast fbank S={S} ({nseg} windows of {m} frames): max |err| {d.max().item():.2e} (normalised units), "
          f"measured/bound {r:.3f}")
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------
# whole forwards
# ------------------------------------------------------------------------------------------------
FORWARD_WINDOWS = [w for w in SSAST_WINDOWS if w.what in ("smallest", "tile edge", "off the hop", "regrid")]


@functools.lru_cache(maxsize=2)
def _oracle(kind, secs, lens, seed):
    """The 12 hidden states of ssast_oracle's fp64 forward (its fbank on the CPU, the rest in fp64 on the GPU)."""
    from s3prl_b200.upstream.ssast import fabricate_ssast_state_dict, num_frames, prepare_ssast_tensors

    geo = geometry(kind, secs)
    sd = prepare_ssast_tensors(fabricate_ssast_state_dict(seed, kind), kind, secs)
    sd = {k: v.double().cuda() for k, v in sd.items()}
    wavs = _wavs(lens, seed=seed + 20)
    L = max(lens)
    x = SO.embed(SO.fbank_windows(wavs, geo["S"], L).cuda(), sd)
    hidden = []
    for l in range(12):
        x = SO.block(x, sd, l)
        hidden.append(SO.fold(x, len(lens), geo["f_dim"], num_frames(kind, secs, L)).cpu())
    return wavs, hidden


def _forward_lens(S):
    """1 sample, k S - 1, k S and k S + 1 (k = 3 for windows under 1 s, else 1) and one in between."""
    k = 3 if S < 16000 else 1
    return (1, k * S - 1, k * S, k * S + 1, k * S // 2 + 7)


@pytest.mark.parametrize("scheme", ["f16q8", "bf16x3"])
@pytest.mark.parametrize("win", FORWARD_WINDOWS, ids=[f"{w.kind}-{w.secs:g}" for w in FORWARD_WINDOWS])
def test_forward_matches_oracle_at_window(s3b_lib, win, scheme):
    """Every element of every hidden state against the fp64 oracle, with test_ssast_gpu's budgets (2e-4 relative
    Frobenius, 1e-3 of the state's largest element)."""
    geo = geometry(win.kind, win.secs)
    lens = _forward_lens(geo["S"])
    wavs, ref = _oracle(win.kind, win.secs, lens, 6)
    ex = _expert(scheme, kind=win.kind, window_secs=win.secs, seed=6)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    assert len(hs) == len(ref) == 12
    for l, (h, r) in enumerate(zip(hs, ref)):
        assert h.shape == r.shape, (l, h.shape, r.shape)
        _assert_close(f"ssast {win.kind} {win.secs:g} s lens={lens} {scheme} state {l}", h.cpu(), r)
