"""MAE-AST on the GPU: the front end (povey 128-bin fbank, batch norm, unfold into patch operand planes) per element
against fp64; the (768, 256) projection against fp64 and the operand-split emulation; the positions + LayerNorm
kernel; attention at MAE-AST's key counts; whole forwards of both models against the executed reference's goldens and
the fp64 oracle in both operand schemes; a long-lived model that gives the bits of a fresh one; the local entry."""
from __future__ import annotations

import ctypes as C
import math
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import mae_ast_oracle as MO  # noqa: E402
from test_gemm_layouts_gpu import _check, _epilogue, _gemm_refs, _linear, _through_planes  # noqa: E402
from test_ssast_gpu import _assert_close, _structured, _wavs  # noqa: E402
from test_xls_r_gpu import _attention, _check_block, _ptr, _stream  # noqa: E402

pytestmark = pytest.mark.gpu

D, H, HD = 768, 12, 64
GOLDENS = ("mae_ast_frame", "mae_ast_patch", "mae_ast_frame_c2", "mae_ast_variant")
# post_extract_proj's rows M = B T' nv on each side of one and two 128-row tiles; tests/test_mae_ast_cpu.py checks that
# every linear of the model has a row here or in the encoder tables it names
PROJ_ROWS = [127, 128, 129, 255, 256, 257, 32 * 499]
# valid key counts of a sequence of N tokens: multiples of 8 (the patch model's nv) that are not multiples of the
# attention kernel's 64-key block, with the full and the one-patch sequence; N = the 10 s patch model's 62 x 8 tokens,
# the 1 s patch model's 6 x 8, and the 10 s frame model's 499
ATTN_CASES = [(496, [496, 200, 8, 136]), (48, [48, 8, 40]), (499, [499, 248, 8, 392])]


def _bn(rm, rv):
    """The affine map the library folds the eval batch norm into: y = x * a + c (fp64 -> fp32, as finalize)."""
    a = 0.5 / math.sqrt(rv + 1e-5)
    return torch.tensor(a, dtype=torch.float32).item(), torch.tensor(-rm * a, dtype=torch.float32).item()


def _frontend(s3b_lib, wavs, kind, rm, rv, fmt, guard=0):
    """s3b_mae_ast_fbank_f32: (fp32 out, decoded planes), each [B, T' nv, 256], plus `guard` NaN rows after it."""
    from s3prl_b200 import lib
    from s3prl_b200.upstream.mae_ast import KINDS, num_frames

    lens = [len(w) for w in wavs]
    L = max(lens)
    N = num_frames(kind, L) * (128 // KINDS[kind][1])
    dev = [w.cuda() for w in wavs]
    out = torch.full((len(wavs) * N + guard, 256), float("nan"), device="cuda")
    planes = torch.full((len(wavs) * N, 256), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_mae_ast_fbank_f32((C.c_void_p * len(dev))(*[w.data_ptr() for w in dev]),
                                            (C.c_int64 * len(dev))(*lens), len(dev), L, int(kind == "patch"), rm, rv,
                                            fmt, out.data_ptr(), planes.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return out.cpu(), planes.cpu().reshape(len(wavs), N, 256)


# n_b = 1 + (L - 400) // 160: 16000 -> 99, 9000 -> 54 (a multiple of 2, not of 16), 5360 -> 32 (a multiple of 16),
# 12345 -> 75, 400 -> 1, 2800 -> 16
FRONT_LENS = [16000, 9000, 5360, 12345, 400, 2800]


@pytest.mark.parametrize("fmt", [0, 1], ids=["bf16x3", "f16q8"])
@pytest.mark.parametrize("kind", ["frame", "patch"])
def test_frontend_matches_fp64(s3b_lib, kind, fmt):
    """Every element of the unfolded, batch-normalised fbank against fp64; padded frames exactly the normalised-zero
    constant; the planes bit for bit the operand of the fp32 values; nothing written past the last patch's rows."""
    rm, rv = -7.5, 11.0
    wavs = [_structured(n, i) for i, n in enumerate(FRONT_LENS)]
    guard = 64
    out, planes = _frontend(s3b_lib, wavs, kind, rm, rv, fmt, guard)
    assert torch.isnan(out[-guard:]).all()  # past T' kt frames
    got = out[:-guard].reshape(planes.shape)
    assert torch.equal(planes, _through_planes(got, fmt))
    sd = {"batch_norm.running_mean": torch.tensor([rm]), "batch_norm.running_var": torch.tensor([rv])}
    ref = MO.frontend(wavs, sd, kind)
    assert ref.shape == got.shape
    # the padded frames: fp32(-rm * a) exactly
    kt, kc = MO.KINDS[kind]
    _, c = _bn(rm, rv)
    pad = MO.unfold(torch.stack([
        (torch.arange(ref.shape[1] // (128 // kc) * kt) >= 1 + (n - 400) // 160)[:, None].expand(-1, 128)
        for n in FRONT_LENS]).double(), kind).bool()
    assert pad.any() and (~pad).any()
    assert torch.all(got[pad] == c)
    err = (got.double() - ref).abs()
    bound = 2e-4
    print(f"mae_ast {kind} front end fmt {fmt}: max |err| {err.max().item():.2e} (measured/bound "
          f"{err.max().item() / bound:.3f}), padded elements {int(pad.sum())} at {c}")
    assert err.max().item() < bound


@pytest.mark.parametrize("scheme", [0, 1], ids=["bf16x3", "f16q8"])
@pytest.mark.parametrize("M", PROJ_ROWS)
def test_projection_matches_fp64_and_emulation(s3b_lib, M, scheme):
    """post_extract_proj (N = 768, K = 256, fp32 output + bias) as the forward runs it, against fp64 and the scheme's
    operand-split emulation."""
    g = torch.Generator(device="cuda").manual_seed(M + scheme)
    a = torch.randn(M, 256, device="cuda", generator=g) * 0.7 + 0.2
    w = torch.randn(D, 256, device="cuda", generator=g) / 16
    bias = torch.randn(D, device="cuda", generator=g) * 0.02
    out, o = _linear(a, w, bias, scheme=scheme, out_fmt=-1)
    assert o.scheme_used == scheme
    exact, emu, e1, e2 = _gemm_refs(a, w, scheme)
    ref1, b1 = _epilogue(exact, e1, bias)
    ref2, b2 = _epilogue(emu, e2, bias)
    _check(f"mae_ast post_extract_proj M={M} s{scheme}", out, ref1, b1, ref2, b2, (e1, e2), scheme)


def _embed(s3b_lib, x, valid, pe, ln=None, fmt=0):
    """s3b_mae_ast_embed_f32 on a copy of x [B, N, 768]: (x after, decoded planes or None)."""
    from s3prl_b200 import lib

    B, N, _ = x.shape
    y = x.cuda().contiguous().clone()
    planes = torch.full_like(y, float("nan")) if ln is not None else None
    g, b = (ln[0].cuda(), ln[1].cuda()) if ln is not None else (None, None)
    p = pe.cuda().contiguous() if pe is not None else None
    lib.check(s3b_lib.s3b_mae_ast_embed_f32(y.data_ptr(), B, N, (C.c_int32 * B)(*valid), _ptr(p), _ptr(g), _ptr(b), fmt,
                                            _ptr(planes), _stream()))
    torch.cuda.synchronize()
    return y.cpu(), (planes.cpu() if planes is not None else None)


@pytest.mark.parametrize("fmt", [0, 1], ids=["bf16x3", "f16q8"])
def test_positions_and_layernorm(s3b_lib, fmt):
    """Post-LN: LayerNorm(x + pe on the valid tokens) against fp64 per row, its planes bit for bit; padded tokens get
    no pe. Pre-LN: the sum alone, exactly fp32(x + pe), padded tokens untouched."""
    from s3prl_b200.upstream.mae_ast import sinusoid_table

    B, N = 4, 392
    valid = [392, 200, 8, 0]
    g = torch.Generator().manual_seed(8 + fmt)
    x = torch.randn(B, N, D, generator=g) * 1.3 + 0.1
    pe = sinusoid_table(512)[0]
    gm, bt = 1 + 0.1 * torch.randn(D, generator=g), 0.05 * torch.randn(D, generator=g)
    keep = (torch.arange(N)[None, :] < torch.tensor(valid)[:, None])[..., None]
    summed = x + pe[:N] * keep
    post, planes = _embed(s3b_lib, x, valid, pe, (gm, bt), fmt)
    ref = torch.nn.functional.layer_norm(summed.double(), (D,), gm.double(), bt.double(), 1e-5)
    err = ((post.double() - ref).abs().amax(-1) / ref.abs().amax(-1)).max().item()
    print(f"mae_ast positions + LayerNorm fmt {fmt}: max row-relative error {err:.2e} (measured/bound {err / 2e-6:.3f})")
    assert err < 2e-6
    assert torch.equal(planes, _through_planes(post, fmt))
    # padded tokens normalised without pe: the same rows of x alone
    no_pe, _ = _embed(s3b_lib, x, [0] * B, pe, (gm, bt), fmt)
    assert torch.equal(post[~keep[..., 0]], no_pe[~keep[..., 0]])
    assert not torch.equal(post[keep[..., 0]], no_pe[keep[..., 0]])
    pre, none = _embed(s3b_lib, x, valid, pe)
    assert none is None and torch.equal(pre, summed)
    assert torch.equal(pre[~keep[..., 0]], x[~keep[..., 0]])
    # without positions the kernel leaves x as it is (pre-LN, no enc_sine_pos) or normalises it (post-LN)
    assert torch.equal(_embed(s3b_lib, x, valid, None)[0], x)


def test_perturbed_pe_row_changes_that_token_only(s3b_lib):
    from s3prl_b200.upstream.mae_ast import sinusoid_table

    B, N, r = 3, 96, 37
    valid = [96, 40, 24]  # token 37 is valid in utterances 0 and 1, padded in 2
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, N, D, generator=g)
    pe = sinusoid_table(N)[0]
    pe2 = pe.clone()
    pe2[r] += 0.25
    gm, bt = torch.ones(D), torch.zeros(D)
    for ln in (None, (gm, bt)):
        a, _ = _embed(s3b_lib, x, valid, pe, ln)
        b, _ = _embed(s3b_lib, x, valid, pe2, ln)
        changed = (a != b).any(-1)
        want = torch.zeros(B, N, dtype=torch.bool)
        want[0, r] = want[1, r] = True
        assert torch.equal(changed, want), ln is None


def _attention_ref(q, k, v, valid):
    B, N, _ = q.shape
    qh, kh, vh = (t.double().view(B, N, H, HD).transpose(1, 2) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) * HD**-0.5
    mask = torch.arange(N, device=q.device)[None, :] < torch.tensor(valid, device=q.device)[:, None]
    s = s.masked_fill(~mask[:, None, None, :], float("-inf"))
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, N, D)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("N,valid", ATTN_CASES, ids=[str(n) for n, _ in ATTN_CASES])
def test_attention_at_patch_key_counts(s3b_lib, N, valid, fmt):
    """Key counts that are multiples of 8 but not of the kernel's 64-key block, as the patch model's masks give."""
    g = torch.Generator(device="cuda").manual_seed(N + fmt)
    q, k, v = (torch.randn(len(valid), N, D, device="cuda", generator=g) for _ in range(3))
    out = _attention(q, k, v, valid, H, HD, fmt)
    _check_block(out, _attention_ref(q, k, v, valid), f"mae_ast attention N={N} valid={valid} ctx_format={fmt}")


def _fabricated(kind, seed=0, **kw):
    from s3prl_b200.upstream.mae_ast import fabricate_mae_ast_state_dict

    return fabricate_mae_ast_state_dict(seed, kind, **kw)


def _expert(scheme, ckpt_dict=None, kind="frame", tmp=None, **kw):
    from s3prl_b200.upstream.mae_ast import MaeAstExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        if ckpt_dict is not None:
            path = tmp / f"mae_ast_{kind}.pt"
            torch.save(ckpt_dict, path)
            kw["ckpt"] = str(path)
        ex = MaeAstExpert(kind=kind, **kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


@pytest.mark.parametrize("scheme", ["f16q8", "bf16x3"])
@pytest.mark.parametrize("fixture", GOLDENS)
def test_matches_reference_golden(s3b_lib, tmp_path, fixture, scheme):
    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ck = _fabricated(g["kind"], g["weight_seed"], max_token_length=g["max_token_length"], **g["fabricate"])
    ex = _expert(scheme, ck, g["kind"], tmp_path)
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        hs = ex([w.cuda() for w in _wavs(case["lens"], case["wav_seed"], case["wav_scale"])])["hidden_states"]
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            _assert_close(f"{fixture} lens={case['lens']} {scheme} state {l}",
                          h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu(), case["sub"][l])


@pytest.mark.parametrize("kind", ["frame", "patch"])
def test_matches_oracle_32x10s(s3b_lib, kind):
    """32 utterances around 10 s (the frame model: 499 patches of 2 frames) against the fp64 oracle, three utterances
    each run alone at the batch's length."""
    from s3prl_b200.upstream.mae_ast import prepare_mae_ast_tensors

    ex = _expert(None, kind=kind, seed=3)
    lens = [160000 - 2011 * i for i in range(32)]
    wavs = _wavs(lens, seed=13)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    cfg, sd = prepare_mae_ast_tensors(_fabricated(kind, 3), kind)
    for b in (0, 17, 31):
        ref = _oracle_alone(wavs[b], max(lens), sd, cfg, layers=6)
        for l in (0, 5):
            _assert_close(f"32x10s {kind} utterance {b} state {l}", hs[l][b:b + 1].cpu(), ref[l])


def _oracle_alone(wav, max_len, sd, cfg, layers):
    """The oracle's hidden states of one utterance in a batch padded to max_len: its fbank frames, zero rows up to the
    batch's F (whose batch norm is the padded-frame constant), its own key mask."""
    import torch.nn.functional as F

    kind = cfg["kind"]
    kt, kc = MO.KINDS[kind]
    nv = 128 // kc
    Fm = 1 + (max_len - 400) // 160
    f = MO.fbank(wav)
    x = F.pad(f, (0, 0, 0, Fm - f.shape[0]))[None]
    a = MO.unfold(MO.normalise(x, sd), kind)
    N = a.shape[1]
    valid = MO.valid_tokens([len(wav)], kind, N // nv)
    key_valid = torch.arange(N)[None, :] < torch.tensor(valid)[:, None]
    h = MO.embed(a, sd, cfg, valid)
    out = []
    for l in range(layers):
        h = MO.layer(h, sd, l, key_valid, cfg["layer_norm_first"])
        out.append(h.reshape(1, N // nv, nv * D))
    return out


def test_long_lived_model_gives_a_fresh_models_bits(s3b_lib):
    """A model that has run other batch shapes and lane counts, next to a model of the other kind, gives the bits of a
    fresh model; lanes 1 and 2 and forward_host agree bit for bit."""
    lens = [40000, 400, 15999, 16000, 16001, 7000, 23000, 31999]
    wavs = [w.cuda() for w in _wavs(lens, seed=17)]
    fresh = torch.stack(_expert(None, kind="patch", seed=4)(wavs)["hidden_states"]).clone()
    old = _expert(None, kind="patch", seed=4)
    other = _expert(None, kind="frame", seed=4)
    for n, lanes in ((3, 1), (8, 2), (1, 0), (5, 2)):
        old.lanes = lanes
        old(wavs[:n])
        other(wavs[n - 1:])
        old([w[: max(2800, w.numel() // 3)] for w in wavs])
    old.lanes = 0
    assert torch.equal(torch.stack(old(wavs)["hidden_states"]), fresh)
    for lanes in (1, 2):
        old.lanes = lanes
        assert torch.equal(torch.stack(old(wavs)["hidden_states"]), fresh), lanes
    old.lanes = 0
    assert torch.equal(old.forward_host([w.cpu() for w in wavs]), fresh.cpu())
    old.global_max_len = max(lens)
    assert torch.equal(torch.stack(old([wavs[3]])["hidden_states"])[:, 0], fresh[:, 3])


def test_local_entry_equals_named_entry(s3b_lib, tmp_path):
    from s3prl_b200 import hub

    path = tmp_path / "frame.pt"
    torch.save(_fabricated("frame", 6, max_token_length=2048), path)
    wavs = [w.cuda() for w in _wavs([16000, 9000, 400], seed=21)]
    a = torch.stack(hub.mae_ast_local(str(path))(wavs)["hidden_states"])
    b = torch.stack(hub.mae_ast_frame(str(path))(wavs)["hidden_states"])
    assert torch.equal(a, b)


def test_forward_ex_refusals(s3b_lib, tmp_path):
    from s3prl_b200 import lib

    ex = _expert(None, kind="frame")
    wavs = [w.cuda() for w in _wavs([16000, 9001], seed=5)]
    native, ws, lens, max_len, T = ex._prepare(wavs)
    ffn = torch.empty((12, 2, T, 768), device="cuda")
    with pytest.raises(lib.S3BError, match="MAE-AST"):
        ex._forward_ex(native, ws, lens, max_len, T, ffn_out=ffn)
    # more tokens than enc_sine_pos_embed.pe has rows: refused by the expert, and by the library itself
    short = _expert(None, _fabricated("frame", 0, max_token_length=40), "frame", tmp_path)
    with pytest.raises(ValueError, match="enc_sine_pos_embed.pe"):
        short(wavs)
    native, ws, lens, max_len, T = short._prepare(wavs)
    with pytest.raises(lib.S3BError, match="enc_sine_pos_embed.pe"):
        short._forward_ex(native, ws, lens, max_len, T)
