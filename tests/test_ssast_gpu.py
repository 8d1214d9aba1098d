"""SSAST on the GPU: the 128-bin hanning fbank, the patch operand, the patch GEMM with the token assembly, LayerNorm at
eps 1e-6 and the output fold against fp64 per element; whole forwards of both models against the executed reference's
goldens and the fp64 oracle in both operand schemes (ragged, window-boundary and 32 x 10 s batches); and a long-lived
model that gives the bits of a fresh one after calls of other shapes, windows and lane counts."""
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

import ssast_oracle as SO  # noqa: E402

pytestmark = pytest.mark.gpu

REL_TOL = 2e-4  # relative Frobenius error per hidden state, as tests/test_upstream_gpu.py
ELEM_TOL = 1e-3  # per element, relative to the state's absolute maximum
GOLDENS = ("ssast_frame", "ssast_patch", "ssast_frame_w10", "ssast_patch_w10")


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _wavs(lens, seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) * scale for n in lens]


def _structured(n, seed):
    """Noise under a chirp, with a loud step and a silent stretch: the frames across a window edge see all three."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64) / 16000
    x = 0.05 * torch.randn(n, generator=g, dtype=torch.float64) + 0.3 * torch.sin(2 * math.pi * (200 + 900 * t) * t)
    x[n // 3: n // 3 + 2000] *= 8.0
    x[2 * n // 3: 2 * n // 3 + 1200] = 0.0
    return x.float()


@pytest.mark.parametrize("S", [16000, 4000])
def test_fbank_matches_fp64(s3b_lib, S):
    from s3prl_b200 import lib

    lens = [40000, 16000, 1, 23457, 15999]
    wavs = [_structured(n, i) for i, n in enumerate(lens)]
    L = max(lens)
    nseg, TL = -(-L // S), S // 160
    dev = [w.cuda() for w in wavs]
    out = torch.full((len(lens) * nseg, TL, 128), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_ssast_fbank_f32((C.c_void_p * len(lens))(*[w.data_ptr() for w in dev]),
                                          (C.c_int64 * len(lens))(*lens), len(lens), L, S, out.data_ptr(), _stream()))
    ref = SO.fbank_windows(wavs, S, L)
    got = out.cpu().double()
    m = 1 + (S - 400) // 160
    assert torch.all(got[:, m:] == 0)  # the appended rows
    floor = (math.log(SO.FLOOR) + 4.2677393) / (4.5689974 * 2)
    silent = ref[:, :m].eq(floor).all(-1).all(-1)
    assert silent.sum() >= 4  # the windows past the 1-sample and 15999-sample utterances' ends
    assert (got[silent][:, :m] - floor).abs().max().item() < 1e-6
    err = (got[:, :m] - ref[:, :m]).abs().max().item()
    print(f"ssast fbank S={S}: max |err| {err:.2e} (normalised units, bound 1e-4)")
    assert err < 1e-4


def _planes_tol(scheme):
    # relative representation error of one operand element: bf16 hi + lo keeps 16 bits; f16q8 is held to its fp16
    # plane's half ulp (the e4m3 correction only shrinks it), and its gather is checked bit for bit below
    return 2.0 ** -11 if scheme == 1 else 2.0 ** -16


def _embed(s3b_lib, kind, feat, sd, scheme):
    """s3b_ssast_embed_f32 on [SB, TL, 128] features: (decoded operand planes, [SB, 2 + P, 768] output)."""
    from s3prl_b200 import lib

    SB, tl = feat.shape[0], feat.shape[1]
    P = sd["pos_embed"].shape[1] - 2
    d = {k: v.cuda().contiguous() for k, v in sd.items() if "blocks" not in k}
    fd = feat.cuda()
    shape = (SB, tl, 128) if kind == "frame" else (SB, P, 256)
    planes = torch.full(shape, float("nan"), device="cuda")
    out = torch.full((SB, 2 + P, 768), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_ssast_embed_f32(fd.data_ptr(), SB, tl, int(kind == "patch"), d["patch_embed.proj.weight"].data_ptr(),
                                          d["patch_embed.proj.bias"].data_ptr(), d["cls_token"].data_ptr(),
                                          d["dist_token"].data_ptr(), d["pos_embed"].data_ptr(), scheme,
                                          planes.data_ptr(), out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return planes.cpu(), out


@pytest.mark.parametrize("scheme", [1, 0], ids=["f16q8", "bf16x3"])
@pytest.mark.parametrize("kind,tl", [("frame", 100), ("patch", 100), ("frame", 1000), ("patch", 1000)])
def test_patch_embed_and_tokens(s3b_lib, kind, tl, scheme):
    """The patch operand (frame rows / the 16 x 16 stride-10 gather) against fp64 within its representation error, and
    the gather bit for bit against the frame operand's elements; the (768, 256) patch GEMM against fp64 on the decoded
    operand; the class rows exactly fp32(token + pos)."""
    from s3prl_b200.upstream.ssast import fabricate_ssast_state_dict, prepare_ssast_tensors

    sd = prepare_ssast_tensors(fabricate_ssast_state_dict(5, kind), kind, tl / 100)
    SB = 3
    g = torch.Generator().manual_seed(tl + scheme)
    feat = (torch.randn(SB, tl, 128, generator=g) * 0.4 - 0.2)
    feat[:, -2:] = 0  # the appended rows
    A = SO.patch_operand(feat.double(), kind)
    planes, out = _embed(s3b_lib, kind, feat, sd, scheme)
    pl = planes.double()
    rep = ((pl - A).abs() / (_planes_tol(scheme) * A.abs() + 1e-7)).max().item()
    print(f"ssast {kind} tl={tl} scheme {scheme}: operand planes measured/bound {rep:.3f}")
    assert rep <= 1.0
    if kind == "patch":
        frame_sd = prepare_ssast_tensors(fabricate_ssast_state_dict(5, "frame"), "frame", tl / 100)
        frame_planes, _ = _embed(s3b_lib, "frame", feat, frame_sd, scheme)
        assert torch.equal(planes, SO.patch_operand(frame_planes, "patch").float())
    got = out.cpu().double()
    # fp64 of the same contraction on the decoded operand: the GEMM's own error (weight planes and fp32 sums)
    w = sd["patch_embed.proj.weight"].double().reshape(768, -1)
    if kind == "frame":
        rows = torch.cat([pl[:, :-1], pl[:, 1:]], dim=-1)  # [SB, TL - 1, 256]: frames t, t + 1
        wk = sd["patch_embed.proj.weight"].double()[:, 0].permute(0, 2, 1).reshape(768, 256)  # column dt * 128 + f
        y = rows @ wk.T
    else:
        y = pl @ w.T
    y = y + sd["patch_embed.proj.bias"].double()
    bound = (rows.abs() @ wk.abs().T if kind == "frame" else pl.abs() @ w.abs().T) * 1.5e-4 + 1e-7
    pos = sd["pos_embed"].double()[0]
    assert ((got[:, 2:] - (y + pos[2:])).abs() <= bound + 2e-7 * (y + pos[2:]).abs()).all()
    cls = (sd["cls_token"][0, 0] + sd["pos_embed"][0, 0]).expand(SB, -1)
    dist = (sd["dist_token"][0, 0] + sd["pos_embed"][0, 1]).expand(SB, -1)
    assert torch.equal(out[:, 0].cpu(), cls) and torch.equal(out[:, 1].cpu(), dist)
    # and the whole embedding against fp64 on the fp32 features (operand rounding included)
    full = SO.embed(feat.double(), sd)
    print(f"ssast {kind} tl={tl} scheme {scheme}: embedding vs fp64 {_rel(got, full):.2e}")
    assert _rel(got, full) < 1e-4


def test_layernorm_eps_1e6(s3b_lib):
    from s3prl_b200 import lib

    M, D = 2000, 768
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(M, D, device="cuda", generator=g) * 3 + 5
    x[:500] = 1e-3 * torch.randn(500, D, device="cuda", generator=g)  # variance ~ eps: eps decides the scale
    gm = 1 + 0.3 * torch.randn(D, device="cuda", generator=g)
    bt = 0.3 * torch.randn(D, device="cuda", generator=g)
    out = torch.empty_like(x)
    lib.check(s3b_lib.s3b_layernorm_eps_f32(x.data_ptr(), M, D, gm.data_ptr(), bt.data_ptr(), 0, 1e-6, out.data_ptr(),
                                            _stream()))
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x.double(), (D,), gm.double(), bt.double(), 1e-6)
    other = torch.nn.functional.layer_norm(x.double(), (D,), gm.double(), bt.double(), 1e-5)
    err = ((out.double() - ref).abs().amax(-1) / ref.abs().amax(-1)).max().item()
    print(f"layernorm eps 1e-6: max row-relative error {err:.2e}")
    assert err < 2e-6
    assert _rel(out[:500], other[:500]) > 1e-2  # the small-variance rows tell the two eps apart


@pytest.mark.parametrize("kind,tl,nseg,T", [("frame", 100, 3, 250), ("frame", 100, 2, 198), ("patch", 100, 3, 25),
                                            ("patch", 1000, 2, 107)])
def test_fold_layout(s3b_lib, kind, tl, nseg, T):
    from s3prl_b200 import lib

    B, f_dim = 2, (12 if kind == "patch" else 1)
    tdim = tl - 1 if kind == "frame" else (tl - 16) // 10 + 1
    x = torch.randn(B * nseg, 2 + f_dim * tdim, 768, device="cuda")
    out = torch.full((B, T, f_dim * 768), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_ssast_fold_f32(x.data_ptr(), B, nseg, tl, int(kind == "patch"), T, out.data_ptr(), _stream()))
    assert torch.equal(out.cpu(), SO.fold(x.cpu(), B, f_dim, T))


def _expert(scheme, **kw):
    from s3prl_b200.upstream.ssast import SsastExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        ex = SsastExpert(**kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


def _assert_close(what, h, ref):
    err = _rel(h, ref)
    el = ((h.double() - ref.double()).abs().max() / ref.double().abs().max()).item()
    print(f"{what}: abs max {ref.abs().max().item():.3f}, relative error {err:.3e} (measured/bound "
          f"{err / REL_TOL:.3f}), element {el:.3e} (measured/bound {el / ELEM_TOL:.3f})")
    assert err < REL_TOL and el < ELEM_TOL, what


@pytest.mark.parametrize("scheme", ["f16q8", "bf16x3"])
@pytest.mark.parametrize("fixture", GOLDENS)
def test_matches_reference_golden(s3b_lib, fixture, scheme):
    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ex = _expert(scheme, kind=g["kind"], window_secs=g["window_secs"], seed=g["weight_seed"])
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        hs = ex([w.cuda() for w in _wavs(case["lens"], case["wav_seed"], case["wav_scale"])])["hidden_states"]
        assert len(hs) == case["num_hidden"] == 12 and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            _assert_close(f"{fixture} lens={case['lens']} {scheme} state {l}",
                          h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu(), case["sub"][l])


@pytest.mark.parametrize("scheme", ["f16q8", "bf16x3"])
@pytest.mark.parametrize("kind", ["frame", "patch"])
def test_matches_oracle_ragged(s3b_lib, kind, scheme):
    """Every element of every hidden state against the fp64 oracle: a 1-sample utterance, the window-boundary
    lengths, an utterance that ends windows before the longest."""
    from s3prl_b200.upstream.ssast import fabricate_ssast_state_dict, prepare_ssast_tensors

    ex = _expert(scheme, kind=kind, seed=2)
    lens = [40000, 1, 15999, 16000, 16001, 7000]
    wavs = _wavs(lens, seed=11)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    ref = SO.ssast_forward(wavs, prepare_ssast_tensors(fabricate_ssast_state_dict(2, kind), kind, 1.0), kind, 1.0)
    for l, (h, r) in enumerate(zip(hs, ref)):
        _assert_close(f"ragged {kind} {scheme} state {l}", h.cpu(), r)


@pytest.mark.parametrize("kind", ["frame", "patch"])
def test_matches_oracle_32x10s(s3b_lib, kind):
    """32 x 10 s in 10 s windows (the speaker-identification setting), three utterances checked against the oracle,
    each run alone in fp64 at the batch's max_len (utterances are independent given it)."""
    from s3prl_b200.upstream.ssast import fabricate_ssast_state_dict, prepare_ssast_tensors

    ex = _expert(None, kind=kind, window_secs=10.0, seed=3)
    lens = [160000 - 997 * i for i in range(32)]
    wavs = _wavs(lens, seed=13)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    sd = prepare_ssast_tensors(fabricate_ssast_state_dict(3, kind), kind, 10.0)
    for b in (0, 17, 31):
        ref = SO.ssast_forward([wavs[b]], sd, kind, 10.0, max_len=max(lens))
        for l in (0, 5, 11):
            _assert_close(f"32x10s {kind} utterance {b} state {l}", hs[l][b:b + 1].cpu(), ref[l])


def test_long_lived_model_gives_a_fresh_models_bits(s3b_lib):
    """A model that has run other batch shapes and lane counts, next to a model of another window, gives the bits of a
    fresh model; lanes 1 and 2 and forward_host agree bit for bit."""
    lens = [40000, 1, 15999, 16000, 16001, 7000, 23000, 31999]
    wavs = [w.cuda() for w in _wavs(lens, seed=17)]
    fresh = torch.stack(_expert(None, kind="patch", seed=4)(wavs)["hidden_states"]).clone()
    old = _expert(None, kind="patch", seed=4)
    other = _expert(None, kind="patch", seed=4, window_secs=2.5)
    for n, lanes in ((3, 1), (8, 2), (1, 0), (5, 2)):
        old.lanes = lanes
        old(wavs[:n])
        other(wavs[n - 1:])
        old([w[: max(1, w.numel() // 3)] for w in wavs])
    old.lanes = 0
    assert torch.equal(torch.stack(old(wavs)["hidden_states"]), fresh)
    for lanes in (1, 2):
        old.lanes = lanes
        assert torch.equal(torch.stack(old(wavs)["hidden_states"]), fresh), lanes
    old.lanes = 0
    assert torch.equal(old.forward_host([w.cpu() for w in wavs]), fresh.cpu())
    # an utterance alone at the batch's max_len gives its rows of the batch
    old.global_max_len = max(lens)
    assert torch.equal(torch.stack(old([wavs[3]])["hidden_states"])[:, 0], fresh[:, 3])


def test_forward_ex_refuses_layer_results(s3b_lib):
    from s3prl_b200 import lib

    ex = _expert(None, kind="frame")
    wavs = [w.cuda() for w in _wavs([16000, 9001], seed=5)]
    native, ws, lens, max_len, T = ex._prepare(wavs)
    ffn = torch.empty((12, 2, T, 768), device="cuda")
    with pytest.raises(lib.S3BError, match="SSAST"):
        ex._forward_ex(native, ws, lens, max_len, T, ffn_out=ffn)
