"""GPU tests of DeCoAR 2.0 (``decoar2``): the front end (kaldi fbank with the hamming window, CMVN, y[::2], written as
operand planes) against torchaudio's own ``kaldi.fbank``, and the whole model against the executed-reference goldens
(tests/golden/decoar2_ref*.pt) and the CPU oracle (tests/decoar2_oracle.py) in both GEMM operand schemes, with
determinism across lanes, shards, a checkpoint file and ``forward_host``.
Bounds: front end 1e-4 relative per utterance; the model the golden bars of tests/test_upstream_gpu.py (2e-4 per layer,
1e-3 of the layer's abs max). Every check prints measured / bound."""
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

pytestmark = pytest.mark.gpu

FEAT_REL = 1e-4
REL_TOL = 2e-4
ABS_FRAC = 1e-3


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


def _structured(n, seed):
    """Two tones over a -60 dB noise floor, with a stretch of digital silence (exact zeros: whole frames at the log
    floor) and a silent tail."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64) / 16000
    x = 0.5 * torch.sin(2 * math.pi * 440 * t) + 0.2 * torch.sin(2 * math.pi * (2000 + 97 * seed) * t)
    x = (x + 1e-3 * torch.randn(n, generator=g, dtype=torch.float64)).float()
    x[n // 3 : n // 3 + 2400] = 0.0
    x[-700:] = 0.0
    return x


def _reference_features(wav):
    """decoar2/audio.py:69-86 with torchaudio itself: kaldi.fbank (hamming) -> CMVN -> y[::2]."""
    from torchaudio.compliance import kaldi

    y = kaldi.fbank(wav[None].float(), num_mel_bins=80, sample_frequency=16000, window_type="hamming")
    y = (y - y.mean(0, keepdim=True)) / (1e-10 + y.std(0, keepdim=True))
    return y[::2]


def _features(wavs, out_fmt):
    from s3prl_b200 import lib

    lens = [len(w) for w in wavs]
    from s3prl_b200.upstream.decoar2 import num_frames

    T = num_frames(max(lens))
    dev = [w.cuda() for w in wavs]
    out = torch.full((len(wavs), T, 80), float("nan"), device="cuda")
    ptrs = (C.c_void_p * len(wavs))(*[w.data_ptr() for w in dev])
    lib.check(lib.load().s3b_decoar2_features_f32(ptrs, (C.c_int64 * len(lens))(*lens), len(lens), out_fmt,
                                                  C.c_void_p(out.data_ptr()),
                                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("out_fmt", [0, 1])
@pytest.mark.parametrize("kind", ["random", "structured"])
def test_features_match_torchaudio(s3b_lib, kind, out_fmt):
    lens = [16000, 12345, 800, 560, 160000]
    wavs = _wavs(lens, seed=3) if kind == "random" else [_structured(n, i) for i, n in enumerate(lens)]
    out = _features(wavs, out_fmt)
    worst = 0.0
    for b, w in enumerate(wavs):
        ref = _reference_features(w)
        tb = len(ref)
        got = out[b, :tb]
        assert torch.isfinite(got).all()
        assert torch.equal(out[b, tb:], torch.zeros_like(out[b, tb:])), b  # pad_sequence rows
        worst = max(worst, _rel(got, ref))
    print(f"decoar2 features {kind} out_fmt={out_fmt}: worst relative error {worst:.3e} "
          f"(measured/bound {worst / FEAT_REL:.3f})")
    assert worst < FEAT_REL


def test_features_refusals(s3b_lib):
    from s3prl_b200 import lib

    w = torch.zeros(559, device="cuda")
    out = torch.empty(1, 1, 80, device="cuda")
    r = lib.load().s3b_decoar2_features_f32((C.c_void_p * 1)(w.data_ptr()), (C.c_int64 * 1)(559), 1, 0,
                                            C.c_void_p(out.data_ptr()), None)
    assert r != 0 and b"560" in lib.load().s3b_last_error()


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
_EXPERT = {}


def _expert(scheme):
    from s3prl_b200.upstream.decoar2 import Decoar2Expert

    if scheme not in _EXPERT:
        _EXPERT.clear()
        saved = os.environ.get("S3B_GEMM_SCHEME")
        if scheme is not None:
            os.environ["S3B_GEMM_SCHEME"] = scheme
        try:
            ex = Decoar2Expert().to("cuda")
            ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
            _EXPERT[scheme] = ex
        finally:
            if scheme is not None:
                if saved is None:
                    os.environ.pop("S3B_GEMM_SCHEME", None)
                else:
                    os.environ["S3B_GEMM_SCHEME"] = saved
    return _EXPERT[scheme]


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("fixture", ["decoar2_ref", "decoar2_ref_c2"])
def test_matches_reference_golden(s3b_lib, fixture, scheme):
    fx = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ex = _expert(scheme)
    cs, ts = fx["channel_stride"], fx["time_stride"]
    worst = 0.0
    for case in fx["cases"]:
        res = ex([w.cuda() for w in _wavs(case["lens"], case["wav_seed"])])
        hs = res["hidden_states"]
        assert list(res["_hidden_states_info"]) == case["names"]
        assert res["last_hidden_state"] is hs[-1] and res["hidden_state_12"] is hs[12]
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
    print(f"{fixture} scheme={scheme or 'default'}: worst per-layer relative error vs reference golden {worst:.3e} "
          f"(measured/bound {worst / REL_TOL:.3f})")


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("lens", [[40000, 33333, 900], [16000, 561, 7777, 16000]])
def test_matches_oracle_ragged(s3b_lib, lens, scheme):
    import decoar2_oracle as D

    from s3prl_b200.upstream.decoar2 import fabricate_decoar2_state_dict

    ex = _expert(scheme)
    wavs = _wavs(lens, seed=1234)
    with torch.no_grad():
        ref, _pad = D.decoar2_forward(wavs, fabricate_decoar2_state_dict(0))
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    worst = 0.0
    for l, (h, r) in enumerate(zip(hs, ref)):
        h = h.cpu()
        assert h.shape == r.shape and torch.isfinite(h).all(), l
        rel = _rel(h, r)
        assert rel < REL_TOL, (l, rel)
        assert (h.double() - r.double()).abs().max().item() < ABS_FRAC * r.abs().max().item(), l
        worst = max(worst, rel)
    print(f"decoar2 scheme={scheme or 'default'} lens={lens}: worst per-layer relative error vs oracle {worst:.3e} "
          f"(measured/bound {worst / REL_TOL:.3f})")


def test_lanes_shards_file_and_host_path_are_bit_identical(s3b_lib, tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.decoar2 import fabricate_decoar2_state_dict

    ex = _expert(None)
    lens = [48000, 40000, 33333, 900]
    host = _wavs(lens, seed=99)
    wavs = [w.cuda() for w in host]
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
    assert torch.equal(ex.forward_host(host).cuda(), one)
    out, dev = ex.forward_host(host, keep_device=True)
    assert torch.equal(dev, one) and torch.equal(out.cuda(), one)
    path = tmp_path / "decoar2.pt"
    torch.save({"model": fabricate_decoar2_state_dict(0)}, path)
    local = hub.ENTRIES["decoar2_local"](str(path)).to("cuda")
    assert torch.equal(torch.stack(local(wavs)["hidden_states"]), one)
    named = hub.ENTRIES["decoar2"]().to("cuda")
    assert torch.equal(torch.stack(named(wavs)["hidden_states"]), one)


def test_ffn_out_and_profile(s3b_lib):
    """ffn_out (fc2 output before the residual) is filled for the post-LN encoder, and the profile counts the fbank
    front end under category 2 with no conv-stack GEMMs."""
    from s3prl_b200 import lib

    ex = _expert(None)
    wavs = [w.cuda() for w in _wavs([16000, 9000], seed=5)]
    native = ex._native
    B, T, D, NL = 2, ex.num_frames(16000), 768, 12
    hs = torch.empty(NL + 1, B, T, D, device="cuda")
    ffn = torch.full((NL, B, T, D), float("nan"), device="cuda")
    opts = lib.S3BForwardOpts(lanes=1)
    opts.ffn_out = ffn.data_ptr()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptrs = (C.c_void_p * B)(*[w.data_ptr() for w in wavs])
    lens = (C.c_int64 * B)(16000, 9000)
    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    try:
        lib.check(native.lib.s3b_forward_ex(native.handle, ptrs, lens, B, 16000, C.c_void_p(hs.data_ptr()), st,
                                            C.byref(opts)))
        ms, fl, n = (C.c_double * 5)(), (C.c_double * 5)(), (C.c_int64 * 5)()
        lib.check(native.lib.s3b_profile_read(native.handle, ms, fl, n, 1))
    finally:
        native.lib.s3b_profile_enable(native.handle, 0)
    assert torch.isfinite(ffn).all() and ffn.abs().max() > 0
    assert torch.equal(hs, torch.stack(ex(wavs)["hidden_states"]))
    assert n[2] == 2 and ms[2] > 0, list(n)  # the fbank frame kernel and the CMVN kernel
    assert n[0] == 1 + 1 + 4 * NL, list(n)  # post_extract_proj, pos_conv, four GEMMs per layer
    print(f"decoar2 profile ms: gemm {ms[0]:.3f} attention {ms[1]:.3f} front end {ms[2]:.3f} norm {ms[3]:.3f} "
          f"misc {ms[4]:.3f}")


def test_repeated_calls_are_bit_identical(s3b_lib):
    """10 identical calls after a first one give its result bit for bit and each adds the same launch count."""
    from s3prl_b200.upstream.decoar2 import Decoar2Expert

    g = torch.Generator().manual_seed(5)
    wavs = [torch.randn(n, generator=g).cuda() for n in (24000, 16000, 9000, 20000)]
    e = Decoar2Expert().to("cuda")
    ref = torch.stack(e(wavs)["hidden_states"]).clone()
    native = e._native
    counts = []
    for i in range(10):
        c0 = native.lib.s3b_launch_count(native.handle)
        res = e(wavs)
        counts.append(native.lib.s3b_launch_count(native.handle) - c0)
        assert torch.equal(torch.stack(res["hidden_states"]), ref), f"call {i + 1} changed the result"
    assert len(set(counts)) == 1, counts
