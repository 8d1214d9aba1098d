"""Spectral baselines on the GPU against the fp64 restatement (tests/spectral_ref.py), on structured audio.

Each kernel stage is held to a per-element bound derived from the inputs (module docstring of spectral_ref):
  fbank_frames  : log-mel inside [lo, hi] (FFT bound per frame -> power -> mel sum -> log, floor either side)
  delta         : |D - D64| <= dD, |DD - DD64| <= dDD (5-tap propagation of the log-mel bound)
  cmvn          : |z - z64| <= dz on columns with s >= 10 max df; elsewhere |z| <= sqrt(m - 1) (the kernel
                  normalises the same fp32 residues it squares, so Cauchy-Schwarz holds whatever the rounding),
                  fp64-constant columns give exact zeros, padding rows are exact zeros, NaN exactly where fp64 has NaN
  stft_mel      : log features of every padded frame inside [lo, hi] with the DFT held to FFT-class accuracy
  mel_cmvn      : as cmvn, over feats_len frames, then the kept / zero rows
  trimmed_len   : exact, torch `nonzero` rule (-0.0 is zero)
The worst measured/bound per stage and input kind is printed (pytest -s). For the logs it is split: "logmel" / "log"
over energies the bound resolves (E - dE above the floor), "*_edge" over the rest, where the interval reaches down to
the floor and a value sitting on the floor reads as a ratio just under 1."""
import ctypes as C
import math
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import spectral_ref as R  # noqa: E402

from s3prl_b200 import lib as L  # noqa: E402

U = R.U


def _ptrs(wavs):
    return (C.c_void_p * len(wavs))(*[w.data_ptr() for w in wavs])


def fbank_ex(lib, wavs, cmvn, stream=None):
    """s3b_fbank_ex into a NaN-filled buffer (so rows the call must zero are seen to be written)."""
    lens = [len(w) for w in wavs]
    m = lib.s3b_fbank_num_frames(max(lens))
    st = stream if stream is not None else torch.cuda.current_stream()
    with torch.cuda.stream(st):  # allocated and filled in the order of the stream the call runs on
        out = torch.full((len(wavs), m, 240), float("nan"), device="cuda")
    opts = L.S3BSpectralOpts(cmvn=cmvn)
    L.check(lib.s3b_fbank_ex(_ptrs(wavs), (C.c_int64 * len(wavs))(*lens), len(wavs), C.byref(opts),
                             C.c_void_p(out.data_ptr()), C.c_void_p(st.cuda_stream)))
    return out


def mel_plan(lib, wavs):
    """(trimmed, padded_len, feats_len, final_len, t_out): s3b_trimmed_lengths, then SpectrogramExpert's host plan."""
    from s3prl_b200.upstream.baseline import SpectrogramExpert

    B = len(wavs)
    lens = [len(w) for w in wavs]
    torch.cuda.synchronize()
    trimmed = (C.c_int64 * B)()
    L.check(lib.s3b_trimmed_lengths(_ptrs(wavs), (C.c_int64 * B)(*lens), B, trimmed))
    return (list(trimmed), *SpectrogramExpert.plan_lengths(lens, list(trimmed)))


def melspec_ex(lib, wavs, feat, cmvn, stream=None, plan=None):
    """(output, plan) of s3b_melspec_ex into a NaN-filled buffer."""
    B = len(wavs)
    plan = plan or mel_plan(lib, wavs)
    trimmed, lp, feats_len, final_len, t_out = plan
    dim = 80 if feat == "mel" else 201
    rows = t_out if cmvn else 1 + lp // 160
    st = stream if stream is not None else torch.cuda.current_stream()
    with torch.cuda.stream(st):
        out = torch.full((B, rows, dim), float("nan"), device="cuda")
    opts = L.S3BSpectralOpts(cmvn=cmvn)
    L.check(lib.s3b_melspec_ex(_ptrs(wavs), (C.c_int64 * B)(*trimmed), B, lp, int(feat == "mel"),
                               (C.c_int32 * B)(*feats_len), (C.c_int32 * B)(*final_len), t_out, C.byref(opts),
                               C.c_void_p(out.data_ptr()), C.c_void_p(st.cuda_stream)))
    return out, plan


class Worst:
    """Worst measured/bound per (stage, input kind), printed at the end of a test."""

    def __init__(self, title):
        self.title, self.v = title, {}

    def add(self, stage, kind, ratio):
        r = ratio.max().item() if ratio.numel() else 0.0
        self.v[(stage, kind)] = max(self.v.get((stage, kind), 0.0), r)

    def report(self):
        print(f"\n{self.title}: worst measured/bound")
        for (stage, kind), r in sorted(self.v.items()):
            print(f"  {stage:11s} {kind:18s} {r:.3f}")
        bad = {k: v for k, v in self.v.items() if not v <= 1.0}
        assert not bad, bad


def check_cmvn(z, s, m, kind, worst, stage="cmvn"):
    """z: the kernel's CMVN'd [m, n] rows (fp64 copy); s: the fp64 bounds (z, dz, cond) of the same columns."""
    z64, dz, cond = s
    assert torch.equal(torch.isnan(z), torch.isnan(z64)), f"{kind}: NaN pattern differs from fp64"
    if m < 2:
        return
    worst.add(stage, kind, ((z - z64).abs() / dz)[:, cond])
    assert (z.abs() <= math.sqrt(m - 1) * (1 + 1e-5)).all(), f"{kind}: |z| above sqrt(m - 1)"
    samuelson = (m - 1) / math.sqrt(m) * (1 + 1e-5)
    assert (z[:, cond].abs() <= samuelson + dz[:, cond]).all()
    const = (z64 == 0).all(dim=0) & torch.isfinite(z64).all(dim=0)
    assert torch.count_nonzero(z[:, const]) == 0, f"{kind}: a constant column is not exactly zero"


# ---- fbank ------------------------------------------------------------------------------------------------------------
FBANK_BATCH = [("chirp", 16000), ("pink", 16001), ("brown", 16000), ("bursts", 16000), ("dc", 880),
               ("tone_fbank_bin", 720), ("tone_fbank_half", 560), ("tone_25", 401), ("tone_7990", 4000),
               ("impulses", 3999), ("int16", 6000), ("tiny", 6000), ("zeros", 2000), ("white", 400), ("pink", 399)]


def _fbank_check(lib, wavs, kinds, worst):
    raw = fbank_ex(lib, [w.cuda() for w in wavs], 0).double().cpu()
    z = fbank_ex(lib, [w.cuda() for w in wavs], 1).double().cpu()
    eps_w = R.bank_eps("kaldi")
    for b, (w, kind) in enumerate(zip(wavs, kinds)):
        m = R.num_frames(len(w))
        assert torch.count_nonzero(raw[b, m:]) == 0 and torch.count_nonzero(z[b, m:]) == 0, f"{kind}: padding rows"
        if m == 0:
            continue
        s = R.fbank_bounds(w, eps_w)
        g = raw[b, :m]
        ratio, resolved = R.interval_ratio(g[:, :80], s["f"], s["lo"], s["hi"]), s["E"] - s["dE"] > R.FLOOR
        worst.add("logmel", kind, ratio[resolved])
        worst.add("logmel_edge", kind, ratio[~resolved])
        worst.add("delta", kind, (g[:, 80:160] - s["D"]).abs() / s["dF"][:, 80:160])
        worst.add("delta2", kind, (g[:, 160:] - s["DD"]).abs() / s["dF"][:, 160:])
        check_cmvn(z[b, :m], (s["z"], s["dz"], s["cond"]), m, kind, worst)
        if kind == "zeros":
            assert torch.count_nonzero(z[b, :m]) == 0
        # the no-CMVN output with CMVN applied in fp64 is the CMVN output, up to CMVN's own rounding
        if m > 1:
            zg, dzg, cg = R.cmvn_bound(g, 2 * U * g.abs())
            worst.add("cmvn_of_raw", kind, ((z[b, :m] - zg).abs() / dzg)[:, cg])
    return raw, z


@pytest.mark.gpu
def test_fbank_stages_against_fp64(s3b_lib):
    worst = Worst("fbank vs fp64")
    kinds = [k for k, _ in FBANK_BATCH]
    wavs = [R.structured_wav(k, n, seed=i) for i, (k, n) in enumerate(FBANK_BATCH)]
    raw, z = _fbank_check(s3b_lib, wavs, kinds, worst)
    b400 = kinds.index("white")  # m = 1: CMVN's std is NaN, as in fp64
    assert torch.isnan(z[b400, 0]).all() and not torch.isnan(raw[b400, 0]).any()
    # 10 s, and the same signal at other scales in one batch
    long = [R.structured_wav("chirp", 160000), R.structured_wav("brown", 160000, seed=3)]
    _fbank_check(s3b_lib, long, ["chirp_10s", "brown_10s"], worst)
    worst.report()


@pytest.mark.gpu
def test_fbank_many_short_utterances(s3b_lib):
    """64 utterances of 1..4 frames plus one of 6: grid.y = 65, the delta replicate edges at every m."""
    worst = Worst("fbank, 65 short utterances")
    kinds = ["chirp", "pink", "tone_fbank_half", "impulses", "brown", "dc", "int16", "bursts"]
    lens = [400, 401, 559, 560, 720, 880, 881, 1039]
    wavs, names = [], []
    for i in range(64):
        k = kinds[i % len(kinds)]
        wavs.append(R.structured_wav(k, lens[(i // len(kinds)) % len(lens)], seed=i))
        names.append(f"{k}_m{R.num_frames(len(wavs[-1]))}")
    wavs.append(R.structured_wav("white", 1200, seed=99))
    names.append("white_m6")
    _fbank_check(s3b_lib, wavs, names, worst)
    worst.report()


@pytest.mark.gpu
def test_fbank_no_cmvn_hub_entry(s3b_lib):
    from s3prl_b200 import hub

    assert not hub.fbank_no_cmvn(cmvn=True).cmvn  # the entry is CMVN-free whatever the caller passes
    wavs = [R.structured_wav("chirp", 16000).cuda(), R.structured_wav("pink", 9000).cuda()]
    got = hub.fbank_no_cmvn().to("cuda")(wavs)["hidden_states"][0]
    assert torch.equal(got, fbank_ex(s3b_lib, wavs, 0))
    assert torch.equal(hub.fbank().to("cuda")(wavs)["hidden_states"][0], fbank_ex(s3b_lib, wavs, 1))


# ---- mel / linear -----------------------------------------------------------------------------------------------------
def _stft_batches():
    """(name, waveforms): Lp % 160 in {0, 1, 159}, Lp = 201, the first utterance shorter / longer than the rest,
    trimmed lengths that differ from the original (trailing 0.0 / -0.0, only the first sample non-zero)."""
    w = R.structured_wav
    t = R.with_tail
    return [
        ("lp_mod0", [w("chirp", 16000), w("pink", 12345), t(w("tone_stft_bin", 8000), "zeros"), w("impulses", 3000)]),
        ("lp_mod1", [w("brown", 9000), t(w("tone_stft_half", 16001), "negzeros"), w("dc", 4000), w("zeros", 2000)]),
        ("lp_mod159", [w("tone_7990", 15999), w("bursts", 15000), w("int16", 7000), w("tiny", 5000)]),
        ("lp_201", [w("chirp", 201), w("pink", 150), w("tone_25", 201)]),
        ("first_longer", [t(w("pink", 20000), "zeros"), w("chirp", 16000), t(w("brown", 6000), "first_only")]),
        ("first_shorter", [w("tone_stft_half", 3000), t(w("chirp", 16000), "negzeros"), w("white", 11111)]),
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["mel", "linear"])
def test_stft_stages_against_fp64(s3b_lib, feat):
    from s3prl_b200 import hub

    worst = Worst(f"{feat} vs fp64")
    eps_w = R.bank_eps("htk")
    expert = getattr(hub, feat)().to("cuda")
    for name, wavs in _stft_batches():
        dev = [x.cuda() for x in wavs]
        raw, plan = melspec_ex(s3b_lib, dev, feat, 0)
        trimmed, lp, feats_len, final_len, t_out = plan
        assert trimmed == [R.trimmed_length(x) for x in wavs]
        s = R.stft_bounds(wavs, feat, eps_w)
        assert (lp, feats_len) == (s["lp"], s["feats_len"]) and raw.shape[1] == s["n_frames"]
        raw = raw.double().cpu()
        ratio, resolved = R.interval_ratio(raw, s["f"], s["lo"], s["hi"]), s["E"] - s["dE"] > 0
        worst.add("log", name, ratio[resolved])
        worst.add("log_edge", name, ratio[~resolved])
        z = expert(dev)["hidden_states"][0].double().cpu()
        ref = R.spectrogram_forward(wavs, feat)
        assert z.shape == ref.shape == (len(wavs), t_out, raw.shape[-1])
        for b in range(len(wavs)):
            n, keep = feats_len[b], min(final_len[b], feats_len[b])
            assert torch.count_nonzero(z[b, keep:]) == 0, f"{name}[{b}]: rows past the kept length"
            if n == 0 or keep == 0:
                continue
            zb, dz, cond = R.cmvn_bound(s["f"][b, :n], s["df"][b, :n])
            check_cmvn(z[b, :keep], (zb[:keep], dz[:keep], cond), n if n > 1 else 1, f"{name}[{b}]", worst, "mel_cmvn")
    worst.report()


@pytest.mark.gpu
def test_trimmed_lengths_follow_nonzero(s3b_lib):
    base = R.structured_wav("pink", 5000)
    cases = [R.with_tail(base, t) for t in ("none", "zeros", "negzeros", "first_only")]
    cases += [torch.zeros(777), torch.full((300,), -0.0), torch.tensor([0.0, -0.0, 1e-38, -0.0]), base[:1]]
    x = base.clone()
    x[:-1] = 0.0
    cases.append(x)
    dev = [c.cuda() for c in cases]
    out = (C.c_int64 * len(cases))()
    L.check(s3b_lib.s3b_trimmed_lengths(_ptrs(dev), (C.c_int64 * len(cases))(*[len(c) for c in cases]), len(cases), out))
    assert list(out) == [R.trimmed_length(c) for c in cases]


# ---- calls on two streams ------------------------------------------------------------------------------------------
# Each call stages its waveform pointers and lengths, and melspec its pre-CMVN features, in device blocks of its own,
# allocated and freed in the order of the call's stream (StreamBuf in model.cu). A call queued on one stream therefore
# reads nothing a call on another stream writes.
def _two_stream_inputs(s3b_lib, n_utts, seconds):
    lens = [16000 * seconds - 997 * i for i in range(n_utts)]
    wa = [R.structured_wav("chirp", n).cuda() for n in lens]
    wb = [R.structured_wav("pink", n, seed=5).cuda() for n in lens]
    plan_a, plan_b = mel_plan(s3b_lib, wa), mel_plan(s3b_lib, wb)
    assert plan_a[1:] == plan_b[1:]  # same sizes: a mix-up between the calls stays inside their buffers
    seq = {}
    for key, w, plan in (("a", wa, plan_a), ("b", wb, plan_b)):
        seq["fbank", key] = fbank_ex(s3b_lib, w, 1)
        seq["mel", key] = melspec_ex(s3b_lib, w, "mel", 1, plan=plan)[0]
    torch.cuda.synchronize()
    return wa, wb, plan_a, plan_b, seq


def _run_pair(s3b_lib, what, wa, wb, plan_a, plan_b, sa, sb):
    if what == "fbank":
        return fbank_ex(s3b_lib, wa, 1, stream=sa), fbank_ex(s3b_lib, wb, 1, stream=sb)
    return (melspec_ex(s3b_lib, wa, "mel", 1, stream=sa, plan=plan_a)[0],
            melspec_ex(s3b_lib, wb, "mel", 1, stream=sb, plan=plan_b)[0])


def _same(x, y):
    return torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))


@pytest.mark.gpu
def test_calls_on_two_streams_keep_their_own_inputs(s3b_lib):
    """Ordering check: call 1 is queued on stream A behind a ~0.1 s sleep, call 2 on stream B, same sizes, other audio;
    each must equal its sequential result. The staging copy and the kernels of one call are queued together, so this
    protocol runs all of call 2 before any of call 1: it checks stream order, not the overlap of the test below."""
    wa, wb, plan_a, plan_b, seq = _two_stream_inputs(s3b_lib, 3, 1)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    for what in ("fbank", "mel"):
        gate = torch.cuda.Event()
        with torch.cuda.stream(sa):
            torch.cuda._sleep(200_000_000)
            gate.record(sa)
        sa.wait_event(gate)
        out1, out2 = _run_pair(s3b_lib, what, wa, wb, plan_a, plan_b, sa, sb)
        torch.cuda.synchronize()
        assert _same(out1, seq[what, "a"]) and _same(out2, seq[what, "b"]), what


@pytest.mark.gpu
def test_overlapping_calls_on_two_streams(s3b_lib):
    """Call 1 (32 x 10 s, milliseconds of kernels) on stream A, then at once call 2 with the same sizes and other audio
    on an idle stream B. Call 2's staging lands while call 1's kernels are still queued or running: with one staging
    buffer / tmp shared between calls, call 1's later blocks and stages would read call 2's pointers and features.
    Whether they do depends on scheduling; with per-call, stream-ordered buffers both results are always exact."""
    wa, wb, plan_a, plan_b, seq = _two_stream_inputs(s3b_lib, 32, 10)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    for what in ("fbank", "mel"):
        out1, out2 = _run_pair(s3b_lib, what, wa, wb, plan_a, plan_b, sa, sb)
        torch.cuda.synchronize()
        assert _same(out1, seq[what, "a"]) and _same(out2, seq[what, "b"]), what


# ---- rejected arguments (no kernel is launched: the checks come before any device work) --------------------------------
def test_spectral_entry_points_reject_bad_arguments(s3b_lib):
    lib = s3b_lib
    dummy = torch.zeros(1)
    ptrs = (C.c_void_p * 2)(dummy.data_ptr(), dummy.data_ptr())
    out = C.c_void_p(dummy.data_ptr())
    bad = (C.c_int64 * 2)(16000, -1)
    good_opts = L.S3BSpectralOpts(cmvn=0)
    wrong = L.S3BSpectralOpts()
    wrong.struct_size = 8

    def refused(status, text):
        with pytest.raises(L.S3BError, match=text):
            L.check(status)

    refused(lib.s3b_fbank(ptrs, bad, 2, out, None), "negative")
    refused(lib.s3b_fbank_ex(ptrs, bad, 2, C.byref(good_opts), out, None), "negative")
    refused(lib.s3b_fbank_ex(ptrs, (C.c_int64 * 2)(16000, 400), 2, C.byref(wrong), out, None), "struct_size")
    for cmvn in (2, -1):
        refused(lib.s3b_fbank_ex(ptrs, (C.c_int64 * 2)(16000, 400), 2, C.byref(L.S3BSpectralOpts(cmvn=cmvn)), out,
                                 None), "cmvn must be 0 or 1")
        refused(lib.s3b_melspec_ex(ptrs, (C.c_int64 * 2)(16000, 100), 2, 16000, 1, None, None, 0,
                                   C.byref(L.S3BSpectralOpts(cmvn=cmvn)), out, None), "cmvn must be 0 or 1")
    refused(lib.s3b_trimmed_lengths(ptrs, bad, 2, (C.c_int64 * 2)()), "negative")
    i32 = C.c_int32 * 2
    ok_trim = (C.c_int64 * 2)(16000, 100)
    # trimmed length outside [0, padded_len]
    for tl in ((16001, 100), (16000, -1)):
        refused(lib.s3b_melspec(ptrs, (C.c_int64 * 2)(*tl), 2, 16000, 1, i32(101, 1), i32(101, 1), 101, out, None),
                "trimmed_lens")
        refused(lib.s3b_melspec_ex(ptrs, (C.c_int64 * 2)(*tl), 2, 16000, 1, None, None, 0, C.byref(good_opts), out,
                                   None), "trimmed_lens")
    # feats_len outside [0, 1 + padded_len / 160] (101 frames here), final_len outside [0, t_out]
    refused(lib.s3b_melspec(ptrs, ok_trim, 2, 16000, 1, i32(102, 1), i32(101, 1), 101, out, None), "feats_len")
    refused(lib.s3b_melspec(ptrs, ok_trim, 2, 16000, 0, i32(101, -1), i32(101, 1), 101, out, None), "feats_len")
    refused(lib.s3b_melspec(ptrs, ok_trim, 2, 16000, 1, i32(101, 1), i32(102, 1), 101, out, None), "final_len")
    refused(lib.s3b_melspec(ptrs, ok_trim, 2, 16000, 1, i32(101, 1), i32(101, -2), 101, out, None), "final_len")
    refused(lib.s3b_melspec_ex(ptrs, ok_trim, 2, 16000, 1, i32(101, 1), i32(101, 1), 101, C.byref(wrong), out, None),
            "struct_size")
