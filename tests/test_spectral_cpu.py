"""Spectral baselines on structured audio, CPU side: the fp64 restatement (tests/spectral_ref.py) and the fp32 oracle
against the executed reference (tests/golden/spectral_structured.pt, oracle/make_golden.py --only spectral).

The reference computes in fp32, so "agrees" means: every well-conditioned reference element lies within the fp32 error
bound spectral_ref derives for it from the fp64 values (the same stage bounds the CUDA kernels are held to, see the
module docstring). Elements the bound cannot speak for (floored energies, columns CMVN cannot condition) get the
structural checks instead."""
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "oracle"))
import spectral_ref as R  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "spectral_structured.pt"


@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLDEN, weights_only=False)


def _wavs(spec):
    return [R.with_tail(R.structured_wav(kind, n), tail) for kind, n, tail in spec]


def _checked_wavs(fx, which):
    wavs = _wavs(fx[which + "_spec"])
    got = torch.stack([w.double().sum() for w in wavs] + [w.double().abs().sum() for w in wavs])
    assert torch.allclose(got, fx["checksum_" + which], rtol=1e-12, atol=1e-9), "waveform recipe drifted"
    return wavs


def test_fbank_restatement_matches_reference(fx):
    wavs = _checked_wavs(fx, "fbank")
    eps_w = R.bank_eps("kaldi")
    raw, z = fx["cases"]["fbank_no_cmvn"], fx["cases"]["fbank"]
    assert raw.shape == z.shape == (len(wavs), R.num_frames(max(len(w) for w in wavs)), 240)
    worst = {"logmel": 0.0, "delta": 0.0, "cmvn": 0.0}
    for b, w in enumerate(wavs):
        m = R.num_frames(len(w))
        s = R.fbank_bounds(w, eps_w)
        g = raw[b, :m].double()
        worst["logmel"] = max(worst["logmel"], R.interval_ratio(g[:, :80], s["f"], s["lo"], s["hi"]).max().item())
        r = (g[:, 80:] - s["F"][:, 80:]).abs() / s["dF"][:, 80:]
        worst["delta"] = max(worst["delta"], r.max().item())
        assert torch.count_nonzero(raw[b, m:]) == 0 and torch.count_nonzero(z[b, m:]) == 0
        zb = z[b, :m].double()
        assert torch.equal(torch.isnan(zb), torch.isnan(s["z"]))
        if m > 1:
            rz = ((zb - s["z"]).abs() / s["dz"])[:, s["cond"]]
            worst["cmvn"] = max(worst["cmvn"], rz.max().item() if rz.numel() else 0.0)
        # no |z| <= (m - 1) / sqrt(m) here: torch's fp32 std and mean round separately, so on a column that is
        # constant up to rounding the reference divides a one-ulp residue by ~1e-10 (|z| ~ 1e4 in this fixture)
    print("fbank reference vs fp64, worst measured/bound:", {k: f"{v:.3f}" for k, v in worst.items()})
    assert max(worst.values()) <= 1.0


@pytest.mark.parametrize("feat", ["mel", "linear"])
def test_stft_restatement_matches_reference(fx, feat):
    wavs = _checked_wavs(fx, "stft")
    eps_w = R.bank_eps("htk")
    ref = fx["cases"][feat]
    s = R.stft_bounds(wavs, feat, eps_w)
    assert ref.shape == (len(wavs), max(s["final_len"]), 80 if feat == "mel" else 201)
    worst = 0.0
    for b in range(len(wavs)):
        n, keep = s["feats_len"][b], min(s["final_len"][b], s["feats_len"][b])
        assert torch.count_nonzero(ref[b, keep:]) == 0
        if n < 2:
            continue
        z, dz, cond = R.cmvn_bound(s["f"][b, :n], s["df"][b, :n])
        g = ref[b, :keep].double()
        rz = ((g - z[:keep]).abs() / dz[:keep])[:, cond]
        worst = max(worst, rz.max().item() if rz.numel() else 0.0)
    print(f"{feat} reference vs fp64, worst measured/bound: {worst:.3f}")
    assert worst <= 1.0


def test_fp32_oracle_matches_reference(fx):
    """oracle/fbank_oracle.py (fp32) against the same golden: both sit inside the fp64 restatement's fp32 bound, so they
    may differ by twice it."""
    import fbank_oracle as FO

    wavs = _checked_wavs(fx, "fbank")
    raw = fx["cases"]["fbank_no_cmvn"]
    for b, w in enumerate(wavs):
        m = R.num_frames(len(w))
        s = R.fbank_bounds(w, R.bank_eps("kaldi"))
        x = FO.log_mel(w)
        d = FO.deltas(x)
        o = torch.cat([x, d, FO.deltas(d)], -1).double()
        assert ((o - raw[b, :m].double()).abs() <= 2 * s["dF"]).all()
    full = FO.fbank_forward(wavs)
    assert torch.equal(torch.isnan(full), torch.isnan(fx["cases"]["fbank"]))
    swavs = _checked_wavs(fx, "stft")
    for feat in ("mel", "linear"):
        got, ref = FO.spectrogram_forward(swavs, feat), fx["cases"][feat]
        assert got.shape == ref.shape
        s = R.stft_bounds(swavs, feat, R.bank_eps("htk"))
        for b in range(len(swavs)):
            n, keep = s["feats_len"][b], min(s["final_len"][b], s["feats_len"][b])
            if n < 2:
                continue
            z, dz, cond = R.cmvn_bound(s["f"][b, :n], s["df"][b, :n])
            diff = (got[b, :keep].double() - ref[b, :keep].double()).abs()[:, cond]
            assert (diff <= 2 * dz[:keep][:, cond]).all()


def test_spectrogram_plan_lengths_match_reference(fx):
    from s3prl_b200.upstream.baseline import SpectrogramExpert

    wavs = _checked_wavs(fx, "stft")
    trimmed = [R.trimmed_length(w) for w in wavs]
    assert trimmed != [len(w) for w in wavs]  # the trim rule is exercised (trailing 0.0 and -0.0)
    lp, feats_len, final_len, t_out = SpectrogramExpert.plan_lengths([len(w) for w in wavs], trimmed)
    assert (lp, feats_len, final_len) == (R.plan_lengths([len(w) for w in wavs], trimmed)[0],
                                          *R.plan_lengths([len(w) for w in wavs], trimmed)[2:])
    for feat in ("mel", "linear"):
        ref = fx["cases"][feat]
        assert t_out == ref.shape[1]
        for b, n in enumerate(final_len):
            assert torch.count_nonzero(ref[b, n:]) == 0


# ---- the hamming-window front end of APC, DeCoAR, DeCoAR 2.0 and NPC (tests/test_fbank_frontend_gpu.py) ------------------
def _frontend_inputs():
    from test_fbank_frontend_gpu import batches

    return [(kind, w) for items in batches().values() for kind, w in items]


def _torch_cmvn(f, step):
    """The reference's CMVN module on its [1, D, T] layout ((x - mean) / (eps + std) over dim 2), then y[::step]."""
    y = f.T.unsqueeze(0)
    y = (y - y.mean(2, keepdim=True)) / (1e-10 + y.std(2, keepdim=True))
    return y.squeeze(0).T[::step]


def test_hamming_frontend_matches_torchaudio_fp64(monkeypatch):
    """fbank_cmvn_forward against torchaudio's kaldi.fbank(window_type="hamming", 80 bins) plus the reference's CMVN,
    all in float64, on every input of the GPU test. kaldi.fbank builds its mel banks in fp32 whatever the input dtype;
    they are checked against kaldi_mel_banks within bank_eps and then replaced by the fp64 banks, so what remains to
    compare is framing, DC removal, pre-emphasis, the window, the FFT, the floor and the log. The log-mel agrees to
    1e-10 (the fp32 bounds start near 1e-7), and CMVN to 2e-10 / (1e-10 + std) per column."""
    from torchaudio.compliance import kaldi

    banks64 = R.kaldi_mel_banks(torch.float64)[:, :-1]
    get_mel_banks = kaldi.get_mel_banks

    def fp64_banks(*args, **kwargs):
        b, centers = get_mel_banks(*args, **kwargs)
        assert b.shape == banks64.shape and (b.double() - banks64).abs().max() <= R.bank_eps("kaldi")
        return banks64, centers

    monkeypatch.setattr(kaldi, "get_mel_banks", fp64_banks)
    worst_f = worst_z = 0.0
    for kind, w in _frontend_inputs():
        ta = kaldi.fbank(w.double().unsqueeze(0), num_mel_bins=R.NMEL, sample_frequency=R.SR, window_type="hamming")
        assert ta.dtype == torch.float64
        f = R.fbank_stages(w, torch.float64, "hamming")["f"]
        worst_f = max(worst_f, (ta - f).abs().max().item())
        scale = 1e-10 + f.std(dim=0)
        for step in (1, 2):
            z = R.fbank_cmvn_forward(w, step)
            assert z.shape == (-(-len(f) // step), R.NMEL), kind
            worst_z = max(worst_z, ((_torch_cmvn(ta, step) - z).abs() * scale).max().item())
    print(f"hamming front end vs torchaudio fp64: log-mel {worst_f:.2e}, CMVN x (1e-10 + std) {worst_z:.2e}")
    assert worst_f <= 1e-10 and worst_z <= 2e-10


def _biased_std_cmvn(f, step):
    return ((f - f.mean(dim=0, keepdim=True)) / (R.LOG_EPS + f.std(dim=0, unbiased=False, keepdim=True)))[::step]


FRONTEND_MISTAKES = {  # name -> (steps it applies to, the wrong front end from the fp64 stages and the waveform)
    "biased std": ((1, 2), lambda f, w, step: _biased_std_cmvn(f, step)),
    "y[1::2] for y[::2]": ((2,), lambda f, w, step: R.cmvn(f)[1::2]),
    "statistics over the kept frames only": ((2,), lambda f, w, step: R.cmvn(f[::step])),
    "povey window": ((1, 2), lambda f, w, step: R.cmvn_frames(R.fbank_stages(w, torch.float64, "povey")["f"], step)),
    "no pre-emphasis": ((1, 2), lambda f, w, step: R.cmvn_frames(
        R.fbank_stages(w, torch.float64, "hamming", preemph=0.0)["f"], step)),
}


def test_frontend_bounds_reject_plausible_mistakes():
    """Each plausible wrong formula of the front end lands at least 100 times outside the per-element bound that
    test_fbank_frontend_gpu holds the kernels to (dz on the conditioned columns), at some element of that test's
    inputs: a kernel that made one of these mistakes fails there."""
    eps_w = R.bank_eps("kaldi")
    worst = {name: (0.0, None) for name in FRONTEND_MISTAKES}
    for kind, w in _frontend_inputs():
        s = R.fbank_cmvn_bounds(w, eps_w, 1)
        for name, (steps, wrong) in FRONTEND_MISTAKES.items():
            for step in steps:
                z, dz, cond = s["z"][::step], s["dz"][::step], s["cond"]
                if len(s["f"][::step]) < 2 or not cond.any():
                    continue
                zw = wrong(s["f"], w, step)
                n = min(len(zw), len(z))
                r = ((zw[:n] - z[:n]).abs() / dz[:n])[:, cond].max().item()
                if r > worst[name][0]:
                    worst[name] = (r, f"{kind} step {step}")
    print("\nwrong front ends, largest |wrong - fp64| / dz:")
    for name, (r, where) in worst.items():
        print(f"  {name:38s} {r:12.1f}  ({where})")
    assert all(r >= 100 for r, _ in worst.values()), worst
