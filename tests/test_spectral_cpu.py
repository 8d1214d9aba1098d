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
