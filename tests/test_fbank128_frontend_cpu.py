"""The 128-bin fbank front ends of SSAST (hanning window, (f + 4.2677393) / 9.1379948) and MAE-AST (povey window,
eval batch norm times 0.5, unfolded into patches) as spectral_ref restates them, anchored without a GPU:
- the fp64 restatement equals torchaudio's kaldi.fbank(num_mel_bins=128) run in fp64 with either window, and the fp64
  oracles (mae_ast_oracle.fbank / frontend, ssast_oracle.window_fbank), so the oracles and the bounds
  tests/test_fbank128_frontend_gpu.py holds the kernels to describe one computation;
- the 128-bin bank's structure: bin 3 empty in fp32 and fp64, single-FFT-bin support at the low edge, and the bounds
  finite there (the floor, not NaN);
- plausible wrong front ends land far outside those bounds on the GPU test's inputs, and the one that cannot (the
  first sample's pre-emphasis, multiplied by a window that is 0 there) changes nothing."""
import math
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import mae_ast_oracle as MO  # noqa: E402
import spectral_ref as R  # noqa: E402
import ssast_oracle as SO  # noqa: E402
from test_fbank128_frontend_gpu import BN_PAIRS, corpus  # noqa: E402

NMEL = 128


def test_128bin_restatement_matches_torchaudio_fp64(monkeypatch):
    """fbank_stages(nmel=128) against torchaudio's kaldi.fbank(num_mel_bins=128) in float64, with the povey (MAE-AST)
    and the hanning (SSAST) window, on every input of the GPU test. kaldi.fbank builds its banks in fp32 whatever the
    input dtype; they are checked against kaldi_mel_banks(.., 128) within bank_eps and replaced by the fp64 banks."""
    from torchaudio.compliance import kaldi

    banks64 = R.kaldi_mel_banks(torch.float64, NMEL)[:, :-1]
    get_mel_banks = kaldi.get_mel_banks

    def fp64_banks(*args, **kwargs):
        b, centers = get_mel_banks(*args, **kwargs)
        assert b.shape == banks64.shape and (b.double() - banks64).abs().max() <= R.bank_eps("kaldi", NMEL)
        return banks64, centers

    monkeypatch.setattr(kaldi, "get_mel_banks", fp64_banks)
    worst = {}
    for window in ("povey", "hanning"):
        for kind, w in corpus():
            if len(w) < R.WIN:
                continue
            ta = kaldi.fbank(w.double().unsqueeze(0), num_mel_bins=NMEL, sample_frequency=R.SR, window_type=window)
            assert ta.dtype == torch.float64
            f = R.fbank_stages(w, torch.float64, window, nmel=NMEL)["f"]
            worst[window] = max(worst.get(window, 0.0), (ta - f).abs().max().item())
    print(f"128-bin front end vs torchaudio fp64: {worst}")
    assert all(v <= 1e-10 for v in worst.values()), worst


def test_128bin_restatement_matches_the_oracles():
    """mae_ast_oracle's fbank and normalised, unfolded operand, and ssast_oracle's window features, against
    spectral_ref's stages and bounds' fp64 values on every input."""
    sd = {"batch_norm.running_mean": torch.tensor([-8.25]), "batch_norm.running_var": torch.tensor([12.5])}
    eps_w = R.bank_eps("kaldi", NMEL)
    worst = 0.0
    for kind, w in corpus():
        if len(w) < R.WIN:
            continue
        f = R.fbank_stages(w, torch.float64, "povey", nmel=NMEL)["f"]
        worst = max(worst, (MO.fbank(w) - f).abs().max().item())
        y = R.mae_ast_bounds(w, eps_w, -8.25, 12.5)["y"]
        worst = max(worst, (MO.normalise(MO.fbank(w), sd) - y).abs().max().item())
        S = len(w)
        m = R.num_frames(S)
        ref = SO.window_fbank(w.double(), S // R.SHIFT)[:m]
        worst = max(worst, (ref - R.ssast_bounds(w, eps_w)["y"]).abs().max().item())
    print(f"128-bin restatement vs the fp64 oracles: {worst:.2e}")
    assert worst <= 1e-12


def test_128bin_bank_structure_and_finite_bounds():
    """Bin 3 of the 128-bin bank has no weight in fp32 or fp64 (its energy is 0: the floor in every frame), the
    lowest bins have one FFT bin of support, and the bounds there are finite: bin 3's log-mel is exactly log(eps)
    inside [lo, hi], and every interval of every input is finite."""
    b32, b64 = R.kaldi_mel_banks(torch.float32, NMEL), R.kaldi_mel_banks(torch.float64, NMEL)
    assert torch.equal(b32[3], torch.zeros_like(b32[3])) and torch.equal(b64[3], torch.zeros_like(b64[3]))
    assert torch.equal((b32 > 0).sum(1)[:12], (b64 > 0).sum(1)[:12])
    nnz = (b64 > 0).sum(1)
    assert (nnz == 0).nonzero().flatten().tolist() == [3]
    assert int((nnz[:12] == 1).sum()) >= 6, nnz[:12].tolist()
    eps_w = R.bank_eps("kaldi", NMEL)
    floor = math.log(R.FLOOR)
    for kind, w in corpus():
        if len(w) < R.WIN:
            continue
        for s in (R.mae_ast_bounds(w, eps_w, -8.25, 12.5), R.ssast_bounds(w, eps_w)):
            for k in ("lo", "hi", "ylo", "yhi"):
                assert torch.isfinite(s[k]).all(), (kind, k)
            assert (s["E"][:, 3] == 0).all() and (s["f"][:, 3] == floor).all()
            assert (s["lo"][:, 3] <= floor).all() and (s["hi"][:, 3] >= floor).all()
            assert (s["ylo"] <= s["y"]).all() and (s["y"] <= s["yhi"]).all(), kind


def test_first_sample_preemphasis_is_multiplied_by_zero():
    """Pre-emphasis against 0 instead of the replicated first sample changes only y_0, and the povey and hanning
    windows are 0 at n = 0: both 128-bin front ends are bit for bit the same either way, so no bound can tell the two
    apart (the hamming window of the 80-bin front end is 0.08 there)."""
    for window in ("povey", "hanning"):
        assert R.WINDOWS[window](torch.float64)[0] == 0.0
        for kind, w in corpus():
            if len(w) < R.WIN:
                continue
            a = R.fbank_stages(w, torch.float64, window, nmel=NMEL)["f"]
            b = R.fbank_stages(w, torch.float64, window, nmel=NMEL, replicate_first=False)["f"]
            assert torch.equal(a, b), (window, kind)
    assert R.WINDOWS["hamming"](torch.float64)[0] > 0.07


def _transposed_unfold(x, kind):
    """MO.unfold with each patch's (kt, kc) block read transposed: column j kt + i instead of i kc + j."""
    kt, kc = MO.KINDS[kind]
    B, Fm, C = x.shape
    T = Fm // kt
    p = x[:, : T * kt].reshape(B, T, kt, C // kc, kc).permute(0, 1, 3, 4, 2)
    return p.reshape(B, T * (C // kc), kt * kc)


def _mae(f, rm, rv):
    a, c, _, _ = R.bn_fold(rm, rv)
    return f * a + c


MAE_MISTAKES = {  # name -> the wrong normalised fbank [m, 128 or 80] from (bounds, waveform, rm, rv)
    "hanning for povey": lambda s, w, rm, rv: _mae(R.fbank_stages(w, torch.float64, "hanning", nmel=NMEL)["f"], rm, rv),
    "80-bin bank": lambda s, w, rm, rv: _mae(R.fbank_stages(w, torch.float64, "povey", nmel=80)["f"], rm, rv),
    "batch norm without 0.5": lambda s, w, rm, rv: (s["f"] - rm) / math.sqrt(rv + 1e-5),
    "sqrt(rv) without 1e-5": lambda s, w, rm, rv: 0.5 * (s["f"] - rm) / math.sqrt(rv),
    "log(E + eps)": lambda s, w, rm, rv: _mae((s["E"] + R.FLOOR).log(), rm, rv),
}
SSAST_MISTAKES = {  # name -> the wrong window features [m, 128 or 80] from (bounds, waveform)
    "povey for hanning": lambda s, w: (R.fbank_stages(w, torch.float64, "povey", nmel=NMEL)["f"] + R.SSAST_SHIFT)
    / R.SSAST_SCALE,
    "80-bin bank": lambda s, w: (R.fbank_stages(w, torch.float64, "hanning", nmel=80)["f"] + R.SSAST_SHIFT)
    / R.SSAST_SCALE,
    "shift and scale swapped": lambda s, w: (s["f"] + R.SSAST_SCALE) / R.SSAST_SHIFT,
    "log(E + eps)": lambda s, w: ((s["E"] + R.FLOOR).log() + R.SSAST_SHIFT) / R.SSAST_SCALE,
}


def _ratio(wrong, s):
    n = wrong.shape[-1]
    return R.interval_ratio(wrong, s["y"][..., :n], s["ylo"][..., :n], s["yhi"][..., :n]).max().item()


def test_128bin_bounds_reject_plausible_mistakes():
    """Each plausible wrong formula of either front end lands at least 100 times outside the per-element interval
    test_fbank128_frontend_gpu holds the kernels to, at some element of that test's inputs (MAE-AST at every batch-norm
    pair it runs; the unfold transposed at both patch shapes): a kernel that made one of these mistakes fails there."""
    eps_w = R.bank_eps("kaldi", NMEL)
    worst = {}

    def note(name, r, where):
        if r > worst.get(name, (0.0, None))[0]:
            worst[name] = (r, where)

    for kind, w in corpus():
        if len(w) < R.WIN:
            continue
        for rm, rv in BN_PAIRS:
            s = R.mae_ast_bounds(w, eps_w, rm, rv)
            for name, wrong in MAE_MISTAKES.items():
                note(f"MAE-AST {name}", _ratio(wrong(s, w, rm, rv), s), f"{kind} rm {rm} rv {rv}")
            for mk in MO.KINDS:
                if len(s["y"]) >= MO.KINDS[mk][0]:
                    lo, hi, y = (MO.unfold(s[k][None], mk) for k in ("ylo", "yhi", "y"))
                    r = R.interval_ratio(_transposed_unfold(s["y"][None], mk), y, lo, hi).max().item()
                    note(f"MAE-AST (kt, kc) transposed, {mk}", r, f"{kind} rm {rm} rv {rv}")
        s = R.ssast_bounds(w, eps_w)
        for name, wrong in SSAST_MISTAKES.items():
            note(f"SSAST {name}", _ratio(wrong(s, w), s), kind)
    print("\nwrong 128-bin front ends, largest |wrong - fp64| / distance to the interval's edge:")
    for name, (r, where) in worst.items():
        print(f"  {name:42s} {r:12.1f}  ({where})")
    assert len(worst) == len(MAE_MISTAKES) + len(SSAST_MISTAKES) + len(MO.KINDS)
    assert all(r >= 100 for r, _ in worst.values()), worst
