"""TEST INFRASTRUCTURE — dtype-generic restatement of the spectral baselines (`fbank`, `fbank_no_cmvn`, `mel`, `linear`),
run in float64 by the tests, and the per-element error bounds the fp32 implementations are held to.

What it restates (the reference executes these; tests/golden/spectral_structured.pt pins this module to it):
  fbank: torchaudio.compliance.kaldi.fbank with fbank.yaml (kaldi.py:154-218 framing, DC removal, pre-emphasis with the
    first sample replicated, povey window; :436-512 mel banks; :514-646 512-point rfft, power, max(E, eps), log),
    then 2 x ComputeDeltas(win_length=5, replicate) and per-utterance CMVN with unbiased std
    (s3prl/upstream/baseline/extracter.py:58-90), pad_sequence (expert.py:69-79).
  mel / linear: OnlinePreprocessor.forward (preprocessor.py:150-223): the lengths without trailing exact zeros (torch
    `nonzero`, so -0.0 counts as zero) set the CMVN frame counts, while the STFT runs over the batch padded to the
    longest original length; torch.stft(n_fft 400, hop 160, periodic hann, center, reflect) power, HTK mel banks for `mel`,
    log(x + 1e-10), CMVN over round(len / (Lp / n_frames)) frames, final cut by the first utterance's ratio
    (expert.py:52-66).
The fp32 oracle (oracle/fbank_oracle.py) is a separate, fp32-only restatement; this one keeps every intermediate the
bounds need. The product package never imports this module.

Bounds (u = 2^-24, one fp32 rounding). Stage by stage, each an absolute bound per element, derived from the fp64 values:
  frame  : dy_n <= w_n ((|d_n| + |d_n-1|) C_FRAME u + 1.97 dmu), d = x - mean, dmu <= K_SUM u sum|x| / 400
  DFT    : |dX_k| <= S eta ||y||_1 + ||dy||_1 for every bin of the frame, eta = 7u: each of the S butterfly stages
           adds at most eta times the magnitude of a partial sum, and every partial sum of bin k is bounded by
           ||y||_1 (the componentwise form of Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., 24.1;
           twiddles within u). fbank's FFT: N = 512, S = 9. The mel/linear kernel's direct 400-term DFT is held to
           the same FFT class (S = 9), not to the 400 u ||y||_1 of a serial sum.
  power  : dP_k <= 2 |X_k| dX + dX^2 + 5u P_k
  mel    : dE_j <= sum_k W_jk dP_k + gamma_nnz sum_k W_jk (P_k + dP_k) + eps_W sum_{k in supp_j +- 1} P_k
           (eps_W: twice the largest |fp32 bank - fp64 bank|; the reference builds its banks in fp32)
  log    : the value lies in [log(max(E - dE, floor)), log(max(E + dE, floor))] (fbank) or
           [log(max(E - dE, 0) + 1e-10), log(E + dE + 1e-10)] (mel / linear), widened by the log's own rounding;
           so where |E - floor| < dE either side of the max is accepted
  deltas : dD_t <= (2 df_t-2 + df_t-1 + df_t+1 + 2 df_t+2) / 10 + 6u (2|f_t-2| + |f_t-1| + |f_t+1| + 2|f_t+2|) / 10
           + u |D_t| with the replicate-clamped indices; then the same for delta-delta on (D, dD)
  (SSAST / MAE-AST: the same stages up to the log-mel with 128 bins and the hanning / povey window, then an affine map
  whose fp32 constants' error and roundings ssast_interval / mae_ast_bounds carry)
  (DeCoAR 2.0 / APC / DeCoAR / NPC: the same stages up to the log-mel with the hamming window and no deltas, then the
  CMVN below over all m frames, every step-th row kept: fbank_cmvn_forward, fbank_cmvn_bounds)
  CMVN   : with s the fp64 std and ds <= ||df||_2 / sqrt(m - 1) + 4u s, dmu <= mean(df) + 2u max|f|:
           dz_t <= (df_t + dmu + u |f_t - mu|) / (s - ds) + |z_t| ds / (s - ds) + 3u |z_t|,
           compared only where s >= KAPPA max_t df_t (KAPPA = 10); other columns get structural checks.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

SR = 16000
WIN, SHIFT, NFFT, NMEL = 400, 160, 512, 80  # kaldi fbank
N_STFT, HOP, NBIN = 400, 160, 201  # mel / linear
FLOOR = float(torch.finfo(torch.float32).eps)  # kaldi's max(E, eps): the fp32 epsilon, whatever the dtype
LOG_EPS = 1e-10  # preprocessor.py's eps and CMVN's
U = 2.0 ** -24
C_FRAME, K_SUM, ETA, STAGES, KAPPA = 8.0, 64.0, 7.0 * U, 9, 10.0


def gamma(n) -> float:
    return n * U / (1 - n * U)


# ---- structured inputs (deterministic recipes; float64 math rounded once to fp32) --------------------------------
def structured_wav(kind: str, n: int, seed: int = 0) -> torch.Tensor:
    t = torch.arange(n, dtype=torch.float64) / SR
    g = torch.Generator().manual_seed(seed)
    tone = lambda f, a=0.5: a * torch.sin(2 * math.pi * f * t + 0.3)  # noqa: E731
    if kind == "tone_fbank_bin":  # on a 512-point FFT bin centre (31.25 Hz spacing)
        x = tone(31.25 * 37)
    elif kind == "tone_fbank_half":
        x = tone(31.25 * 37.5)
    elif kind == "tone_stft_bin":  # on a 400-point bin centre (40 Hz spacing)
        x = tone(40.0 * 37)
    elif kind == "tone_stft_half":
        x = tone(40.0 * 37.5)
    elif kind == "tone_25":
        x = tone(25.0)
    elif kind == "tone_7990":
        x = tone(7990.0)
    elif kind == "chirp":  # linear 50 Hz -> 7.9 kHz over the utterance
        T = max(n, 2) / SR
        x = 0.5 * torch.sin(2 * math.pi * (50.0 * t + (7900.0 - 50.0) / (2 * T) * t * t))
    elif kind == "bursts":  # 60 ms 1 kHz bursts separated by 90 ms of exact zeros
        x = tone(1000.0) * ((torch.arange(n) % 2400) < 960).double()
    elif kind in ("pink", "brown"):  # 1/f and 1/f^2 power: ~40 and ~60 dB of tilt over the band
        w = torch.randn(n, generator=g, dtype=torch.float64)
        spec = torch.fft.rfft(w)
        f = torch.arange(spec.numel(), dtype=torch.float64).clamp(min=1.0)
        spec = spec / (f.sqrt() if kind == "pink" else f)
        x = torch.fft.irfft(spec, n=n)
        x = 0.3 * x / x.abs().max()
    elif kind == "dc":
        x = 0.5 + 1e-3 * torch.randn(n, generator=g, dtype=torch.float64)
    elif kind == "impulses":
        x = ((torch.arange(n) % 97) == 5).double()
    elif kind == "clipped":  # a 440 Hz tone at 1.6x full scale, clipped to [-1, 1]
        x = tone(440.0, 1.6).clamp(-1.0, 1.0)
    elif kind == "int16":  # full int16 scale
        x = structured_wav("chirp", n).double()
        x = torch.round(x / x.abs().max() * 32767.0)
    elif kind == "tiny":
        x = 1e-5 * structured_wav("pink", n, seed).double()
    elif kind == "zeros":
        x = torch.zeros(n, dtype=torch.float64)
    elif kind == "white":
        x = torch.randn(n, generator=g, dtype=torch.float64)
    else:
        raise KeyError(kind)
    return x.float()


def with_tail(x: torch.Tensor, tail: str, k: int = 333) -> torch.Tensor:
    """Trim-rule variants: trailing exact zeros, trailing -0.0, or only the first sample non-zero."""
    x = x.clone()
    if tail == "zeros":
        x[-k:] = 0.0
    elif tail == "negzeros":
        x[-k:] = -0.0
    elif tail == "first_only":
        x[1:] = 0.0
        x[0] = 0.25
    elif tail != "none":
        raise KeyError(tail)
    return x


def trimmed_length(w: torch.Tensor) -> int:
    nz = w.nonzero()
    return len(w) if len(nz) == 0 else int(nz[:, -1].max()) + 1


# ---- fbank --------------------------------------------------------------------------------------------------------
def num_frames(n: int) -> int:
    return 0 if n < WIN else 1 + (n - WIN) // SHIFT


def povey_window(dtype) -> torch.Tensor:
    return torch.hann_window(WIN, periodic=False, dtype=dtype).pow(0.85)


def hamming_window(dtype) -> torch.Tensor:
    """kaldi's "hamming" (kaldi.py _get_window): 0.54 - 0.46 cos(2 pi n / (N - 1)), evaluated in float64."""
    n = torch.arange(WIN, dtype=torch.float64)
    return (0.54 - 0.46 * torch.cos(2 * math.pi * n / (WIN - 1))).to(dtype)


def hanning_window(dtype) -> torch.Tensor:
    """kaldi's "hanning" (SSAST's window): torch.hann_window(400, periodic=False)."""
    return torch.hann_window(WIN, periodic=False, dtype=dtype)


WINDOWS = {"povey": povey_window, "hamming": hamming_window, "hanning": hanning_window}


def kaldi_mel_banks(dtype, nmel: int = NMEL) -> torch.Tensor:
    """get_mel_banks(nmel bins, 512-point FFT, 16 kHz, low 20 Hz, high = Nyquist) in `dtype` -> [nmel, 257]."""
    mel_low, mel_high = 1127.0 * math.log(1.0 + 20.0 / 700.0), 1127.0 * math.log(1.0 + 8000.0 / 700.0)
    delta = (mel_high - mel_low) / (nmel + 1)
    b = torch.arange(nmel, dtype=dtype).unsqueeze(1)
    left, center, right = mel_low + b * delta, mel_low + (b + 1.0) * delta, mel_low + (b + 2.0) * delta
    mel = 1127.0 * (1.0 + (SR / NFFT) * torch.arange(NFFT // 2, dtype=dtype) / 700.0).log()
    w = torch.min((mel - left) / (center - left), (right - mel) / (right - center)).clamp(min=0.0)
    return F.pad(w, (0, 1))


def fbank_stages(wav: torch.Tensor, dtype=torch.float64, window: str = "povey", preemph: float = 0.97,
                 nmel: int = NMEL, replicate_first: bool = True) -> Dict[str, torch.Tensor]:
    """Every stage of kaldi fbank + deltas for one utterance: frames [m, 400] after DC removal (d) and after
    pre-emphasis and window (y), spectrum X [m, 257], power P, mel energies E [m, nmel], log-mel f, deltas D and DD.
    window: a key of WINDOWS (the fbank baseline's and MAE-AST's povey, the hamming of DeCoAR 2.0 / APC / DeCoAR / NPC,
    SSAST's hanning); nmel: 80, or SSAST's and MAE-AST's 128. replicate_first=False pre-emphasises the first sample
    against 0 instead of itself (kaldi replicates it; only a window that is not 0 at n = 0 sees the difference)."""
    m = num_frames(len(wav))
    frames = wav.to(dtype).unfold(0, WIN, SHIFT)[:m]
    d = frames - frames.mean(dim=1, keepdim=True)
    prev = torch.cat([d[:, :1] if replicate_first else torch.zeros_like(d[:, :1]), d[:, :-1]], dim=1)
    y = (d - preemph * prev) * WINDOWS[window](dtype)
    X = torch.fft.rfft(F.pad(y, (0, NFFT - WIN)))
    P = X.abs().pow(2)
    E = P @ kaldi_mel_banks(dtype, nmel).T
    f = E.clamp(min=FLOOR).log()
    D = deltas(f)
    return {"x": frames, "d": d, "y": y, "X": X, "P": P, "E": E, "f": f, "D": D, "DD": deltas(D)}


def deltas(x: torch.Tensor, win_length: int = 5) -> torch.Tensor:
    """torchaudio compute_deltas over time (dim 0) with replicate padding: sum_n n (x[t+n] - x[t-n]) / 10."""
    n = (win_length - 1) // 2
    denom = n * (n + 1) * (2 * n + 1) / 3
    m = x.shape[0]
    idx = lambda k: (torch.arange(m) + k).clamp(0, m - 1)  # noqa: E731
    return sum(k * (x[idx(k)] - x[idx(-k)]) for k in range(1, n + 1)) / denom


def cmvn(f: torch.Tensor) -> torch.Tensor:
    """(f - mean) / (1e-10 + unbiased std) per column over dim 0 (NaN for one row, as torch.std)."""
    return (f - f.mean(dim=0, keepdim=True)) / (LOG_EPS + f.std(dim=0, keepdim=True))


def cmvn_frames(f: torch.Tensor, step: int) -> torch.Tensor:
    """DeCoAR 2.0 / APC CMVN (decoar2/audio.py CMVN, apc/audio.py): cmvn over all m frames, then every step-th frame,
    f[::step] (step 2: DeCoAR 2.0's low frame rate; step 1: APC, DeCoAR and NPC keep every frame)."""
    return cmvn(f)[::step]


def fbank_cmvn_forward(wav: torch.Tensor, step: int, dtype=torch.float64) -> torch.Tensor:
    """The front end of DeCoAR 2.0 (step 2) and APC / DeCoAR / NPC (step 1) for one utterance: kaldi fbank with the
    hamming window and 80 bins, no deltas, then cmvn_frames -> [ceil(m / step), 80]."""
    return cmvn_frames(fbank_stages(wav, dtype, "hamming")["f"], step)


def fbank_forward(wavs: Sequence[torch.Tensor], use_cmvn: bool = True, dtype=torch.float64) -> torch.Tensor:
    feats = []
    for w in wavs:
        s = fbank_stages(w, dtype)
        f = torch.cat([s["f"], s["D"], s["DD"]], dim=-1)
        feats.append(cmvn(f) if use_cmvn else f)
    return torch.nn.utils.rnn.pad_sequence(feats, batch_first=True)


# ---- mel / linear ---------------------------------------------------------------------------------------------------
def htk_mel_banks(dtype) -> torch.Tensor:
    """melscale_fbanks(201, f_min 0, f_max 8000, 80, 16 kHz, norm None, htk) in `dtype` -> [201, 80]."""
    all_freqs = torch.linspace(0, SR // 2, NBIN, dtype=dtype)
    m_max = 2595.0 * math.log10(1.0 + 8000.0 / 700.0)
    f_pts = 700.0 * (10.0 ** (torch.linspace(0.0, m_max, NMEL + 2, dtype=dtype) / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    return torch.min(-slopes[:, :-2] / f_diff[:-1], slopes[:, 2:] / f_diff[1:]).clamp(min=0.0)


def plan_lengths(orig_lens: List[int], trimmed: List[int]):
    """(Lp, n_frames, feats_len, final_len) by the reference's Python arithmetic. Lp is the longest ORIGINAL length:
    preprocessor.py:176-182 slices `wav[:wav_len]` on the channel axis of a [1, L] row, so the trim never shortens
    the padded batch; only feats_len sees the trimmed lengths."""
    lp = max(orig_lens)
    n_frames = 1 + lp // HOP
    feats_len = [round(n / (lp / n_frames)) for n in trimmed]
    ratio = max(feats_len) / orig_lens[0]
    final_len = [min(round(n * ratio), max(feats_len)) for n in orig_lens]
    return lp, n_frames, feats_len, final_len


def stft_stages(wavs: Sequence[torch.Tensor], feat: str, dtype=torch.float64) -> Dict[str, object]:
    """The padded batch through the STFT: frames and windowed frames y [B, n_frames, 400], X, P [B, n_frames, 201], E (the
    mel energies, or P for linear) and the log features f [B, n_frames, dim] of every frame, plus the lengths."""
    orig = [len(w) for w in wavs]
    trimmed = [trimmed_length(w) for w in wavs]
    lp, n_frames, feats_len, final_len = plan_lengths(orig, trimmed)
    x = torch.nn.utils.rnn.pad_sequence([w.to(dtype) for w in wavs], batch_first=True)
    xp = F.pad(x.unsqueeze(1), (N_STFT // 2, N_STFT // 2), mode="reflect").squeeze(1)
    frames = xp.unfold(-1, N_STFT, HOP)
    y = frames * torch.hann_window(N_STFT, periodic=True, dtype=dtype)
    X = torch.fft.rfft(y)
    P = X.abs().pow(2)
    E = P @ htk_mel_banks(dtype) if feat == "mel" else P
    return {"frames": frames, "y": y, "X": X, "P": P, "E": E, "f": (E + LOG_EPS).log(), "lp": lp, "n_frames": n_frames,
            "trimmed": trimmed, "feats_len": feats_len, "final_len": final_len}


def spectrogram_forward(wavs: Sequence[torch.Tensor], feat: str, use_cmvn: bool = True, dtype=torch.float64):
    """use_cmvn: the mel / linear entries' output [B, t_out, dim]; else the log features of every padded frame."""
    s = stft_stages(wavs, feat, dtype)
    if not use_cmvn:
        return s["f"]
    outs = [cmvn(f[:n]) for f, n in zip(s["f"], s["feats_len"])]
    feats = torch.nn.utils.rnn.pad_sequence(outs, batch_first=True)
    return torch.nn.utils.rnn.pad_sequence([f[:n] for f, n in zip(feats, s["final_len"])], batch_first=True)


# ---- bounds ---------------------------------------------------------------------------------------------------------
def bank_eps(which: str, nmel: int = NMEL) -> float:
    """Twice the largest |fp32 bank weight - fp64 bank weight|, at least 2u (nmel: kaldi banks only)."""
    fn = (lambda dt: kaldi_mel_banks(dt, nmel)) if which == "kaldi" else htk_mel_banks
    return max(2.0 * (fn(torch.float32).double() - fn(torch.float64)).abs().max().item(), 2 * U)


def frame_error(x: torch.Tensor, d: torch.Tensor, y: torch.Tensor, window: torch.Tensor, fbank: bool) -> torch.Tensor:
    """One absolute bound per frame on every DFT bin. fbank: x / d are the raw and DC-removed frames and y follows
    pre-emphasis and the window; mel / linear: no DC removal or pre-emphasis (d = x)."""
    if fbank:
        dmu = K_SUM * U * x.abs().sum(-1, keepdim=True) / WIN
        dprev = torch.cat([d[..., :1], d[..., :-1]], dim=-1)
        dy = window * ((d.abs() + dprev.abs()) * C_FRAME * U + 1.97 * dmu)
    else:
        dy = window * x.abs() * 2 * U
    return STAGES * ETA * y.abs().sum(-1) + dy.abs().sum(-1)


def energy_error(X: torch.Tensor, dX: torch.Tensor, banks: torch.Tensor, eps_w: float) -> torch.Tensor:
    """dE [..., n_out] from dX (one per frame, [...]) through power and the mel projection banks [n_bins, n_out]."""
    A, P = X.abs(), X.abs().pow(2)
    dXe = dX.unsqueeze(-1)
    dP = 2 * A * dXe + dXe * dXe + 5 * U * P
    nnz = (banks > 0).sum(0).clamp(min=1).to(P.dtype)
    support = (banks > 0).to(P.dtype)
    support = ((support + F.pad(support[1:], (0, 0, 0, 1)) + F.pad(support[:-1], (0, 0, 1, 0))) > 0).to(P.dtype)
    return dP @ banks + gamma(nnz) * ((P + dP) @ banks) + eps_w * (P @ support)


def log_interval(E: torch.Tensor, dE: torch.Tensor, fbank: bool):
    """Interval [lo, hi] the fp32 log feature may take, given the fp64 energy E and its bound dE."""
    if fbank:
        lo, hi = (E - dE).clamp(min=FLOOR).log(), (E + dE).clamp(min=FLOOR).log()
        r = 2 * U * torch.maximum(lo.abs(), hi.abs())
    else:
        lo, hi = ((E - dE).clamp(min=0) + LOG_EPS).log(), (E + dE + LOG_EPS).log()
        r = U + 2 * U * torch.maximum(lo.abs(), hi.abs())
    return lo - r, hi + r


def delta_error(f: torch.Tensor, df: torch.Tensor, D: torch.Tensor) -> torch.Tensor:
    """Bound on compute_deltas(f) along dim 0, given the per-element bound df of its input."""
    m = f.shape[0]
    idx = lambda k: (torch.arange(m) + k).clamp(0, m - 1)  # noqa: E731
    w = {-2: 2.0, -1: 1.0, 1: 1.0, 2: 2.0}
    prop = sum(c * df[idx(k)] for k, c in w.items()) / 10
    mag = sum(c * f[idx(k)].abs() for k, c in w.items()) / 10
    return prop + 6 * U * mag + U * D.abs()


def cmvn_bound(f: torch.Tensor, df: torch.Tensor):
    """(z, dz, conditioned) per column of f [m, n] with per-element input bound df: the fp64 CMVN, its bound, and
    the columns where s >= KAPPA max df (dz is only meaningful there)."""
    m = f.shape[0]
    z = cmvn(f)
    s = f.std(dim=0, keepdim=True)
    ds = df.norm(dim=0, keepdim=True) / math.sqrt(max(m - 1, 1)) + 4 * U * s
    dmu = df.mean(dim=0, keepdim=True) + 2 * U * f.abs().amax(dim=0, keepdim=True)
    mu = f.mean(dim=0, keepdim=True)
    den = (s - ds).clamp(min=1e-300)
    dz = (df + dmu + U * (f - mu).abs()) / den + z.abs() * ds / den + 3 * U * z.abs()
    cond = (s >= KAPPA * df.amax(dim=0, keepdim=True)).squeeze(0) & (m > 1)
    return z, dz, cond


def logmel_bounds(wav: torch.Tensor, eps_w: float, window: str = "povey", nmel: int = NMEL) -> Dict[str, torch.Tensor]:
    """fp64 stages of one utterance (fbank_stages with `window` and nmel bins) and lo/hi, df of an fp32 log-mel of
    them. eps_w: bank_eps("kaldi", nmel)."""
    s = fbank_stages(wav, torch.float64, window, nmel=nmel)
    dX = frame_error(s["x"], s["d"], s["y"], WINDOWS[window](torch.float64), fbank=True)
    dE = energy_error(s["X"], dX, kaldi_mel_banks(torch.float64, nmel).T, eps_w)
    lo, hi = log_interval(s["E"], dE, fbank=True)
    return {**s, "dE": dE, "lo": lo, "hi": hi, "df": torch.maximum(s["f"] - lo, hi - s["f"])}


def fbank_cmvn_bounds(wav: torch.Tensor, eps_w: float, step: int) -> Dict[str, torch.Tensor]:
    """The front end of fbank_cmvn_forward and its bounds: logmel_bounds with the hamming window, then cmvn_bound of
    the log-mel over all m frames, carried through the decimation: z, dz [ceil(m / step), 80] are the rows t of frame
    step * t, and the statistics (mean, std and their bounds) stay those of all m frames, so the per-element bound of a
    kept row is that row's bound before decimation; cond [80] is the columns' conditioning over all m frames."""
    s = logmel_bounds(wav, eps_w, "hamming")
    z, dz, cond = cmvn_bound(s["f"], s["df"])
    return {**s, "z": z[::step], "dz": dz[::step], "cond": cond}


def _f32(v: float) -> float:
    return torch.tensor(v, dtype=torch.float64).float().item()


def bn_fold(rm: float, rv: float):
    """MAE-AST's eval batch norm times 0.5 as y = x a + c: (a, c) in fp64 and as the library rounds them to fp32
    (a = fp32(0.5 / sqrt(rv + 1e-5)), c = fp32(-rm a) with a in fp64)."""
    a = 0.5 / math.sqrt(rv + 1e-5)
    return a, -rm * a, _f32(a), _f32(-rm * a)


def mae_ast_bounds(wav: torch.Tensor, eps_w: float, rm: float, rv: float) -> Dict[str, torch.Tensor]:
    """MAE-AST's normalised fbank of one utterance (povey window, 128 bins, y = f a + c) in fp64 and the interval an
    fp32 fma(f32, a32, c32) of the kernel's log-mel f32 lies in: f32 in [lo, hi], so f32 a32 + c32 is within
    a (f32 - f) + |a32 - a| |f32| + |c32 - c| of y, plus the fma's one rounding u |y|."""
    s = logmel_bounds(wav, eps_w, "povey", 128)
    a, c, a32, c32 = bn_fold(rm, rv)
    e = abs(a32 - a) * torch.maximum(s["lo"].abs(), s["hi"].abs()) + abs(c32 - c)
    lo, hi = a * s["lo"] + c - e, a * s["hi"] + c + e
    r = U * torch.maximum(lo.abs(), hi.abs())
    return {**s, "y": a * s["f"] + c, "ylo": lo - r, "yhi": hi + r}


SSAST_SHIFT, SSAST_SCALE = 4.2677393, 4.5689974 * 2  # (f + shift) / scale (ssast/audio.py)


def ssast_interval(lo: torch.Tensor, hi: torch.Tensor):
    """The interval of fp32 (f32 + shift32) / scale32 for f32 in [lo, hi]: the sum and the quotient each rounded once
    (u |.|), with the fp32 constants' error carried (the interval holds both the fp32 and the fp64 constants' value)."""
    sh, sc = (SSAST_SHIFT, _f32(SSAST_SHIFT)), (SSAST_SCALE, _f32(SSAST_SCALE))
    glo, ghi = lo + min(sh), hi + max(sh)
    glo, ghi = glo - U * glo.abs(), ghi + U * ghi.abs()
    qlo = torch.minimum(glo / sc[0], glo / sc[1])
    qhi = torch.maximum(ghi / sc[0], ghi / sc[1])
    return qlo - U * qlo.abs(), qhi + U * qhi.abs()


def ssast_bounds(seg: torch.Tensor, eps_w: float) -> Dict[str, torch.Tensor]:
    """SSAST's normalised fbank of one zero-padded window of S samples (hanning window, 128 bins) in fp64, y = (f +
    shift) / scale [m, 128], and the interval ssast_interval gives the kernel's value from the log-mel's [lo, hi]."""
    s = logmel_bounds(seg, eps_w, "hanning", 128)
    ylo, yhi = ssast_interval(s["lo"], s["hi"])
    return {**s, "y": (s["f"] + SSAST_SHIFT) / SSAST_SCALE, "ylo": ylo, "yhi": yhi}


def fbank_bounds(wav: torch.Tensor, eps_w: float) -> Dict[str, torch.Tensor]:
    """fp64 stages of one utterance and the bounds of an fp32 implementation of them: lo/hi of the log-mel, df, dD,
    dDD, then the no-CMVN features F [m, 240] with dF, and z, dz, cond of CMVN."""
    s = logmel_bounds(wav, eps_w)
    dD = delta_error(s["f"], s["df"], s["D"])
    dDD = delta_error(s["D"], dD, s["DD"])
    Fe = torch.cat([s["f"], s["D"], s["DD"]], -1)
    dF = torch.cat([s["df"], dD, dDD], -1)
    z, dz, cond = cmvn_bound(Fe, dF)
    return {**s, "F": Fe, "dF": dF, "z": z, "dz": dz, "cond": cond}


def stft_bounds(wavs: Sequence[torch.Tensor], feat: str, eps_w: float) -> Dict[str, object]:
    """fp64 stages of a mel / linear batch and the lo/hi interval of every log feature of every padded frame."""
    s = stft_stages(wavs, feat, torch.float64)
    win = torch.hann_window(N_STFT, periodic=True, dtype=torch.float64)
    dX = frame_error(s["frames"], s["frames"], s["y"], win, fbank=False)
    banks = htk_mel_banks(torch.float64) if feat == "mel" else torch.eye(NBIN, dtype=torch.float64)
    dE = energy_error(s["X"], dX, banks, eps_w if feat == "mel" else 0.0)
    lo, hi = log_interval(s["E"], dE, fbank=False)
    return {**s, "dE": dE, "lo": lo, "hi": hi, "df": torch.maximum(s["f"] - lo, hi - s["f"])}


def interval_ratio(got: torch.Tensor, ref: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor) -> torch.Tensor:
    """|got - ref| over the distance from ref to the interval's edge on got's side (<= 1 inside the interval)."""
    got = got.double()
    up = (got - ref) / (hi - ref).clamp(min=1e-300)
    dn = (ref - got) / (ref - lo).clamp(min=1e-300)
    return torch.where(got >= ref, up, dn).clamp(min=0)
