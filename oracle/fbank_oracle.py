"""TEST INFRASTRUCTURE — CPU oracle of the `fbank` baseline upstream (kaldi-style log-mel + deltas + CMVN).

Restates, with plain fp32 torch-CPU ops, what ``s3prl.hub.fbank()(wavs)`` computes:
``torchaudio.compliance.kaldi.fbank`` (third-party, un-vendored: torchaudio >= 0.8, 2.11.0 installed; algorithm
restated from its published source, kaldi.py:154-218, 436-512, 514-646) with the arguments of
s3prl/upstream/baseline/fbank.yaml, then 2 x ComputeDeltas(win_length=5) and per-utterance CMVN
(s3prl/upstream/baseline/extracter.py:44-90), then pad_sequence (baseline/expert.py:69-79).
Pinned by tests/golden/fbank.pt, produced by executing the reference (oracle/make_golden.py).
"""
from __future__ import annotations

import math
from typing import List, Sequence

import torch
import torch.nn.functional as F

WIN, SHIFT, NFFT, NMEL = 400, 160, 512, 80
EPS = torch.finfo(torch.float32).eps


def num_frames(n: int) -> int:
    """snip_edges=True: m = 1 + (n - window) // shift (kaldi.py _get_strided)."""
    return 0 if n < WIN else 1 + (n - WIN) // SHIFT


def mel_banks() -> torch.Tensor:
    """get_mel_banks(80, 512, 16000, low 20, high 0 -> nyquist, no vtln) (kaldi.py:436-512) -> [80, 256]."""
    nyquist = 8000.0
    fft_bin_width = 16000.0 / NFFT
    mel_low = 1127.0 * math.log(1.0 + 20.0 / 700.0)
    mel_high = 1127.0 * math.log(1.0 + nyquist / 700.0)
    delta = (mel_high - mel_low) / (NMEL + 1)
    b = torch.arange(NMEL).unsqueeze(1)
    left, center, right = mel_low + b * delta, mel_low + (b + 1.0) * delta, mel_low + (b + 2.0) * delta
    mel = (1127.0 * (1.0 + fft_bin_width * torch.arange(NFFT / 2) / 700.0).log()).unsqueeze(0)
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    return torch.max(torch.zeros(1), torch.min(up, down))


def log_mel(wav: torch.Tensor) -> torch.Tensor:
    """kaldi fbank of one utterance: [n] -> [m, 80] (kaldi.py:_get_window + fbank body)."""
    m = num_frames(len(wav))
    frames = wav.float().unfold(0, WIN, SHIFT)[:m]
    frames = frames - frames.mean(dim=1, keepdim=True)  # remove_dc_offset
    prev = torch.cat([frames[:, :1], frames[:, :-1]], dim=1)  # replicate pad on the left
    frames = frames - 0.97 * prev  # preemphasis
    window = torch.hann_window(WIN, periodic=False).pow(0.85)  # povey
    frames = F.pad(frames * window, (0, NFFT - WIN))
    spec = torch.fft.rfft(frames).abs().pow(2.0)  # use_power
    banks = F.pad(mel_banks(), (0, 1))  # [80, 257]
    return torch.max(spec @ banks.T, torch.tensor(EPS)).log()


def deltas(x: torch.Tensor, win_length: int = 5) -> torch.Tensor:
    """torchaudio.functional.compute_deltas over time, replicate padding: x [m, d] -> [m, d]."""
    n = (win_length - 1) // 2
    denom = n * (n + 1) * (2 * n + 1) / 3
    spec = F.pad(x.t().unsqueeze(0), (n, n), mode="replicate")
    kernel = torch.arange(-n, n + 1, dtype=x.dtype).repeat(spec.shape[1], 1, 1)
    return (F.conv1d(spec, kernel, groups=spec.shape[1]) / denom).squeeze(0).t()


def fbank_forward(wavs: Sequence[torch.Tensor]) -> torch.Tensor:
    """[B, max_frames, 240] = pad_sequence(CMVN(cat(x, d, dd)))."""
    feats: List[torch.Tensor] = []
    for w in wavs:
        x = log_mel(w)
        d = deltas(x)
        dd = deltas(d)
        f = torch.cat([x, d, dd], dim=-1)
        f = (f - f.mean(dim=0, keepdim=True)) / (1e-10 + f.std(dim=0, keepdim=True))
        feats.append(f)
    return torch.nn.utils.rnn.pad_sequence(feats, batch_first=True)


# ------------------------------------------------------------------------------------------------
# mel / linear (torch.stft path): s3prl/upstream/baseline/preprocessor.py:150-223 + expert.py:52-79
# ------------------------------------------------------------------------------------------------
def melscale_fbanks_htk(n_freqs: int = 201, n_mels: int = 80, f_max: float = 8000.0, sample_rate: int = 16000) -> torch.Tensor:
    """torchaudio.functional.melscale_fbanks(201, 0, 8000, 80, 16000, norm=None, mel_scale="htk") -> [201, 80]."""
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_min, m_max = 0.0, 2595.0 * math.log10(1.0 + f_max / 700.0)
    m_pts = torch.linspace(m_min, m_max, n_mels + 2)
    f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = -slopes[:, :-2] / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.max(torch.zeros(1), torch.min(down, up))


def spectrogram_forward(wavs: Sequence[torch.Tensor], feat_type: str = "mel") -> torch.Tensor:
    """[B, T_out, 80 | 201] for the `mel` / `linear` upstreams, length quirks of the reference included."""
    eps = 1e-10
    orig_lens = [len(w) for w in wavs]
    trimmed = []
    for w in wavs:  # last non-zero sample + 1 (the whole thing if all zero), preprocessor.py:166-175
        nz = w.nonzero()
        trimmed.append(len(w) if len(nz) == 0 else int(nz[:, -1].max()) + 1)
    # the reference's trim slices the channel axis of a [1, L] row (preprocessor.py:176-182): the batch keeps its
    # original padding, and only feats_len below sees the trimmed lengths
    x = torch.nn.utils.rnn.pad_sequence([w.float() for w in wavs], batch_first=True)
    spec = torch.stft(x, n_fft=400, hop_length=160, win_length=400, window=torch.hann_window(400), center=True,
                      pad_mode="reflect", normalized=False, onesided=True, return_complex=True)
    feat = spec.abs().pow(2)  # [B, 201, n_frames]
    if feat_type == "mel":
        feat = (feat.transpose(-1, -2) @ melscale_fbanks_htk()).transpose(-1, -2)
    feat = (feat + eps).log()
    downsample_rate = x.size(-1) / feat.size(-1)
    feats_len = [round(n / downsample_rate) for n in trimmed]
    outs = []
    for f, n in zip(feat, feats_len):
        f = f[:, :n]
        outs.append(((f - f.mean(dim=-1, keepdim=True)) / (f.std(dim=-1, keepdim=True) + eps)).transpose(-1, -2))
    feats = torch.nn.utils.rnn.pad_sequence(outs, batch_first=True)
    ratio = len(feats[0]) / orig_lens[0]  # expert.py:62 uses the FIRST utterance's length
    final = [round(n * ratio) for n in orig_lens]
    return torch.nn.utils.rnn.pad_sequence([f[:n] for f, n in zip(feats, final)], batch_first=True)
