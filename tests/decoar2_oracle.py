"""TEST INFRASTRUCTURE — CPU oracle of DeCoAR 2.0 (``decoar2``).

A plain fp32 torch-CPU restatement of what the reference computes for ``UpstreamExpert(wavs)["hidden_states"]``
(s3prl/upstream/decoar2/{audio,decoar2,expert}.py): per utterance kaldi fbank (80 bins, hamming window; the mel banks
are the fbank oracle's, oracle/fbank_oracle.py), CMVN over all frames with the unbiased std, every second frame, then
pad_sequence, post_extract_proj on the padded rows, the padding mask t >= T_b, and the wav2vec 2.0 TransformerEncoder
(positional conv and attention from oracle/upstream_oracle.py; 12 post-LN layers). Pinned by the goldens that
tools/make_decoar2_golden.py writes by executing the reference (tests/test_decoar2_cpu.py). The product package never
imports this module.
"""
from __future__ import annotations

import sys
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "oracle"))
import fbank_oracle as FO  # noqa: E402
import upstream_oracle as O  # noqa: E402


def log_mel_hamming(wav: torch.Tensor) -> torch.Tensor:
    """torchaudio.compliance.kaldi.fbank(wav[None], num_mel_bins=80, sample_frequency=16000, window_type="hamming"):
    [n] -> [m, 80]. The fbank oracle's steps with the hamming window instead of povey."""
    m = FO.num_frames(len(wav))
    frames = wav.float().unfold(0, FO.WIN, FO.SHIFT)[:m]
    frames = frames - frames.mean(dim=1, keepdim=True)
    prev = torch.cat([frames[:, :1], frames[:, :-1]], dim=1)
    frames = frames - 0.97 * prev
    window = torch.hamming_window(FO.WIN, periodic=False, alpha=0.54, beta=0.46)
    frames = F.pad(frames * window, (0, FO.NFFT - FO.WIN))
    spec = torch.fft.rfft(frames).abs().pow(2.0)
    banks = F.pad(FO.mel_banks(), (0, 1))
    return torch.max(spec @ banks.T, torch.tensor(FO.EPS)).log()


def features(wav: torch.Tensor) -> torch.Tensor:
    """FeatureExtractor.forward (audio.py:69-86): log-mel -> CMVN over all m frames -> y[::2]: [(m + 1) // 2, 80]."""
    y = log_mel_hamming(wav)
    y = (y - y.mean(dim=0, keepdim=True)) / (1e-10 + y.std(dim=0, keepdim=True))
    return y[::2]


def batch_features(wavs: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, List[int]]:
    """pad_sequence of the per-utterance features [B, T, 80] and the frame counts T_b."""
    feats = [features(w) for w in wavs]
    return torch.nn.utils.rnn.pad_sequence(feats, batch_first=True), [len(f) for f in feats]


def decoar2_forward(wavs: Sequence[torch.Tensor], sd: Dict[str, torch.Tensor], layers: Optional[int] = None,
                    heads: int = 12, groups: int = 16) -> Tuple[List[torch.Tensor], torch.Tensor]:
    """hidden_states (layers + 1 tensors [B, T, 768]) and the frame padding mask of Decoar2.forward + the expert's hooks
    (decoar2.py:45-59, expert.py:33-48, wav2vec2_model.py:3046-3121). layers: the first `layers` encoder layers only."""
    sd = {k: v.float() for k, v in sd.items()}
    x, tb = batch_features(wavs)
    T = x.size(1)
    pad = torch.arange(T).unsqueeze(0) >= torch.tensor(tb).unsqueeze(1)
    h = F.linear(x, sd["post_extract_proj.weight"], sd["post_extract_proj.bias"])
    h = h.masked_fill(pad.unsqueeze(-1), 0.0)
    h = h + O.positional_conv(h, sd, groups)
    h = F.layer_norm(h, (h.size(-1),), sd["encoder.layer_norm.weight"], sd["encoder.layer_norm.bias"], 1e-5)
    n = layers if layers is not None else 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.layers."))

    def ln(t, name):
        return F.layer_norm(t, (t.size(-1),), sd[f"{name}.weight"], sd[f"{name}.bias"], 1e-5)

    hidden = []
    for l in range(n):
        p = f"encoder.layers.{l}"
        hidden.append(h)
        h = ln(h + O.self_attention(h, sd, f"{p}.self_attn", heads, pad), f"{p}.self_attn_layer_norm")
        f = F.linear(F.gelu(F.linear(h, sd[f"{p}.fc1.weight"], sd[f"{p}.fc1.bias"])), sd[f"{p}.fc2.weight"],
                     sd[f"{p}.fc2.bias"])
        h = ln(h + f, f"{p}.final_layer_norm")
    hidden.append(h)
    return hidden, pad
