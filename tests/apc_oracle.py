"""TEST INFRASTRUCTURE — CPU oracle of APC / VQ-APC (``apc``, ``vq_apc``).

A plain fp32 torch-CPU restatement of what the reference computes for ``UpstreamExpert(wavs)["hidden_states"]``
(s3prl/upstream/apc/{audio,apc,expert}.py): per utterance the DeCoAR 2.0 oracle's kaldi fbank with the hamming window
and CMVN over all frames (tests/decoar2_oracle.py) without its ``[::2]``, pad_sequence, then the GRU stack written out
from PyTorch's equations (gate order r, z, n; h_0 = 0) and the residual. Pinned by the goldens that
tools/make_apc_golden.py writes by executing the reference (tests/test_apc_cpu.py). The product package never imports
this module.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

import decoar2_oracle as D2


def features(wav: torch.Tensor) -> torch.Tensor:
    """FeatureExtractor.forward (apc/audio.py:69-86): log-mel -> CMVN over all m frames: [m, 80]."""
    y = D2.log_mel_hamming(wav)
    return (y - y.mean(dim=0, keepdim=True)) / (1e-10 + y.std(dim=0, keepdim=True))


def batch_features(wavs: Sequence[torch.Tensor]) -> Tuple[torch.Tensor, List[int]]:
    """pad_sequence of the per-utterance features [B, T, 80] and the frame counts m_b."""
    feats = [features(w) for w in wavs]
    return torch.nn.utils.rnn.pad_sequence(feats, batch_first=True), [len(f) for f in feats]


def gru(xg: torch.Tensor, w_hh: torch.Tensor, b_hh: torch.Tensor, lens: Sequence[int]) -> torch.Tensor:
    """One nn.GRU layer over packed sequences from the input projection xg = x W_ih^T + b_ih [B, T, 3H]: outputs
    [B, T, H], zero at t >= lens[b] (pad_packed_sequence)."""
    B, T, H3 = xg.shape
    H = H3 // 3
    h = torch.zeros(B, H, dtype=xg.dtype, device=xg.device)
    out = torch.zeros(B, T, H, dtype=xg.dtype, device=xg.device)
    valid = torch.tensor(lens, device=xg.device)
    for t in range(T):
        gh = h @ w_hh.T + b_hh
        x = xg[:, t]
        r = torch.sigmoid(x[:, :H] + gh[:, :H])
        z = torch.sigmoid(x[:, H:2 * H] + gh[:, H:2 * H])
        n = torch.tanh(x[:, 2 * H:] + r * gh[:, 2 * H:])
        hn = (1 - z) * n + z * h
        live = (t < valid).unsqueeze(1)
        h = torch.where(live, hn, h)
        out[:, t] = torch.where(live, hn, torch.zeros_like(hn))
    return out


def apc_forward(wavs: Sequence[torch.Tensor], sd: Dict[str, torch.Tensor], residual: bool = True,
                num_layers: int = 3, dtype: torch.dtype = torch.float32,
                feats: Optional[Tuple[torch.Tensor, List[int]]] = None) -> Tuple[List[torch.Tensor], List[int]]:
    """The three hidden states of APC.forward + the expert's hooks (apc.py:101-169, expert.py:27-42) and the frame
    counts m_b. feats: precomputed ``batch_features(wavs)``."""
    x, lens = feats if feats is not None else batch_features(wavs)
    x = x.to(dtype)
    hidden = []
    for l in range(num_layers):
        p = f"rnn_layers.{l}."
        xg = x @ sd[p + "weight_ih_l0"].to(dtype).T + sd[p + "bias_ih_l0"].to(dtype)
        y = gru(xg, sd[p + "weight_hh_l0"].to(dtype), sd[p + "bias_hh_l0"].to(dtype), lens)
        if residual and l > 0:
            y = y + x
        hidden.append(y)
        x = y
    return hidden, lens
