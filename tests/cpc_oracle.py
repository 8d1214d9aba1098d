"""fp64 CPU restatement of modified CPC's forward (s3prl/upstream/cpc/{expert,model}.py), written from the model's
definition: pad the waveforms with zeros to the longest, five strided convolutions each followed by a per-frame norm
over the channels (unbiased variance, eps inside the square root) and ReLU, then an LSTM stack over every frame of the
padded batch from zero state. Returns the two hidden states the expert's hooks record, [B, T, 256] each."""
from __future__ import annotations

from typing import Dict, List

import torch

STRIDES = (5, 4, 2, 2, 2)
PADDINGS = (3, 2, 1, 1, 1)


def channel_norm_relu(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """x [B, C, T]: normalise each frame over C with the unbiased variance, affine, ReLU."""
    mean = x.mean(dim=1, keepdim=True)
    var = ((x - mean) ** 2).sum(dim=1, keepdim=True) / (x.shape[1] - 1)
    y = (x - mean) / torch.sqrt(var + 1e-5)
    return torch.clamp(y * w.reshape(1, -1, 1) + b.reshape(1, -1, 1), min=0.0)


def encoder(wav_pad: torch.Tensor, sd: Dict[str, torch.Tensor]) -> torch.Tensor:
    """[B, L] fp64 -> [B, T, 256]."""
    x = wav_pad.unsqueeze(1)
    for i, (s, p) in enumerate(zip(STRIDES, PADDINGS)):
        w = sd[f"gEncoder.conv{i}.weight"].double()
        x = torch.nn.functional.conv1d(x, w, sd[f"gEncoder.conv{i}.bias"].double(), stride=s, padding=p)
        x = channel_norm_relu(x, sd[f"gEncoder.batchNorm{i}.weight"].double(), sd[f"gEncoder.batchNorm{i}.bias"].double())
    return x.transpose(1, 2)


def lstm_layer(x: torch.Tensor, w_ih, w_hh, b_ih, b_hh) -> torch.Tensor:
    """One LSTM layer over [B, T, D] from h = c = 0, gates i, f, g, o."""
    B, T, _ = x.shape
    H = w_hh.shape[1]
    xg = x @ w_ih.T + b_ih + b_hh
    h = x.new_zeros(B, H)
    c = x.new_zeros(B, H)
    out = []
    for t in range(T):
        z = xg[:, t] + h @ w_hh.T
        i, f, g, o = z.split(H, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        out.append(h)
    return torch.stack(out, dim=1)


def forward(wavs: List[torch.Tensor], sd: Dict[str, torch.Tensor], num_layers: int, max_len: int = 0) -> List[torch.Tensor]:
    L = max(max(int(w.numel()) for w in wavs), max_len)
    pad = torch.zeros(len(wavs), L, dtype=torch.float64)
    for b, w in enumerate(wavs):
        pad[b, : w.numel()] = w.double()
    enc = encoder(pad, sd)
    x = enc
    for k in range(num_layers):
        x = lstm_layer(x, *(sd[f"gAR.baseNet.{n}_l{k}"].double() for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")))
    return [enc, x]
