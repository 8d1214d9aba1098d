"""TEST INFRASTRUCTURE — CPU oracle of DeCoAR (``decoar``, ``decoar_layers``).

A plain torch-CPU restatement of what the reference computes for ``UpstreamExpert(wavs)["hidden_states"]``
(s3prl/upstream/decoar/{audio,decoar,expert}.py, decoar_layers/{decoar,expert}.py): the APC oracle's front end
(tests/apc_oracle.py: kaldi fbank with the hamming window, CMVN over all frames, pad_sequence), post_extract_proj, then
each direction's 4-layer LSTM stack written out from PyTorch's equations (gate order i, f, g, o; h_0 = c_0 = 0) with
an explicit time loop; the backward stack walks each utterance from its last valid frame down to frame 0. Pinned by
the goldens that tools/make_decoar_golden.py writes by executing the reference (tests/test_decoar_cpu.py). The
product package never imports this module.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

import apc_oracle as AO

NUM_LAYERS = 4


def lstm(xg: torch.Tensor, w_hh: torch.Tensor, lens: Sequence[int], backward: bool = False) -> torch.Tensor:
    """One nn.LSTM layer over packed sequences from the input projection xg = x W_ih^T + b_ih + b_hh [B, T, 4H]:
    outputs [B, T, H] in natural time, zero at t >= lens[b]. ``backward``: utterance b runs from frame lens[b] - 1 down
    to 0 (the reference's flipBatch around its LSTM)."""
    B, T, H4 = xg.shape
    H = H4 // 4
    h = torch.zeros(B, H, dtype=xg.dtype)
    c = torch.zeros(B, H, dtype=xg.dtype)
    out = torch.zeros(B, T, H, dtype=xg.dtype)
    valid = torch.tensor(list(lens))
    rows = torch.arange(B)
    for step in range(T):
        live = step < valid
        t = (valid - 1 - step).clamp(min=0) if backward else torch.full((B,), step)
        g = xg[rows, t.clamp(max=T - 1)] + h @ w_hh.T
        i, f, gg, o = g[:, :H].sigmoid(), g[:, H:2 * H].sigmoid(), g[:, 2 * H:3 * H].tanh(), g[:, 3 * H:].sigmoid()
        cn = f * c + i * gg
        hn = o * cn.tanh()
        lv = live.unsqueeze(1)
        c = torch.where(lv, cn, c)
        h = torch.where(lv, hn, h)
        for b in torch.nonzero(live).flatten().tolist():
            out[b, t[b]] = hn[b]
    return out


def decoar_forward(wavs: Optional[Sequence[torch.Tensor]], sd: Dict[str, torch.Tensor],
                   dtype: torch.dtype = torch.float32,
                   feats: Optional[Tuple[torch.Tensor, List[int]]] = None) -> Tuple[List[torch.Tensor], List[int]]:
    """The four layer outputs cat(forward, backward) [B, T, 2048] of decoar_layers (the last one is decoar's only
    hidden state) and the frame counts m_b. feats: precomputed ``apc_oracle.batch_features(wavs)``."""
    x, lens = feats if feats is not None else AO.batch_features(wavs)
    x = x.to(dtype) @ sd["post_extract_proj.weight"].to(dtype).T + sd["post_extract_proj.bias"].to(dtype)
    layers = []
    inputs = [x, x]
    for k in range(NUM_LAYERS):
        outs = []
        for d, name in enumerate(("forward_lstm.", "backward_lstm.")):
            xg = (inputs[d] @ sd[f"{name}weight_ih_l{k}"].to(dtype).T + sd[f"{name}bias_ih_l{k}"].to(dtype)
                  + sd[f"{name}bias_hh_l{k}"].to(dtype))
            outs.append(lstm(xg, sd[f"{name}weight_hh_l{k}"].to(dtype), lens, backward=d == 1))
        inputs = outs
        layers.append(torch.cat(outs, dim=-1))
    return layers, lens
