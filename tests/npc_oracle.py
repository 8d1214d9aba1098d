"""TEST INFRASTRUCTURE — CPU oracle of NPC (``npc``).

An fp64 torch-CPU restatement of what the reference computes for ``UpstreamExpert(wavs)["hidden_states"]``
(s3prl/upstream/npc/{audio,npc,expert}.py): APC's features (tests/apc_oracle.py: kaldi fbank with the hamming window,
CMVN over all frames), pad_sequence, then per block the ConvBlock (conv k = 3 -> BatchNorm -> act -> 1x1 linear ->
BatchNorm (+ input) -> act) and the masked conv (tanh of the conv with the checkpoint's conv_mask applied), and feat as
the running sum of the masked convs. BatchNorm is applied as written (eval mode), not folded. Pinned by the goldens
that tools/make_npc_golden.py writes by executing the reference (tests/test_npc_cpu.py). The product package never
imports this module.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

import apc_oracle as AO


def _bn(x: torch.Tensor, sd: Dict[str, torch.Tensor], p: str) -> torch.Tensor:
    """BatchNorm1d in eval mode on [B, C, T] (eps 1e-5)."""
    d = x.dtype
    mean, var = sd[p + "running_mean"].to(d), sd[p + "running_var"].to(d)
    return (x - mean[:, None]) / torch.sqrt(var[:, None] + 1e-5) * sd[p + "weight"].to(d)[:, None] + \
        sd[p + "bias"].to(d)[:, None]


def npc_forward(wavs: Optional[Sequence[torch.Tensor]], sd: Dict[str, torch.Tensor], paras: dict,
                dtype: torch.dtype = torch.float64,
                feats: Optional[Tuple[torch.Tensor, List[int]]] = None) -> Tuple[List[torch.Tensor], List[int]]:
    """The 2 n_blocks + 1 hidden states of NPC.forward + the expert's hooks (npc.py NPC.forward, expert.py:27-41),
    each [B, T, 512], and the frame counts m_b. feats: precomputed ``apc_oracle.batch_features(wavs)``."""
    x, lens = feats if feats is not None else AO.batch_features(wavs)
    act = torch.relu if paras["activate"] == "relu" else torch.tanh
    h = x.to(dtype).transpose(1, 2)  # [B, C, T]
    hidden: List[torch.Tensor] = []
    feat = None
    k = paras["kernel_size"]
    for i in range(paras["n_blocks"]):
        b = f"blocks.{i}."
        res = h
        out = F.conv1d(h, sd[b + "conv.weight"].to(dtype), sd[b + "conv.bias"].to(dtype), padding=1)
        if paras["batch_norm"]:
            out = _bn(out, sd, b + "bn1.")
        out = act(out)
        out = F.conv1d(out, sd[b + "linear.weight"].to(dtype), sd[b + "linear.bias"].to(dtype))
        if paras["batch_norm"]:
            out = _bn(out, sd, b + "bn2.")
        if paras["residual"] and i > 0:
            out = out + res
        h = act(out)
        hidden.append(h.transpose(1, 2))
        mc = f"masked_convs.{i}."
        w = sd[mc + "conv_mask"].to(dtype) * sd[mc + "conv.weight"].to(dtype)
        m = torch.tanh(F.conv1d(h, w, sd[mc + "conv.bias"].to(dtype), padding=(k - 1) // 2)).transpose(1, 2)
        hidden.append(m)
        feat = m if feat is None else feat + m
    hidden.append(feat)
    return hidden, lens
