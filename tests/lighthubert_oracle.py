"""fp64 CPU restatement of LightHuBERT's forward on a cut subnet (s3prl/upstream/lighthubert/{expert,lighthubert}.py,
modules/scaling_transformer.py): per-utterance layer_norm of the waveform, zero padding, the conv stack, LayerNorm(512),
post_extract_proj with HuBERT's padded frames zeroed (hidden state 0), pos_conv + residual, encoder.layer_norm, then 12
post-LN layers. Built from oracle/upstream_oracle.py's pieces, which follow the same fairseq modules."""
from __future__ import annotations

import sys
from pathlib import Path
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "oracle"))
import upstream_oracle as O  # noqa: E402


def lighthubert_forward(wavs: Sequence[torch.Tensor], sd: Dict[str, torch.Tensor], sub,
                        max_len: Optional[int] = None) -> List[torch.Tensor]:
    """The 13 hidden states [B, T, E] (fp64) of the subnet ``sub`` (an ``ArchConfig``) with cut weights ``sd``."""
    sd = {k: v.double() for k, v in sd.items()}
    wavs = [F.layer_norm(w.double(), w.shape) for w in wavs]
    lens = [len(w) for w in wavs]
    L = max_len or max(lens)
    x = torch.zeros(len(wavs), L, dtype=torch.float64)
    for i, w in enumerate(wavs):
        x[i, : len(w)] = w
    feats = O.conv_feature_extractor(x, sd, sub.extractor_mode, sub.conv_bias).transpose(1, 2)
    T = feats.size(1)

    def ln(t, name):
        return F.layer_norm(t, (t.size(-1),), sd[f"{name}.weight"], sd[f"{name}.bias"], 1e-5)

    pad = O.frame_padding_mask_chunk_all(O.sample_padding_mask(lens, L), T)
    h = F.linear(ln(feats, "layer_norm"), sd["post_extract_proj.weight"], sd["post_extract_proj.bias"])
    h = h.masked_fill(pad.unsqueeze(-1), 0.0)
    hidden = [h]
    h = ln(h + O.positional_conv(h, sd, sub.conv_pos_groups), "encoder.layer_norm")
    for l in range(sub.encoder_layers):
        p = f"encoder.layers.{l}"
        h = ln(h + O.self_attention(h, sd, f"{p}.self_attn", sub.encoder_attention_heads, pad), f"{p}.self_attn_layer_norm")
        f = F.linear(F.gelu(F.linear(h, sd[f"{p}.fc1.weight"], sd[f"{p}.fc1.bias"])), sd[f"{p}.fc2.weight"], sd[f"{p}.fc2.bias"])
        h = ln(h + f, f"{p}.final_layer_norm")
        hidden.append(h)
    return hidden
