"""TEST INFRASTRUCTURE — CPU oracle of the wav2vec 2.0 Conformer with rotary attention (``wav2vec2_conformer_rope``).

A plain fp32 torch-CPU restatement of what the reference computes for ``UpstreamExpert(wavs)["hidden_states"]`` with a
``layer_type="conformer"``, ``attn_type="espnet"``, ``pos_enc_type="rope"`` checkpoint. The front end (waveform
normalisation, conv stack, LayerNorm(512), post_extract_proj, the wav2vec 2.0 frame mask) is the shared oracle's
(oracle/upstream_oracle.py); the encoder is restated here. Pinned by the goldens tools/make_conformer_golden.py writes by
executing the reference (tests/test_conformer_cpu.py). The product package never imports this module.
"""
from __future__ import annotations

import math
import sys
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "oracle"))
import upstream_oracle as O  # noqa: E402


def rotary_inv_freq(sd: Dict[str, torch.Tensor], layer: int) -> torch.Tensor:
    """RotaryPositionalEmbedding.inv_freq of a 64-wide head (wav2vec2_model.py:51): the checkpoint's buffer if present."""
    key = f"encoder.layers.{layer}.self_attn.rotary_emb.inv_freq"
    return sd[key] if key in sd else 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))


def rope(x: torch.Tensor, inv_freq: torch.Tensor, heads: int) -> torch.Tensor:
    """apply_rotary_pos_emb per 64-wide head at frame index t of the padded batch (wav2vec2_model.py:25-71, 288-295):
    x * cos + rotate_half(x) * sin, rotate_half(u) = cat(-u[32:], u[:32]), angles fp32(t) * inv_freq."""
    B, T, D = x.shape
    f = torch.einsum("i,j->ij", torch.arange(T).type_as(inv_freq), inv_freq)
    emb = torch.cat((f, f), dim=-1)  # [T, 64]
    cos, sin = emb.cos()[None, :, None, :], emb.sin()[None, :, None, :]
    xh = x.view(B, T, heads, 64)
    rot = torch.cat((-xh[..., 32:], xh[..., :32]), dim=-1)
    return (xh * cos + rot * sin).view(B, T, D)


def conformer_encoder(h: torch.Tensor, sd: Dict[str, torch.Tensor], cfg, pad: Optional[torch.Tensor]) -> List[torch.Tensor]:
    """ConformerEncoder.extract_features (wav2vec2_model.py:3171-3211) on the masked projection h [B, T, D] and
    TransformerEncoder.forward's final LayerNorm for pre-LN models (:3046-3052); no pos_conv. The hidden states are the
    inputs of the layers plus the encoder output. One ConformerEncoderLayer (:537-578):
      x = x + 0.5 ffn1(x); x = x + linear_out(attn(rope(LN(x)) -> q, k; LN(x) -> v)); x = x + conv_module(x);
      x = final_layer_norm(x + 0.5 ffn2(x))
    with ffn = LN -> w_1 -> SiLU -> w_2 and conv_module = LN -> pointwise_conv1 -> GLU -> depthwise Conv1d(k, padding
    k // 2) over the whole padded T -> BatchNorm1d (eval) -> SiLU -> pointwise_conv2 (:371-393). Padded frames are not
    re-zeroed anywhere; only the attention masks padded keys."""
    heads = cfg.encoder_attention_heads

    def ln(t, name):
        return F.layer_norm(t, (t.size(-1),), sd[f"{name}.weight"], sd[f"{name}.bias"], 1e-5)

    def ffn(t, p):
        u = F.silu(F.linear(ln(t, f"{p}.layer_norm"), sd[f"{p}.w_1.weight"], sd[f"{p}.w_1.bias"]))
        return F.linear(u, sd[f"{p}.w_2.weight"], sd[f"{p}.w_2.bias"])

    def attention(t, p, inv_freq):
        B, T, D = t.shape
        y = ln(t, f"{p}.self_attn_layer_norm")
        yr = rope(y, inv_freq, heads)
        a = f"{p}.self_attn"
        q = F.linear(yr, sd[f"{a}.linear_q.weight"], sd[f"{a}.linear_q.bias"]).view(B, T, heads, 64).transpose(1, 2)
        k = F.linear(yr, sd[f"{a}.linear_k.weight"], sd[f"{a}.linear_k.bias"]).view(B, T, heads, 64).transpose(1, 2)
        v = F.linear(y, sd[f"{a}.linear_v.weight"], sd[f"{a}.linear_v.bias"]).view(B, T, heads, 64).transpose(1, 2)
        s = (q @ k.transpose(-2, -1)) / math.sqrt(64)
        if pad is not None:
            s = s.masked_fill(pad[:, None, None, :], float("-inf"))
        o = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(B, T, D)
        return F.linear(o, sd[f"{a}.linear_out.weight"], sd[f"{a}.linear_out.bias"])

    def conv_module(t, p):
        c = f"{p}.conv_module"
        u = ln(t, f"{c}.layer_norm").transpose(1, 2)
        u = F.glu(F.conv1d(u, sd[f"{c}.pointwise_conv1.weight"]), dim=1)
        w = sd[f"{c}.depthwise_conv.weight"]
        u = F.conv1d(u, w, padding=(w.size(2) - 1) // 2, groups=u.size(1))
        u = F.batch_norm(u, sd[f"{c}.batch_norm.running_mean"], sd[f"{c}.batch_norm.running_var"],
                         sd[f"{c}.batch_norm.weight"], sd[f"{c}.batch_norm.bias"], False, 0.0, 1e-5)
        u = F.conv1d(F.silu(u), sd[f"{c}.pointwise_conv2.weight"])
        return u.transpose(1, 2)

    if not cfg.layer_norm_first:
        h = ln(h, "encoder.layer_norm")
    hidden = []
    for l in range(cfg.encoder_layers):
        p = f"encoder.layers.{l}"
        hidden.append(h)
        h = h + 0.5 * ffn(h, f"{p}.ffn1")
        h = h + attention(h, p, rotary_inv_freq(sd, l))
        h = h + conv_module(h, p)
        h = ln(h + 0.5 * ffn(h, f"{p}.ffn2"), f"{p}.final_layer_norm")
    if cfg.layer_norm_first:
        h = ln(h, "encoder.layer_norm")
    hidden.append(h)
    return hidden


def conformer_forward(
    wavs: Sequence[torch.Tensor], sd: Dict[str, torch.Tensor], cfg, max_len: Optional[int] = None
) -> Tuple[List[torch.Tensor], Optional[torch.Tensor]]:
    """hidden_states (NL+1 tensors [B, T, D]) and the frame padding mask: Wav2Vec2Model.forward's front end
    (wav2vec2_model.py:2638-2684, the same steps as upstream_oracle.upstream_forward up to the masked projection) and
    the Conformer encoder above."""
    sd = {k: v.float() for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point()}
    wavs = [w.float() for w in wavs]
    lens = [len(w) for w in wavs]
    x = O.pad_waveforms(wavs, cfg.normalize, max_len)
    sample_mask = O.sample_padding_mask(lens, x.size(1))
    feats = O.conv_feature_extractor(x, sd, cfg.extractor_mode, cfg.conv_bias).transpose(1, 2)
    T = feats.size(1)
    feats = F.layer_norm(feats, (feats.size(-1),), sd["layer_norm.weight"], sd["layer_norm.bias"], 1e-5)
    pad = O.frame_padding_mask_conv_length(sample_mask, T)
    h = F.linear(feats, sd["post_extract_proj.weight"], sd["post_extract_proj.bias"])
    if pad is not None:
        h = h.masked_fill(pad.unsqueeze(-1), 0.0)
    return conformer_encoder(h, sd, cfg, pad), pad
