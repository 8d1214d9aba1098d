"""Weights for the upstreams: deterministic fabricated checkpoints (there is no network, so the pretrained
files the reference downloads — s3prl/upstream/hubert/hubconf.py:90-95 — are unreachable) and a reader for
the reference's converted-checkpoint formats.

State-dict keys and shapes are the reference's on-disk format, so a fabricated
state dict loads unchanged into the reference ``HubertModel`` / ``Wav2Vec2Model`` / ``WavLM`` (that is how the
golden fixtures in tests/golden are produced, see oracle/make_golden.py).
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch

from .configs import CONV_LAYERS, ArchConfig, arch_from_reference_cfg


def fabricate_state_dict(cfg: ArchConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Random weights with the initialisation *scales* of the reference constructors (kaiming conv
    wav2vec2_model.py:2880, pos_conv normal :2946-2948, BERT-style linears) but with every affine / bias
    parameter perturbed away from its (1, 0) default so that indexing and bias bugs cannot hide.
    Deterministic in (cfg, seed) for a fixed torch version."""
    g = torch.Generator().manual_seed(seed)

    def randn(*shape, std=1.0, mean=0.0):
        return torch.randn(*shape, generator=g) * std + mean

    D, F, H = cfg.encoder_embed_dim, cfg.encoder_ffn_embed_dim, cfg.encoder_attention_heads
    sd: Dict[str, torch.Tensor] = {}
    in_d = 1
    for i, (dim, k, _s) in enumerate(CONV_LAYERS):
        p = f"feature_extractor.conv_layers.{i}"
        sd[f"{p}.0.weight"] = randn(dim, in_d, k, std=math.sqrt(2.0 / (in_d * k)))
        if cfg.conv_bias:
            sd[f"{p}.0.bias"] = randn(dim, std=0.05)
        if cfg.extractor_mode == "layer_norm":
            sd[f"{p}.2.1.weight"] = randn(dim, std=0.1, mean=1.0)
            sd[f"{p}.2.1.bias"] = randn(dim, std=0.1)
        elif i == 0:
            sd[f"{p}.2.weight"] = randn(dim, std=0.1, mean=1.0)
            sd[f"{p}.2.bias"] = randn(dim, std=0.1)
        in_d = dim
    if cfg.feature_layer_norm:
        sd["layer_norm.weight"] = randn(in_d, std=0.1, mean=1.0)
        sd["layer_norm.bias"] = randn(in_d, std=0.1)
    sd["post_extract_proj.weight"] = randn(D, in_d, std=1.0 / math.sqrt(in_d))
    sd["post_extract_proj.bias"] = randn(D, std=0.05)
    cpg = D // cfg.conv_pos_groups
    if cfg.conformer:
        return _fabricate_conformer(cfg, sd, randn, g)
    if cfg.pos_conv_depth > 1:
        # data2vec: plain Conv1d blocks (make_conv_block, wav2vec2_model.py:3000-3022; every block is followed by a LayerNorm, so the scale is immaterial)
        k = cfg.pos_conv_kernel
        for i in range(cfg.pos_conv_depth):
            sd[f"encoder.pos_conv.{i}.0.weight"] = randn(D, cpg, k, std=1.0 / math.sqrt(cpg * k))
            sd[f"encoder.pos_conv.{i}.0.bias"] = randn(D, std=0.05)
    else:
        # pos_conv with weight_norm(dim=2): g has one entry per kernel tap
        v = randn(D, cpg, cfg.conv_pos, std=math.sqrt(4.0 / (cfg.conv_pos * D)))
        sd["encoder.pos_conv.0.weight_v"] = v
        sd["encoder.pos_conv.0.weight_g"] = v.norm(dim=(0, 1), keepdim=True) * randn(1, 1, cfg.conv_pos, std=0.1, mean=1.0)
        sd["encoder.pos_conv.0.bias"] = randn(D, std=0.05)
    sd["encoder.layer_norm.weight"] = randn(D, std=0.1, mean=1.0)
    sd["encoder.layer_norm.bias"] = randn(D, std=0.1)
    for l in range(cfg.encoder_layers):
        p = f"encoder.layers.{l}"
        for name in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[f"{p}.self_attn.{name}.weight"] = randn(D, D, std=1.0 / math.sqrt(D))
            sd[f"{p}.self_attn.{name}.bias"] = randn(D, std=0.05)
        sd[f"{p}.self_attn_layer_norm.weight"] = randn(D, std=0.1, mean=1.0)
        sd[f"{p}.self_attn_layer_norm.bias"] = randn(D, std=0.1)
        sd[f"{p}.fc1.weight"] = randn(F, D, std=1.0 / math.sqrt(D))
        sd[f"{p}.fc1.bias"] = randn(F, std=0.05)
        sd[f"{p}.fc2.weight"] = randn(D, F, std=1.0 / math.sqrt(F))
        sd[f"{p}.fc2.bias"] = randn(D, std=0.05)
        sd[f"{p}.final_layer_norm.weight"] = randn(D, std=0.1, mean=1.0)
        sd[f"{p}.final_layer_norm.bias"] = randn(D, std=0.1)
        if cfg.relative_position_embedding and cfg.gru_rel_pos:
            sd[f"{p}.self_attn.grep_linear.weight"] = randn(8, 64, std=0.2)
            sd[f"{p}.self_attn.grep_linear.bias"] = randn(8, std=0.2)
            sd[f"{p}.self_attn.grep_a"] = randn(1, H, 1, 1, std=0.3, mean=1.0)
    if cfg.relative_position_embedding:
        sd["encoder.layers.0.self_attn.relative_attention_bias.weight"] = randn(cfg.num_buckets, H, std=0.5)
    if cfg.pred_heads > 0:  # Distiller output_layer = Linear -> GELU -> SplitLinear (distiller/model.py:150-160, module.py:55-90)
        N = cfg.pred_heads
        sd["output_layer.0.weight"] = randn(N * D, D, std=1.0 / math.sqrt(D))
        sd["output_layer.0.bias"] = randn(N * D, std=0.05)
        sd["output_layer.2.weight"] = randn(N, D, D, std=1.0 / math.sqrt(D))  # [task][in][out]
        sd["output_layer.2.bias"] = randn(1, 1, N, D, std=0.05)
    return sd


def _fabricate_conformer(cfg: ArchConfig, sd: Dict[str, torch.Tensor], randn, g) -> Dict[str, torch.Tensor]:
    """The encoder of a rotary Conformer (ConformerEncoder / ConformerEncoderLayer, wav2vec2_model.py:441-578,
    3132-3211): no pos_conv; per layer two half-step FFNs, rotary attention, the convolution module and the final
    LayerNorm. BatchNorm statistics are non-trivial (running_var in [0.5, 1.5], non-zero running_mean) so that the
    folding of eval-mode BatchNorm into the depthwise taps is exercised. The rotary inv_freq buffer is left to the
    model (it is not a learned parameter)."""
    D, F, k = cfg.encoder_embed_dim, cfg.encoder_ffn_embed_dim, cfg.depthwise_conv_kernel_size

    def ln(name):
        sd[f"{name}.weight"] = randn(D, std=0.1, mean=1.0)
        sd[f"{name}.bias"] = randn(D, std=0.1)

    ln("encoder.layer_norm")
    for l in range(cfg.encoder_layers):
        p = f"encoder.layers.{l}"
        for f in ("ffn1", "ffn2"):
            ln(f"{p}.{f}.layer_norm")
            sd[f"{p}.{f}.w_1.weight"] = randn(F, D, std=1.0 / math.sqrt(D))
            sd[f"{p}.{f}.w_1.bias"] = randn(F, std=0.05)
            sd[f"{p}.{f}.w_2.weight"] = randn(D, F, std=1.0 / math.sqrt(F))
            sd[f"{p}.{f}.w_2.bias"] = randn(D, std=0.05)
        ln(f"{p}.self_attn_layer_norm")
        for name in ("linear_q", "linear_k", "linear_v", "linear_out"):
            sd[f"{p}.self_attn.{name}.weight"] = randn(D, D, std=1.0 / math.sqrt(D))
            sd[f"{p}.self_attn.{name}.bias"] = randn(D, std=0.05)
        c = f"{p}.conv_module"
        ln(f"{c}.layer_norm")
        sd[f"{c}.pointwise_conv1.weight"] = randn(2 * D, D, 1, std=1.0 / math.sqrt(D))
        sd[f"{c}.depthwise_conv.weight"] = randn(D, 1, k, std=1.0 / math.sqrt(k))
        sd[f"{c}.batch_norm.weight"] = randn(D, std=0.1, mean=1.0)
        sd[f"{c}.batch_norm.bias"] = randn(D, std=0.1)
        sd[f"{c}.batch_norm.running_mean"] = randn(D, std=0.1)
        sd[f"{c}.batch_norm.running_var"] = torch.rand(D, generator=g) + 0.5
        sd[f"{c}.pointwise_conv2.weight"] = randn(D, D, 1, std=1.0 / math.sqrt(D))
        ln(f"{p}.final_layer_norm")
    return sd


def load_reference_checkpoint(path: str, family: str) -> Tuple[ArchConfig, Dict[str, torch.Tensor]]:
    """Read a converted reference checkpoint: ``{"task_cfg","model_cfg","model_weight"[,"dictionaries_symbols"]}``
    (s3prl/upstream/hubert/convert.py:37-56, wav2vec2/convert.py:26-39, data2vec/convert.py:31-52) or WavLM's ``{"cfg","model"}``
    (s3prl/upstream/wavlm/expert.py:37-40)."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if "model_weight" in state:
        for key in ("task_cfg", "model_cfg", "model_weight"):
            if key not in state:
                raise ValueError(f"{path} is not a valid checkpoint since the required key: {key} is missing")
        cfg = arch_from_reference_cfg(family, dict(state["model_cfg"]), dict(state["task_cfg"]))
        weights = state["model_weight"]
        if family == "data2vec":  # the EMA teacher travels in the checkpoint and is dropped (data2vec/convert.py:48-49)
            weights = {k: v for k, v in weights.items() if k != "_ema"}
        return cfg, weights
    if "cfg" in state and "model" in state:
        return arch_from_reference_cfg("wavlm", dict(state["cfg"])), state["model"]
    if "Config" in state and "Distiller" in state:  # distiller/builder.py:41-47,129-131
        return arch_from_reference_cfg("distiller", dict(state["Config"]["distiller"])), state["Distiller"]
    raise ValueError(f"{path}: unrecognised checkpoint layout (keys: {sorted(state)[:8]})")
