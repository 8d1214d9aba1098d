"""Checkpoint formats adjacent to the hot path.

Three on-disk layouts reach the upstream forward in the reference:

* the reference's **converted** checkpoints (``{"task_cfg", "model_cfg", "model_weight"[, "dictionaries_symbols"]}``
  for HuBERT / wav2vec 2.0 — s3prl/upstream/hubert/convert.py:37-56, wav2vec2/convert.py:26-39 — and WavLM's
  ``{"cfg", "model"}`` — wavlm/expert.py:37-40). ``weights.load_reference_checkpoint`` reads them;
  ``save_converted_checkpoint`` writes them (what the ``*_local`` hub entries take).
* **fairseq** training checkpoints (``{"cfg": {"task", "model"}, "model", "task_state"}``), which the reference
  converts with ``load_and_convert_fairseq_ckpt`` (hubert/convert.py:17-34, wav2vec2/convert.py:14-23 over
  upstream/utils.py:14-29). ``convert_fairseq_state`` is the same dictionary surgery on an already un-pickled state
  (un-pickling needs fairseq importable, exactly as in the reference; nothing here imports it).
* **HuggingFace transformers** state dicts (``HubertModel`` / ``Wav2Vec2Model`` / ``WavLMModel``; the reference's
  ``hf_hubert`` / ``hf_wav2vec2`` experts run them directly, hf_hubert/expert.py:12-41). ``hf_to_fairseq_state_dict``
  renames them to the fairseq keys the native model takes, which also gives a second, independent CPU oracle
  (tests/test_host_cpu.py runs transformers' own forward against oracle/upstream_oracle.py on the mapped weights).
"""
from __future__ import annotations

import re
from pathlib import Path
from typing import Dict, Mapping, Optional, Tuple

import torch

from .configs import CONV_LAYERS, ArchConfig


# ------------------------------------------------------------------------------------------------
# converted checkpoints
# ------------------------------------------------------------------------------------------------
def reference_model_cfg(cfg: ArchConfig) -> Dict:
    """The ``model_cfg`` fields the reference constructors read for the extraction forward
    (HubertConfig hubert_model.py:76-278, Wav2Vec2Config wav2vec2_model.py:2103-2350, WavLMConfig WavLM.py:162-245)."""
    d = dict(
        extractor_mode=cfg.extractor_mode,
        conv_bias=cfg.conv_bias,
        layer_norm_first=cfg.layer_norm_first,
        encoder_layers=cfg.encoder_layers,
        encoder_embed_dim=cfg.encoder_embed_dim,
        encoder_ffn_embed_dim=cfg.encoder_ffn_embed_dim,
        encoder_attention_heads=cfg.encoder_attention_heads,
        conv_feature_layers=str(CONV_LAYERS),
        conv_pos=cfg.conv_pos,
        conv_pos_groups=cfg.conv_pos_groups,
        activation_fn="gelu",
    )
    if cfg.pos_conv_depth > 1:
        d.update(pos_conv_depth=cfg.pos_conv_depth)
    if cfg.conformer:
        d.update(layer_type="conformer", pos_enc_type=cfg.pos_enc_type, attn_type=cfg.attn_type,
                 depthwise_conv_kernel_size=cfg.depthwise_conv_kernel_size)
    if cfg.family == "wavlm":
        d.update(
            normalize=cfg.normalize,
            relative_position_embedding=cfg.relative_position_embedding,
            num_buckets=cfg.num_buckets,
            max_distance=cfg.max_distance,
            gru_rel_pos=cfg.gru_rel_pos,
        )
    return d


def distiller_config(cfg: ArchConfig) -> Dict:
    """The ``Config["distiller"]`` dict of a Distiller checkpoint (DistillerConfig, distiller/model.py:17-79)."""
    n = cfg.pred_heads
    return dict(
        extractor_mode=cfg.extractor_mode,
        extractor_conv_feature_layers=str(CONV_LAYERS),
        conv_pos=cfg.conv_pos,
        conv_pos_groups=cfg.conv_pos_groups,
        encoder_layers=cfg.encoder_layers,
        encoder_embed_dim=cfg.encoder_embed_dim,
        encoder_ffn_embed_dim=cfg.encoder_ffn_embed_dim,
        encoder_attention_heads=cfg.encoder_attention_heads,
        activation_fn="gelu",
        layer_norm_first=cfg.layer_norm_first,
        attention_type="original",
        final_dim=cfg.encoder_embed_dim,
        out_layer_type="expand-last",
        n_tasks=n,
        task_emb_type="expand-last",
        pred_layer_id=[4 * (i + 1) for i in range(n)],
    )


def converted_checkpoint(cfg: ArchConfig, state_dict: Mapping[str, torch.Tensor]) -> Dict:
    """In-memory converted checkpoint of ``cfg.family``'s layout."""
    weights = {k: v.detach().cpu() for k, v in state_dict.items()}
    if cfg.family == "distiller":  # distiller/builder.py:41-47,129-131
        return {"Config": {"distiller": distiller_config(cfg)}, "Distiller": weights}
    model_cfg = reference_model_cfg(cfg)
    if cfg.family == "wavlm":
        return {"cfg": model_cfg, "model": weights}
    out = {
        "task_cfg": {"normalize": cfg.normalize, "sample_rate": 16000},
        "model_cfg": model_cfg,
        "model_weight": weights,
    }
    if cfg.family == "data2vec":  # the reference deletes this key unconditionally (data2vec/convert.py:48-49)
        out["model_weight"]["_ema"] = {}
    if cfg.family == "hubert":
        out["task_cfg"]["label_rate"] = 50.0
        out["model_cfg"]["label_rate"] = 50.0
        out["dictionaries_symbols"] = [[str(i) for i in range(504)]]
    return out


def save_converted_checkpoint(path, cfg: ArchConfig, state_dict: Mapping[str, torch.Tensor]) -> None:
    Path(path).parent.mkdir(parents=True, exist_ok=True)
    torch.save(converted_checkpoint(cfg, state_dict), str(path))


# ------------------------------------------------------------------------------------------------
# fairseq -> converted
# ------------------------------------------------------------------------------------------------
def _to_container(cfg):
    """OmegaConf -> plain dict when the checkpoint carries an OmegaConf (upstream/utils.py:26)."""
    if isinstance(cfg, dict):
        return {k: _to_container(v) for k, v in cfg.items()}
    try:
        from omegaconf import OmegaConf  # optional

        if OmegaConf.is_config(cfg):
            return OmegaConf.to_container(cfg)
    except Exception:
        pass
    return cfg


def convert_fairseq_state(state: Mapping, family: str) -> Dict:
    """``load_and_convert_fairseq_ckpt`` without the I/O: fairseq state -> converted checkpoint dict.

    hubert  : task_cfg, model_cfg, model_weight, dictionaries_symbols (hubert/convert.py:17-34)
    wav2vec2: task_cfg, model_cfg, model_weight                       (wav2vec2/convert.py:14-23)
    """
    if "cfg" not in state or "model" not in state:
        raise ValueError("not a fairseq checkpoint: 'cfg' / 'model' missing")
    cfg = _to_container(state["cfg"])
    if not isinstance(cfg, dict) or "task" not in cfg or "model" not in cfg:
        raise ValueError("fairseq cfg must hold 'task' and 'model' sections")
    out = {"task_cfg": cfg["task"], "model_cfg": cfg["model"], "model_weight": state["model"]}
    if family == "hubert":
        dicts = (state.get("task_state") or {}).get("dictionaries")
        if dicts is None:
            raise ValueError("HuBERT fairseq checkpoint without task_state.dictionaries")
        out["dictionaries_symbols"] = [list(getattr(d, "symbols", d)) for d in dicts]
    elif family != "wav2vec2":
        raise ValueError(f"no fairseq converter for family '{family}' (WavLM ships {{'cfg','model'}} already)")
    return out


def convert_fairseq_checkpoint(fairseq_path: str, output_path: str, family: str) -> None:
    """File-to-file form. Un-pickling a fairseq checkpoint needs ``fairseq`` importable, like the reference."""
    state = torch.load(fairseq_path, map_location="cpu", weights_only=False)
    Path(output_path).parent.mkdir(parents=True, exist_ok=True)
    torch.save(convert_fairseq_state(state, family), output_path)


# ------------------------------------------------------------------------------------------------
# HuggingFace transformers <-> fairseq parameter names
# ------------------------------------------------------------------------------------------------
_HF_LAYER = [
    ("attention.q_proj", "self_attn.q_proj"),
    ("attention.k_proj", "self_attn.k_proj"),
    ("attention.v_proj", "self_attn.v_proj"),
    ("attention.out_proj", "self_attn.out_proj"),
    ("attention.gru_rel_pos_linear", "self_attn.grep_linear"),
    ("attention.gru_rel_pos_const", "self_attn.grep_a"),
    ("attention.rel_attn_embed", "self_attn.relative_attention_bias"),
    ("layer_norm", "self_attn_layer_norm"),
    ("feed_forward.intermediate_dense", "fc1"),
    ("feed_forward.output_dense", "fc2"),
    ("final_layer_norm", "final_layer_norm"),
]


def hf_to_fairseq_key(key: str, extractor_mode: str) -> Optional[str]:
    """fairseq name of a ``transformers`` Hubert/Wav2Vec2/WavLM *base model* parameter, or None for parameters the
    extraction forward does not use (masked_spec_embed, adapter / head weights)."""
    key = re.sub(r"^(hubert|wav2vec2|wavlm|data2vec_audio)\.", "", key)
    m = re.match(r"feature_extractor\.conv_layers\.(\d+)\.(conv|layer_norm)\.(weight|bias)$", key)
    if m:
        i, kind, wb = m.groups()
        if kind == "conv":
            return f"feature_extractor.conv_layers.{i}.0.{wb}"
        # "group" models: GroupNorm after conv 0 at index 2; "layer" models: Sequential(Transpose, LN, Transpose) -> 2.1
        return f"feature_extractor.conv_layers.{i}.2.1.{wb}" if extractor_mode == "layer_norm" else f"feature_extractor.conv_layers.{i}.2.{wb}"
    m = re.match(r"feature_projection\.(layer_norm|projection)\.(weight|bias)$", key)
    if m:
        return ("layer_norm." if m.group(1) == "layer_norm" else "post_extract_proj.") + m.group(2)
    m = re.match(r"encoder\.pos_conv_embed\.conv\.(.+)$", key)
    if m:
        tail = {
            "bias": "bias",
            "weight_g": "weight_g",
            "weight_v": "weight_v",
            "parametrizations.weight.original0": "weight_g",  # torch.nn.utils.parametrizations.weight_norm
            "parametrizations.weight.original1": "weight_v",
        }.get(m.group(1))
        return None if tail is None else f"encoder.pos_conv.0.{tail}"
    m = re.match(r"encoder\.pos_conv_embed\.layers\.(\d+)\.conv\.(weight|bias)$", key)
    if m:  # Data2VecAudio: plain conv blocks (modeling_data2vec_audio.py Data2VecAudioPositionalConvLayer)
        return f"encoder.pos_conv.{m.group(1)}.0.{m.group(2)}"
    m = re.match(r"encoder\.layer_norm\.(weight|bias)$", key)
    if m:
        return f"encoder.layer_norm.{m.group(1)}"
    m = re.match(r"encoder\.layers\.(\d+)\.(.+?)(?:\.(weight|bias))?$", key)
    if m:
        l, mid, wb = m.groups()
        for hf, fs in _HF_LAYER:
            if mid == hf:
                return f"encoder.layers.{l}.{fs}" + (f".{wb}" if wb else "")
    return None


def hf_to_fairseq_state_dict(hf_state: Mapping[str, torch.Tensor], extractor_mode: str) -> Dict[str, torch.Tensor]:
    """Rename a ``transformers`` state dict to the reference's (fairseq) keys; tensors are shared, not copied.
    WavLM's ``gru_rel_pos_const`` [1, H, 1, 1] and relative-position embedding keep their shapes."""
    out: Dict[str, torch.Tensor] = {}
    for k, v in hf_state.items():
        fk = hf_to_fairseq_key(k, extractor_mode)
        if fk is not None:
            out[fk] = v
    return out


def arch_from_hf_config(hf_cfg) -> ArchConfig:
    """ArchConfig of a ``transformers`` HubertConfig / Wav2Vec2Config / WavLMConfig (base-model fields)."""
    model_type = getattr(hf_cfg, "model_type", "hubert")
    family = {"hubert": "hubert", "wav2vec2": "wav2vec2", "wavlm": "wavlm", "unispeech-sat": "wavlm",
              "data2vec-audio": "data2vec"}.get(model_type)
    if family is None:
        raise ValueError(f"unsupported transformers model_type '{model_type}'")
    convs = list(zip(hf_cfg.conv_dim, hf_cfg.conv_kernel, hf_cfg.conv_stride))
    if [tuple(c) for c in convs] != CONV_LAYERS:
        raise ValueError(f"unsupported conv feature extractor: {convs}")
    if family == "data2vec":
        # Data2VecAudioConfig has neither feat_extract_norm nor do_stable_layer_norm: always "layer" + post-LN, and
        # num_conv_pos_embeddings counts the conv blocks of conv_pos_kernel_size taps each
        depth, k = int(hf_cfg.num_conv_pos_embeddings), int(hf_cfg.conv_pos_kernel_size)
        return ArchConfig(
            family="data2vec",
            extractor_mode="layer_norm",
            conv_bias=bool(hf_cfg.conv_bias),
            normalize=True,
            encoder_layers=hf_cfg.num_hidden_layers,
            encoder_embed_dim=hf_cfg.hidden_size,
            encoder_ffn_embed_dim=hf_cfg.intermediate_size,
            encoder_attention_heads=hf_cfg.num_attention_heads,
            conv_pos=depth * k,
            conv_pos_groups=hf_cfg.num_conv_pos_embedding_groups,
            pos_conv_depth=depth,
        )
    return ArchConfig(
        family=family,
        extractor_mode="layer_norm" if hf_cfg.feat_extract_norm == "layer" else "default",
        conv_bias=bool(hf_cfg.conv_bias),
        layer_norm_first=bool(hf_cfg.do_stable_layer_norm),
        normalize=hf_cfg.feat_extract_norm == "layer",  # the feature extractor's do_normalize of the "layer" models
        encoder_layers=hf_cfg.num_hidden_layers,
        encoder_embed_dim=hf_cfg.hidden_size,
        encoder_ffn_embed_dim=hf_cfg.intermediate_size,
        encoder_attention_heads=hf_cfg.num_attention_heads,
        conv_pos=hf_cfg.num_conv_pos_embeddings,
        conv_pos_groups=hf_cfg.num_conv_pos_embedding_groups,
        relative_position_embedding=family == "wavlm" and model_type == "wavlm",
        num_buckets=getattr(hf_cfg, "num_buckets", 320),
        max_distance=getattr(hf_cfg, "max_bucket_distance", 800),
        gru_rel_pos=family == "wavlm" and model_type == "wavlm",
    )


def load_hf_model(hf_model) -> Tuple[ArchConfig, Dict[str, torch.Tensor]]:
    """(ArchConfig, fairseq-keyed state dict) of an instantiated ``transformers`` base model — feed to
    ``UpstreamExpert(arch=..., state_dict=...)``."""
    cfg = arch_from_hf_config(hf_model.config)
    return cfg, hf_to_fairseq_state_dict(hf_model.state_dict(), cfg.extractor_mode)
