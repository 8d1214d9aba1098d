"""Architecture descriptions of the wav2vec 2.0 / HuBERT / WavLM upstreams served by the H100 path.

Field values are those of the public checkpoints; names follow the reference's
``HubertConfig`` (s3prl/upstream/hubert/hubert_model.py:76-278), ``Wav2Vec2Config``
(s3prl/upstream/wav2vec2/wav2vec2_model.py:2103-2350) and ``WavLMConfig`` (s3prl/upstream/wavlm/WavLM.py:162-245).
"""
from __future__ import annotations

from dataclasses import dataclass, replace
from typing import Dict

CONV_LAYERS = [(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2
DOWNSAMPLE_RATE = 320


@dataclass(frozen=True)
class ArchConfig:
    family: str  # "hubert" | "wav2vec2" | "wavlm" | "distiller" | "data2vec"
    extractor_mode: str = "default"  # "default" (GroupNorm after conv 0) | "layer_norm"
    conv_bias: bool = False
    layer_norm_first: bool = False
    normalize: bool = False  # task_cfg.normalize: per-utterance waveform layer_norm
    encoder_layers: int = 12
    encoder_embed_dim: int = 768
    encoder_ffn_embed_dim: int = 3072
    encoder_attention_heads: int = 12
    conv_pos: int = 128
    conv_pos_groups: int = 16
    # data2vec (Wav2Vec2Config.pos_conv_depth, wav2vec2_model.py:2303-2306, 2995-3026): > 1 replaces the weight-normed
    # conv by that many blocks Conv1d(k = max(3, conv_pos // depth)) -> LayerNorm(no affine) -> GELU
    pos_conv_depth: int = 1
    # WavLM
    relative_position_embedding: bool = False
    num_buckets: int = 320
    max_distance: int = 800
    gru_rel_pos: bool = False
    # Distiller (DistilHuBERT, s3prl/upstream/distiller/model.py:17-79): no LayerNorm(512) in front of
    # post_extract_proj, and `pred_heads` prediction heads (Linear -> GELU -> SplitLinear) on the encoder output
    feature_layer_norm: bool = True
    pred_heads: int = 0
    # wav2vec 2.0 Conformer (Wav2Vec2Config.layer_type / attn_type / pos_enc_type / depthwise_conv_kernel_size,
    # wav2vec2_model.py:2448, 3132-3211): ConformerEncoderLayer instead of the transformer layer, no pos_conv. Served:
    # attn_type "espnet" with rotary position encoding ("rope") only.
    layer_type: str = "transformer"  # "transformer" | "conformer"
    pos_enc_type: str = "abs"  # "abs" | "rope" | "rel_pos"
    attn_type: str = ""  # "" (fairseq MultiheadAttention) | "espnet"
    depthwise_conv_kernel_size: int = 31
    # What feeds post_extract_proj: "conv" = the waveform conv stack + LayerNorm(512); "fbank" = DeCoAR 2.0's kaldi
    # fbank (hamming window) + per-utterance CMVN + every second frame (s3prl/upstream/decoar2/audio.py:41-86)
    frontend: str = "conv"

    @property
    def family_id(self) -> int:
        # data2vec's forward builds its frame mask the wav2vec 2.0 way (data2vec_model.py:455-476)
        return {"hubert": 0, "wav2vec2": 1, "wavlm": 2, "distiller": 3, "data2vec": 1}[self.family]

    @property
    def pos_conv_kernel(self) -> int:
        """Taps of one positional conv (wav2vec2_model.py:2996-2998)."""
        return max(3, self.conv_pos // self.pos_conv_depth) if self.pos_conv_depth > 1 else self.conv_pos

    @property
    def conformer(self) -> bool:
        return self.layer_type == "conformer"

    @property
    def num_outputs(self) -> int:
        """Entries of ``hidden_states``: NL+1, or feat_final + NL layer outputs + prediction heads for the distiller."""
        return self.encoder_layers + 1 + self.pred_heads


_BASE = ArchConfig(family="hubert")
_LARGE = dict(encoder_layers=24, encoder_embed_dim=1024, encoder_ffn_embed_dim=4096, encoder_attention_heads=16)
_LL60K = dict(extractor_mode="layer_norm", conv_bias=True, layer_norm_first=True, normalize=True, **_LARGE)
# WavLM-Large / UniSpeech-SAT-Large: WavLMConfig's default conv_bias=False (WavLM.py:174) with extractor_mode
# "layer_norm". (A real checkpoint loaded through *_local carries its own cfg; this table only shapes the fabricated
# checkpoints, and the two variants give golden coverage of layer_norm with and without conv bias.)
_WAVLM_LARGE = dict(_LL60K, conv_bias=False)
_WAVLM = dict(family="wavlm", relative_position_embedding=True, gru_rel_pos=True)

ARCHS: Dict[str, ArchConfig] = {
    # HuBERT (s3prl/upstream/hubert/hubconf.py:85-108)
    "hubert_base": _BASE,
    "hubert_large_ll60k": replace(_BASE, **_LL60K),
    # wav2vec 2.0 (s3prl/upstream/wav2vec2/hubconf.py:83-120)
    "wav2vec2_base_960": replace(_BASE, family="wav2vec2"),
    "wav2vec2_large_960": replace(_BASE, family="wav2vec2", **_LARGE),
    "wav2vec2_large_ll60k": replace(_BASE, family="wav2vec2", **_LL60K),
    # WavLM (s3prl/upstream/wavlm/hubconf.py:38-78)
    "wavlm_base": replace(_BASE, **_WAVLM),
    "wavlm_base_plus": replace(_BASE, **_WAVLM),
    "wavlm_large": replace(_BASE, **_WAVLM, **_WAVLM_LARGE),
    # UniSpeech-SAT runs the WavLM model class without relative position bias
    # (s3prl/upstream/unispeech_sat/expert.py:20,37-38; hubconf.py:47-82)
    "unispeech_sat_base": replace(_BASE, family="wavlm"),
    "unispeech_sat_base_plus": replace(_BASE, family="wavlm"),
    "unispeech_sat_large": replace(_BASE, family="wavlm", **_WAVLM_LARGE),
}
# DistilHuBERT (s3prl/upstream/distiller/hubconf.py:31-48; config of distilhubert_ls960_4-8-12: 2 layers, heads for
# teacher layers 4 / 8 / 12)
ARCHS["distilhubert_base"] = ArchConfig(family="distiller", encoder_layers=2, feature_layer_norm=False, pred_heads=3)
ARCHS["distilhubert"] = ARCHS["distilhubert_base"]

# data2vec audio (s3prl/upstream/data2vec/hubconf.py:25-52; fairseq examples/data2vec base_librispeech / large_vox:
# extractor_mode layer_norm, post-LN encoder, normalize, pos_conv_depth 5 with conv_pos 95 -> five k=19 blocks)
_DATA2VEC = dict(family="data2vec", extractor_mode="layer_norm", normalize=True, conv_pos=95, pos_conv_depth=5)
ARCHS["data2vec_base_960"] = replace(_BASE, **_DATA2VEC)
ARCHS["data2vec_large_ll60k"] = replace(_BASE, **_DATA2VEC, **_LARGE)

# Same-skeleton relatives: identical architecture, different pre-training data (only the checkpoint differs).
for _alias, _arch in {
    # s3prl/upstream/wav2vec2/hubconf.py:123-160
    "wav2vec2_large_lv60_cv_swbd_fsh": "wav2vec2_large_ll60k",
    "xlsr_53": "wav2vec2_large_ll60k",
    "xls_r_300m": "wav2vec2_large_ll60k",
    # s3prl/upstream/hubert/hubconf.py:111-156
    "hubert_base_robust_mgr": "hubert_base",
    "mhubert_base_vp_en_es_fr_it3": "hubert_base",
    "contentvec": "hubert_base",
    "contentvec_km100": "hubert_base",
    "contentvec_km500": "hubert_base",
    "ms_hubert": "hubert_base",
}.items():
    ARCHS[_alias] = ARCHS[_arch]
# wav2vec 2.0 Conformer with rotary attention (s3prl/upstream/wav2vec2/hubconf.py wav2vec2_conformer_rope). The values
# are those of fairseq's Conformer-large LibriLight pre-training config as far as they are public; they were NOT checked
# against the released checkpoint (not reachable offline). They only shape the fabricated checkpoint: a real checkpoint
# loaded through wav2vec2_local carries its own cfg (arch_from_reference_cfg).
ARCHS["wav2vec2_conformer_rope"] = replace(
    _BASE, family="wav2vec2", **_LL60K, layer_type="conformer", pos_enc_type="rope", attn_type="espnet"
)
# XLS-R 1B and 2B (s3prl/upstream/wav2vec2/hubconf.py xls_r_1b / xls_r_2b: wav2vec2_custom on the released files):
# the LibriLight-large options with 48 layers and 80- / 120-wide heads. The values are those of fairseq's public XLS-R
# configs; they were NOT checked against the released checkpoints (not reachable offline). A real checkpoint loaded
# through wav2vec2_local / wav2vec2_custom carries its own cfg (arch_from_reference_cfg); this table shapes fabricated
# checkpoints. It is kept apart from ARCHS, whose every key is a hub entry: these models are reached through
# wav2vec2_local / wav2vec2_custom / wav2vec2_url, or UpstreamExpert(arch=XLS_R[...]).
XLS_R: Dict[str, ArchConfig] = {
    "xls_r_1b": replace(_BASE, family="wav2vec2", **dict(_LL60K, encoder_layers=48, encoder_embed_dim=1280,
                                                         encoder_ffn_embed_dim=5120, encoder_attention_heads=16)),
    "xls_r_2b": replace(_BASE, family="wav2vec2", **dict(_LL60K, encoder_layers=48, encoder_embed_dim=1920,
                                                         encoder_ffn_embed_dim=7680, encoder_attention_heads=16)),
}
ALIASES = {
    "hubert": "hubert_base",
    "hubert_large": "hubert_large_ll60k",
    "wav2vec2": "wav2vec2_base_960",
    "wav2vec2_large": "wav2vec2_large_960",
    "wavlm": "wavlm_base",
    "unispeech_sat": "unispeech_sat_base_plus",
    "data2vec": "data2vec_base_960",
}


def get_arch(name: str) -> ArchConfig:
    name = ALIASES.get(name, name)
    if name not in ARCHS:
        raise KeyError(f"unknown upstream architecture '{name}'; known: {sorted(ARCHS) + sorted(ALIASES)}")
    return ARCHS[name]


def arch_from_reference_cfg(family: str, model_cfg: dict, task_cfg: dict | None = None) -> ArchConfig:
    """Build an ArchConfig from the ``model_cfg`` / ``task_cfg`` (or WavLM ``cfg``) dict of a converted
    reference checkpoint (s3prl/upstream/hubert/convert.py:37-56, wavlm/expert.py:37-40)."""
    g = model_cfg.get
    normalize = bool((task_cfg or {}).get("normalize", g("normalize", False)))
    layers = g("conv_feature_layers", None)
    if layers is not None and list(eval(layers) if isinstance(layers, str) else layers) != CONV_LAYERS:
        raise ValueError(f"unsupported conv_feature_layers: {layers}")
    if family == "distiller":  # DistillerConfig (distiller/model.py:17-79)
        if g("task_emb_type", "expand-last") != "expand-last" or g("out_layer_type", "expand-last") != "expand-last":
            raise ValueError("only the expand-last Distiller (DistilHuBERT) is supported")
        if g("attention_type", "original") != "original" or int(g("final_dim", 768)) != int(g("encoder_embed_dim", 768)):
            raise ValueError("unsupported Distiller variant (attention_type / final_dim)")
        layers = g("extractor_conv_feature_layers", None)
        if layers is not None and list(eval(layers) if isinstance(layers, str) else layers) != CONV_LAYERS:
            raise ValueError(f"unsupported conv_feature_layers: {layers}")
        return ArchConfig(
            family="distiller",
            extractor_mode=g("extractor_mode", "default"),
            layer_norm_first=bool(g("layer_norm_first", False)),
            encoder_layers=int(g("encoder_layers", 1)),
            encoder_embed_dim=int(g("encoder_embed_dim", 768)),
            encoder_ffn_embed_dim=int(g("encoder_ffn_embed_dim", 3072)),
            encoder_attention_heads=int(g("encoder_attention_heads", 12)),
            conv_pos=int(g("conv_pos", 128)),
            conv_pos_groups=int(g("conv_pos_groups", 16)),
            feature_layer_norm=False,
            pred_heads=int(g("n_tasks", 12)),
        )
    layer_type = g("layer_type", "transformer") or "transformer"
    conformer = {}
    if layer_type == "conformer":
        pos_enc, attn, k = g("pos_enc_type", "abs"), g("attn_type", ""), int(g("depthwise_conv_kernel_size", 31))
        if family != "wav2vec2":
            raise ValueError(f"a Conformer encoder is a wav2vec2 model, not family '{family}'")
        if pos_enc == "rel_pos":
            raise ValueError("Conformer with pos_enc_type 'rel_pos' (Transformer-XL attention) is not supported; "
                             "only the rotary variant ('rope') is")
        if pos_enc != "rope":
            raise ValueError(f"Conformer with pos_enc_type {pos_enc!r} is not supported; only 'rope' is")
        if attn != "espnet":
            raise ValueError(f"Conformer with attn_type {attn!r} is not supported; only 'espnet' is")
        if k % 2 == 0 or not 1 <= k <= 63:
            raise ValueError(f"depthwise_conv_kernel_size {k}: must be odd and at most 63")
        conformer = dict(layer_type="conformer", pos_enc_type=pos_enc, attn_type=attn, depthwise_conv_kernel_size=k)
    elif layer_type != "transformer":
        raise ValueError(f"unsupported layer_type {layer_type!r}")
    return ArchConfig(
        family=family,
        extractor_mode=g("extractor_mode", "default"),
        conv_bias=bool(g("conv_bias", False)),
        layer_norm_first=bool(g("layer_norm_first", False)),
        normalize=normalize,
        encoder_layers=int(g("encoder_layers", 12)),
        encoder_embed_dim=int(g("encoder_embed_dim", 768)),
        encoder_ffn_embed_dim=int(g("encoder_ffn_embed_dim", 3072)),
        encoder_attention_heads=int(g("encoder_attention_heads", 12)),
        conv_pos=int(g("conv_pos", 128)),
        conv_pos_groups=int(g("conv_pos_groups", 16)),
        pos_conv_depth=int(g("pos_conv_depth", 1)),
        relative_position_embedding=bool(g("relative_position_embedding", False)),
        num_buckets=int(g("num_buckets", 320)),
        max_distance=int(g("max_distance", 800)),
        gru_rel_pos=bool(g("gru_rel_pos", False)),
        **conformer,
    )
