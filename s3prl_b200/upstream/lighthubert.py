"""LightHuBERT (``lighthubert``, ``lighthubert_small``, ``lighthubert_base``, ``lighthubert_stage1``,
``lighthubert_local``, ``lighthubert_url``) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/lighthubert/{expert,lighthubert}.py, modules/scaling_*.py) loads a once-for-all
supernet and serves one subnet of it: ``hubert_pruner`` checkpoints the supernet's ``subnet`` (384 channels for a
"small" supernet, 640 for "base"), ``student_hubert`` checkpoints its ``max_subnet`` (768 for "base", 512 for
"small"). Every such subnet has 12 post-LN layers of global attention with 64-wide heads and ``atten_dim ==
embed_dim``, the same in every layer. The subnet is a HuBERT encoder whose weights are cut out of the supernet's:

- q/k/v_proj rows ``[:A]``, columns ``[:E]``; out_proj rows ``[:E]``, columns ``[:A]``; post_extract_proj rows
  ``[:E]``; every LayerNorm ``[:E]``.
- fc1's rows form ``F_super / E_super`` splits of ``E_super`` rows, and the subnet takes the first
  ``F / ceil(F / E)`` rows of each of the first ``ceil(F / E)`` splits (scaling_linear.py:75-125); fc2's columns are
  cut the same way. A subnet as wide as the supernet keeps fc1 / fc2 whole.
- pos_conv is weight-normed (``dim=2``): ``weight_g * weight_v / ||weight_v||`` is formed at supernet size and only
  then cut to ``[:E, :E / 16, :]``, so its norm runs over the whole supernet ``weight_v``. The cut ``weight_v`` is
  sent with a ``weight_g`` rescaled by ``||cut|| / ||supernet||`` per tap, which the library's own fold turns back into
  the reference's weight.

The forward is the reference's: per-utterance ``F.layer_norm`` of the waveform, the conv stack, LayerNorm(512),
post_extract_proj; that output, with HuBERT's padded frames zeroed (the encoder's in-place ``index_put``), is hidden
state 0, followed by the 12 layer outputs. The library runs it as a HuBERT model with ``proj_hidden0`` set. Padding T
to an even length (``required_seq_len_multiple=2``) adds masked keys whose rows are trimmed, so it changes nothing
and is not reproduced.

Checkpoint: the reference's ``{"cfg": {"model": {...}}, "model": state_dict}`` file. Keys the cfg omits take
``LightHuBERTConfig``'s defaults. Refused with ``ValueError`` naming the field: another ``_name``, ``encoder_layers``
other than 12, ``layer_type`` other than "transformer", a non-standard ``conv_feature_layers``, ``pos_conv_depth``
other than 1, ``layer_norm_first``, ``activation_fn`` other than "gelu", and a supernet narrower than its subnet. A
missing supernet tensor raises ``KeyError`` naming it; the reference's ``load_state_dict(strict=False)`` would keep
random weights instead. Prediction heads, ``mask_emb`` and label embeddings are ignored. The released files are not
reachable offline: their supernets were not checked (the fabricated ones are 768 wide, 12 heads, FFN 3072).
"""
from __future__ import annotations

import math
from dataclasses import replace
from typing import Dict, List, Optional, Tuple

import torch

from .configs import ArchConfig, DOWNSAMPLE_RATE
from .expert import NativeExpert, _c_config
from .weights import fabricate_state_dict

NAMES = ("hubert_pruner", "student_hubert")
_CONV_FEATURE_LAYERS = "[(512,10,5)] + [(512,3,2)] * 4 + [(512,2,2)] * 2"

# LightHuBERTConfig's defaults (lighthubert.py:341-428) for the fields the port reads
_DEFAULTS = {"supernet_type": "base", "pos_conv_depth": 1, "extractor_mode": "layer_norm", "encoder_layers": 12,
             "encoder_embed_dim": 768, "encoder_ffn_embed_dim": 3072, "encoder_attention_heads": 12,
             "activation_fn": "gelu", "layer_type": "transformer", "layer_norm_first": False,
             "conv_feature_layers": _CONV_FEATURE_LAYERS, "conv_bias": False, "conv_pos": 128, "conv_pos_groups": 16}

# (embed_dim, heads, ffn_dim) of LightHuBERTSupernetConfig.subnet / .max_subnet (lighthubert.py:219-272)
SUBNETS = {("hubert_pruner", "small"): (384, 6, 1536), ("hubert_pruner", "base"): (640, 10, 2560),
           ("student_hubert", "small"): (512, 8, 2048), ("student_hubert", "base"): (768, 12, 3072)}

# hub name -> (_name, pruner_supernet) of the fabricated checkpoint
KINDS = {"small": ("hubert_pruner", "lighthubert_small.yaml"), "base": ("hubert_pruner", "lighthubert_base.yaml"),
         "stage1": ("student_hubert", None)}


def lighthubert_config(kind: str = "small", **over) -> dict:
    """``cfg["model"]`` of a fabricated checkpoint of ``kind`` ("small", "base" or "stage1"): a 768-wide supernet
    whose served subnet is 384, 640 or 768 wide. ``over`` replaces fields."""
    name, pruner = KINDS[kind]
    c = {"_name": name, "supernet_type": "base", "encoder_layers": 12, "encoder_embed_dim": 768,
         "encoder_ffn_embed_dim": 3072, "encoder_attention_heads": 12}
    if pruner is not None:
        c["pruner_supernet"] = pruner
    c.update(over)
    return c


def supernet_arch(cfg: dict) -> ArchConfig:
    """The supernet as a HuBERT ``ArchConfig`` (the shapes of its state dict)."""
    c = dict(_DEFAULTS, **cfg)
    return ArchConfig(family="hubert", extractor_mode=c["extractor_mode"], conv_bias=bool(c["conv_bias"]),
                      normalize=True, encoder_layers=c["encoder_layers"], encoder_embed_dim=c["encoder_embed_dim"],
                      encoder_ffn_embed_dim=c["encoder_ffn_embed_dim"],
                      encoder_attention_heads=c["encoder_attention_heads"], conv_pos=c["conv_pos"],
                      conv_pos_groups=c["conv_pos_groups"])


def select_subnet(cfg: dict, where: str = "cfg") -> Tuple[str, ArchConfig]:
    """``(supernet_type, served subnet)`` of a checkpoint's ``cfg["model"]``, by the reference expert's rule
    (expert.py:16-44); refuses what is not served with a ``ValueError`` naming the field."""
    if not isinstance(cfg, dict):
        raise ValueError(f"{where}: cfg['model'] must be a dict, not {type(cfg).__name__}")
    name = cfg.get("_name")
    if name not in NAMES:
        raise ValueError(f"{where}: _name={name!r} is not served (served: {', '.join(map(repr, NAMES))})")
    c = dict(_DEFAULTS, **cfg)
    checks = (("encoder_layers", c["encoder_layers"] == 12, "12"),
              ("layer_type", c["layer_type"] == "transformer", "'transformer'"),
              ("conv_feature_layers", str(c["conv_feature_layers"]).replace(" ", "") == _CONV_FEATURE_LAYERS.replace(" ", ""),
               repr(_CONV_FEATURE_LAYERS)),
              ("pos_conv_depth", c["pos_conv_depth"] == 1, "1"),
              ("layer_norm_first", not c["layer_norm_first"], "False"),
              ("activation_fn", c["activation_fn"] == "gelu", "'gelu'"),
              ("extractor_mode", c["extractor_mode"] in ("default", "layer_norm"), "'default', 'layer_norm'"))
    for key, ok, served in checks:
        if not ok:
            raise ValueError(f"{where}: {key}={c[key]!r} is not served (served: {served})")
    stype = c["supernet_type"]
    if name == "hubert_pruner":
        if "pruner_supernet" not in cfg:
            raise ValueError(f"{where}: pruner_supernet is missing (hubert_pruner checkpoints name their supernet)")
        ps = str(cfg["pruner_supernet"]).lower()
        stype = "small" if ps.endswith("small.yaml") else "base" if ps.endswith("base.yaml") else stype
    if stype not in ("small", "base"):
        raise ValueError(f"{where}: supernet_type={stype!r} is not served (served: 'small', 'base')")
    E, H, F = SUBNETS[(name, stype)]
    sup = supernet_arch(cfg)
    if sup.encoder_embed_dim <= 512 or sup.encoder_embed_dim < E or sup.encoder_ffn_embed_dim < F:
        raise ValueError(f"{where}: encoder_embed_dim={sup.encoder_embed_dim} / encoder_ffn_embed_dim="
                         f"{sup.encoder_ffn_embed_dim}: the supernet must be wider than 512 and hold the {E}-wide "
                         f"subnet (FFN {F})")
    return stype, replace(sup, encoder_embed_dim=E, encoder_attention_heads=H, encoder_ffn_embed_dim=F)


def required_keys(sup: ArchConfig) -> List[str]:
    """The supernet tensors the served subnet is cut from."""
    keys = []
    for i in range(7):
        p = f"feature_extractor.conv_layers.{i}"
        keys.append(f"{p}.0.weight")
        if sup.conv_bias:
            keys.append(f"{p}.0.bias")
        if sup.extractor_mode == "layer_norm":
            keys += [f"{p}.2.1.weight", f"{p}.2.1.bias"]
        elif i == 0:
            keys += [f"{p}.2.weight", f"{p}.2.bias"]
    keys += ["layer_norm.weight", "layer_norm.bias", "post_extract_proj.weight", "post_extract_proj.bias",
             "encoder.pos_conv.0.weight_g", "encoder.pos_conv.0.weight_v", "encoder.pos_conv.0.bias",
             "encoder.layer_norm.weight", "encoder.layer_norm.bias"]
    for l in range(sup.encoder_layers):
        p = f"encoder.layers.{l}"
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            keys += [f"{p}.self_attn.{n}.weight", f"{p}.self_attn.{n}.bias"]
        for n in ("self_attn_layer_norm", "fc1", "fc2", "final_layer_norm"):
            keys += [f"{p}.{n}.weight", f"{p}.{n}.bias"]
    return keys


def fabricate_lighthubert_state_dict(seed: int = 0, cfg: Optional[dict] = None) -> Dict[str, torch.Tensor]:
    """Deterministic supernet weights for ``cfg`` (``lighthubert_config("small")`` by default), with the keys and
    shapes of the reference's ``LightHuBERT`` state dict: those of ``fabricate_state_dict`` for the supernet (random
    everywhere, so the rows and columns outside a subnet, and fc1 / fc2's other splits, differ from what any other cut
    would take), plus the prediction head of layer 12 and ``mask_emb``, which the forward does not read."""
    sup = supernet_arch(cfg if cfg is not None else lighthubert_config("small"))
    sd = fabricate_state_dict(sup, seed)
    g = torch.Generator().manual_seed(seed + 1)
    E = sup.encoder_embed_dim
    sd["layer_pred_heads.11.weight"] = torch.randn(768, E, generator=g) / math.sqrt(E)
    sd["mask_emb"] = torch.rand(E, generator=g)
    return sd


def _split_cut(t: torch.Tensor, dim: int, split: int, n: int, m: int) -> torch.Tensor:
    """SLinear's cut of ``t`` along ``dim`` to ``n`` of ``m``-wide splits (scaling_linear.py:84-94, 106-116): the
    splits are ``split`` wide, the subnet's ``n / ceil(n / m)`` wide, and it takes the first ``ceil(n / m)`` of them."""
    if n == t.size(dim):
        return t
    ratio = n / m
    size = int(n / ratio)
    parts = torch.split(t, split, dim=dim)[: int(math.ceil(ratio))]
    return torch.cat([p.narrow(dim, 0, min(size, n - i * size)) for i, p in enumerate(parts)], dim=dim)


def cut_subnet(sd: Dict[str, torch.Tensor], sup: ArchConfig, sub: ArchConfig) -> Dict[str, torch.Tensor]:
    """The subnet's HuBERT state dict, cut from the supernet's ``sd`` as ``set_sample_config`` cuts it. A missing
    supernet tensor raises ``KeyError`` naming it."""
    missing = [k for k in required_keys(sup) if k not in sd]
    if missing:
        raise KeyError(f"LightHuBERT checkpoint lacks {len(missing)} supernet tensor(s), first '{missing[0]}'")
    E, F, A = sub.encoder_embed_dim, sub.encoder_ffn_embed_dim, sub.encoder_embed_dim
    Es = sup.encoder_embed_dim
    G = sub.conv_pos_groups
    out: Dict[str, torch.Tensor] = {}
    for k in required_keys(sup):
        t = sd[k].detach().to("cpu", torch.float32)
        if k.startswith("feature_extractor.") or k.startswith("layer_norm."):
            out[k] = t
        elif k.startswith("post_extract_proj.") or k.startswith("encoder.layer_norm.") or k == "encoder.pos_conv.0.bias":
            out[k] = t[:E]
        elif k in ("encoder.pos_conv.0.weight_g", "encoder.pos_conv.0.weight_v"):
            continue
        elif ".self_attn." in k:
            if ".out_proj." in k:
                out[k] = t[:E, :A] if t.dim() == 2 else t[:E]
            else:
                out[k] = t[:A, :E] if t.dim() == 2 else t[:A]
        elif ".fc1." in k:
            t = t[:, :E] if t.dim() == 2 else t
            out[k] = _split_cut(t, 0, Es, F, E)
        elif ".fc2." in k:
            out[k] = _split_cut(t, 1, Es, F, E)[:E] if t.dim() == 2 else t[:E]
        else:  # self_attn_layer_norm, final_layer_norm
            out[k] = t[:E]
    # pos_conv: the reference cuts weight_g * weight_v / ||weight_v|| (norm over the whole supernet weight_v, per
    # tap); the library folds its own weight_g * v / ||v|| over the cut v, so g is rescaled by ||v_cut|| / ||v||
    v = sd["encoder.pos_conv.0.weight_v"].detach().to("cpu", torch.float64)
    g = sd["encoder.pos_conv.0.weight_g"].detach().to("cpu", torch.float64)
    vc = v[:E, : E // G, :]
    out["encoder.pos_conv.0.weight_v"] = vc.float().contiguous()
    out["encoder.pos_conv.0.weight_g"] = (g * vc.norm(dim=(0, 1), keepdim=True) / v.norm(dim=(0, 1), keepdim=True)).float()
    return {k: t.contiguous() for k, t in out.items()}


def load_lighthubert_checkpoint(path: str) -> Tuple[dict, Dict[str, torch.Tensor]]:
    """``(cfg["model"], supernet tensors)`` of a reference LightHuBERT checkpoint file."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(state, dict) or "cfg" not in state or "model" not in state or "model" not in state["cfg"]:
        raise ValueError(f"{path}: not a LightHuBERT checkpoint (expected {{'cfg': {{'model': ...}}, 'model': ...}})")
    return dict(state["cfg"]["model"]), state["model"]


class LighthubertExpert(NativeExpert):
    """``UpstreamExpert`` of LightHuBERT: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms returns the
    reference's ``{"hidden_states": [features, layer 1, ..., layer 12]}``, 13 tensors [B, T, E] with E = 384, 640,
    768 or 512 by subnet, at a downsample rate of 320. The waveforms are always normalised. ``lanes``,
    ``global_max_len``, the inference-only refusal, the training-mode warning and ``forward_host`` are those of every
    expert (``NativeExpert``)."""

    model_label = "LightHuBERT"
    num_outputs = 13

    def __init__(self, ckpt: Optional[str] = None, name: str = "lighthubert_small", kind: str = "small", seed: int = 0,
                 randomize_seed: Optional[int] = None, hooks=None, feature_selection=None, **kwargs):
        if hooks or feature_selection is not None:
            raise TypeError("hooks and feature_selection are not available for LightHuBERT: the reference expert "
                            "registers none (lighthubert/expert.py); use the default hidden_states")
        if ckpt is not None:
            cfg, sd = load_lighthubert_checkpoint(ckpt)
            where = ckpt
        else:
            cfg, sd, where = lighthubert_config(kind), None, f"lighthubert_{kind}"
        stype, sub = select_subnet(cfg, where)
        sup = supernet_arch(cfg)
        if sd is None or randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights, same shapes
            sd = fabricate_lighthubert_state_dict(seed if randomize_seed is None else randomize_seed, cfg)
        super().__init__(cut_subnet(sd, sup, sub))
        self.name = name
        self.supernet_type = stype
        self.arch = sub
        self.num_layers = sub.encoder_layers

    def _native_args(self):
        c = _c_config(self.arch)
        c.proj_hidden0 = 1
        return "s3b_model_create", c, self._state_dict_host

    def get_downsample_rates(self, key: str) -> int:
        return DOWNSAMPLE_RATE

    @property
    def hidden_size(self) -> int:
        return self.arch.encoder_embed_dim

    def num_frames(self, max_len: int) -> int:
        n = max_len
        for k, s in ((10, 5), (3, 2), (3, 2), (3, 2), (3, 2), (2, 2), (2, 2)):
            n = (n - k) // s + 1 if n >= k else 0
        return n

    def forward(self, wavs: List[torch.Tensor]) -> Dict:
        out = self._forward_ex(*self._prepare(wavs))
        return {"hidden_states": [out[i] for i in range(self.num_outputs)]}
