"""MAE-AST (``mae_ast_frame``, ``mae_ast_patch``) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/mae_ast/{expert,mae_ast}.py) runs, per utterance, ``torchaudio.compliance.kaldi.fbank``
with 128 mel bins at kaldi defaults (povey window, 25 / 10 ms, dither 0, pre-emphasis 0.97, no energy), zero-pads the
features to the batch's longest, F frames, and then:

- ``BatchNorm2d(1, affine=False)`` in eval times 0.5 on every element, padded frames included:
  ``y = (x - running_mean) * rsqrt(running_var + 1e-5) * 0.5``;
- ``nn.Unfold`` with kernel = stride = (kt, kc) over the [F, 128] image: T' = F // kt time patches times nv = 128 // kc
  frequency patches, token ``t * nv + fi``, column ``i * kc + j`` (frame model (2, 128), patch model (16, 16); K = 256);
- ``post_extract_proj`` = Linear(256, 768);
- a key mask of one prefix per utterance, ``valid_b = min(ceil(n_b / kt), T') * nv`` tokens (n_b the utterance's own
  frames; a partly padded last patch is valid);
- with ``enc_sine_pos``, rows 0 .. T' nv - 1 of the checkpoint's ``enc_sine_pos_embed.pe`` added to the valid tokens;
- the fairseq ``TransformerEncoder`` of wav2vec 2.0 layers: post-LN (``encoder.layer_norm`` on the input) or pre-LN
  (no input norm, hidden states before the final norm). The hidden states are the ``encoder_layers`` layer outputs,
  each [B, T' nv, 768] read as [B, T', nv * 768]; the reference's cut to ``len(range(0, max_len, 160 kt))`` frames never
  removes one.

Checkpoint: ``{"cfg": {"model": {...}, "task": {...}}, "model": MAE_AST.state_dict()}``. The decoder,
``dec_*_pos_embed``, ``final_proj_*``, ``*_mask_emb``, the unused ``layer_norm.*`` and ``num_batches_tracked`` are
ignored. A missing encoder, projection, batch-norm or (with ``enc_sine_pos``) ``pe`` tensor raises ``KeyError`` naming
it; a configuration outside the served one raises ``ValueError`` naming the field.

The released files (``random_frame_75_12LayerEncoder.pt``, ``chunk_patch_75_12LayerEncoder.pt``) are not reachable
offline. ``fabricate_mae_ast_state_dict`` writes their believed configuration (12-layer post-LN encoder, 2-layer
decoder, ``enc_sine_pos`` and ``dec_sine_pos``, ``max_token_length`` 48000), which was not checked against them.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from .. import lib as _lib
from .expert import NativeExpert

SAMPLE_RATE = 16000
FBANK_STRIDE = 160
NUM_BINS = 128
EMBED, HEADS, FFN = 768, 12, 3072
# kind -> (kt, kc): patch size in frames and mel bins (stride equal to it)
KINDS = {"frame": (2, 128), "patch": (16, 16)}
# the MAE_AST_Config defaults (mae_ast.py) of the fields this port reads, for a file whose cfg omits one
MODEL_DEFAULTS = {
    "ast_kernel_size_chan": 16, "ast_kernel_size_time": 16, "ast_kernel_stride_chan": 16,
    "ast_kernel_stride_time": 16, "encoder_layers": 12, "encoder_embed_dim": 768, "encoder_ffn_embed_dim": 3072,
    "encoder_attention_heads": 12, "activation_fn": "gelu", "layer_norm_first": False, "decoder_embed_dim": 768,
    "decoder_layers": 2, "use_post_enc_proj": False, "max_token_length": 48000, "enc_sine_pos": False,
    "enc_conv_pos": False, "dec_sine_pos": False, "dec_conv_pos": False,
}
MIN_SAMPLES = 400  # one fbank frame per utterance; the reference's kaldi fbank refuses fewer samples


def frames(n: int) -> int:
    """kaldi fbank frames of n samples (snip_edges)."""
    return 0 if n < 400 else 1 + (n - 400) // FBANK_STRIDE


def num_frames(kind: str, max_len: int) -> int:
    """Output frames (time patches) T' = F // kt of a batch padded to max_len."""
    return frames(max_len) // KINDS[kind][0]


def min_batch_samples(kind: str) -> int:
    """The shortest longest-utterance that gives one time patch: 400 + 160 (kt - 1) samples."""
    return 400 + FBANK_STRIDE * (KINDS[kind][0] - 1)


def valid_frames(kind: str, lens: List[int], max_len: int) -> List[int]:
    """Valid time patches per utterance: min(ceil(n_b / kt), T')."""
    kt, T = KINDS[kind][0], num_frames(kind, max_len)
    return [min(-(-frames(n) // kt), T) for n in lens]


def sinusoid_table(rows: int, d: int = EMBED) -> torch.Tensor:
    """The ``SinusoidalPositionalEncoding`` table [1, rows, d]: sin at even columns, cos at odd ones, fp32 as torch
    computes it."""
    position = torch.arange(rows).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d, 2) * (-math.log(10000.0) / d))
    pe = torch.zeros(1, rows, d)
    pe[0, :, 0::2] = torch.sin(position * div_term)
    pe[0, :, 1::2] = torch.cos(position * div_term)
    return pe


def fabricate_mae_ast_state_dict(seed: int = 0, kind: str = "frame", layers: int = 12, layer_norm_first: bool = False,
                                 enc_sine_pos: bool = True, max_token_length: int = 48000) -> Dict:
    """A deterministic checkpoint in the reference's format, ``{"cfg": {"model", "task"}, "model": state_dict}``, by
    default in the believed released configuration: a 12-layer post-LN 768 encoder, a 2-layer decoder, (2, 128) or
    (16, 16) patches, ``enc_sine_pos`` and ``dec_sine_pos`` with ``pe`` filled by the sinusoid formula, and non-trivial
    batch-norm statistics. Linear weights have fan-in variance and LayerNorm gains are near 1, so activations stay in
    a trained encoder's range."""
    kt, kc = KINDS[kind]
    g = torch.Generator().manual_seed(seed)
    D, F, K = EMBED, FFN, kt * kc

    def lin(n, k):
        return torch.randn(n, k, generator=g) / math.sqrt(k), torch.randn(n, generator=g) * 0.02

    def ln(d):
        return 1.0 + 0.1 * torch.randn(d, generator=g), 0.05 * torch.randn(d, generator=g)

    def layer(prefix, sd):
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[f"{prefix}self_attn.{n}.weight"], sd[f"{prefix}self_attn.{n}.bias"] = lin(D, D)
        sd[prefix + "self_attn_layer_norm.weight"], sd[prefix + "self_attn_layer_norm.bias"] = ln(D)
        sd[prefix + "fc1.weight"], sd[prefix + "fc1.bias"] = lin(F, D)
        sd[prefix + "fc2.weight"], sd[prefix + "fc2.bias"] = lin(D, F)
        sd[prefix + "final_layer_norm.weight"], sd[prefix + "final_layer_norm.bias"] = ln(D)

    sd: Dict[str, torch.Tensor] = {}
    sd["encoder_mask_emb"] = torch.rand(D, generator=g)
    sd["decoder_mask_emb"] = torch.rand(D, generator=g)
    # the normalised features have unit scale: (x - mean) * 0.5 / std of a log-mel around -8 with std ~3.5
    sd["post_extract_proj.weight"], sd["post_extract_proj.bias"] = lin(D, K)
    sd["layer_norm.weight"], sd["layer_norm.bias"] = ln(NUM_BINS)
    sd["batch_norm.running_mean"] = torch.tensor([-8.25])
    sd["batch_norm.running_var"] = torch.tensor([12.5])
    sd["batch_norm.num_batches_tracked"] = torch.tensor(100000)
    pe = sinusoid_table(max_token_length)
    if enc_sine_pos:
        sd["enc_sine_pos_embed.pe"] = pe
    for l in range(layers):
        layer(f"encoder.layers.{l}.", sd)
    sd["encoder.layer_norm.weight"], sd["encoder.layer_norm.bias"] = ln(D)
    sd["dec_sine_pos_embed.pe"] = pe.clone()
    for l in range(2):
        layer(f"decoder.layers.{l}.", sd)
    sd["decoder.layer_norm.weight"], sd["decoder.layer_norm.bias"] = ln(D)
    for n in ("final_proj_reconstruction", "final_proj_classification"):
        sd[n + ".weight"], sd[n + ".bias"] = lin(K, D)
    # the file carries every MAE_AST_Config field: the reference builds its model from SimpleNamespace(**cfg)
    model = dict(MODEL_DEFAULTS, feature_grad_mult=1.0, decoder_layerdrop=0.0, dropout=0.1, attention_dropout=0.1,
                 activation_dropout=0.0, encoder_layerdrop=0.0, dropout_input=0.0, random_mask_prob=0.75,
                 mask_length=10, mask_selection="static", mask_other=0, no_mask_overlap=False, mask_min_space=0,
                 conv_pos=128, conv_pos_groups=16, checkpoint_activations=False)
    model.update(ast_kernel_size_time=kt, ast_kernel_size_chan=kc, ast_kernel_stride_time=kt,
                 ast_kernel_stride_chan=kc, encoder_layers=layers, layer_norm_first=layer_norm_first,
                 enc_sine_pos=enc_sine_pos, dec_sine_pos=True, max_token_length=max_token_length)
    task = {"sample_rate": SAMPLE_RATE, "feature_dim": NUM_BINS, "feature_rate": 100, "feature_type": "fbank",
            "mask_type": "random_mask" if kind == "frame" else "chunk_mask", "deltas": False}
    return {"cfg": {"model": model, "task": task}, "model": sd}


def kind_of(ckpt: Dict, where: str = "checkpoint") -> str:
    """'frame' or 'patch', from a checkpoint's ast_kernel_size_time / ast_kernel_size_chan."""
    model = dict(MODEL_DEFAULTS, **(ckpt.get("cfg", {}).get("model", {}) if isinstance(ckpt, dict) else {}))
    shape = (model["ast_kernel_size_time"], model["ast_kernel_size_chan"])
    for kind, ks in KINDS.items():
        if ks == shape:
            return kind
    raise ValueError(f"{where}: MAE-AST ast_kernel_size_time/ast_kernel_size_chan={shape!r} is not served "
                     "((2, 128) or (16, 16))")


def served_config(cfg: Dict, kind: str, where: str = "checkpoint") -> Dict:
    """The fields the library needs from ``{"model", "task"}``; a value outside the served scope raises
    ``ValueError`` naming the field."""
    model = dict(MODEL_DEFAULTS, **cfg.get("model", {}))
    task = cfg.get("task", {})

    def refuse(field, value, served):
        raise ValueError(f"{where}: MAE-AST {field}={value!r} is not served ({served})")

    if task.get("sample_rate", SAMPLE_RATE) != SAMPLE_RATE:
        refuse("task.sample_rate", task.get("sample_rate"), "16000")
    if task.get("feature_dim") != NUM_BINS:
        refuse("task.feature_dim", task.get("feature_dim"), "128 mel bins")
    kt, kc = model["ast_kernel_size_time"], model["ast_kernel_size_chan"]
    if (kt, kc) not in KINDS.values():
        refuse("ast_kernel_size_time/ast_kernel_size_chan", (kt, kc), "(2, 128) or (16, 16)")
    if (kt, kc) != KINDS[kind]:
        refuse("ast_kernel_size_time/ast_kernel_size_chan", (kt, kc), f"the {kind} model has {KINDS[kind]}")
    for f, k in (("ast_kernel_stride_time", kt), ("ast_kernel_stride_chan", kc)):
        if model[f] != k:
            refuse(f, model[f], f"a stride equal to the kernel, {k}")
    for f, v in (("encoder_embed_dim", EMBED), ("encoder_attention_heads", HEADS), ("encoder_ffn_embed_dim", FFN)):
        if model[f] != v:
            refuse(f, model[f], str(v))
    if not isinstance(model["encoder_layers"], int) or not 1 <= model["encoder_layers"] <= 63:
        refuse("encoder_layers", model["encoder_layers"], "1..63")
    if model["activation_fn"] != "gelu":
        refuse("activation_fn", model["activation_fn"], "gelu")
    if model["enc_conv_pos"]:
        refuse("enc_conv_pos", model["enc_conv_pos"], "false: the convolutional positions are not used by MAE-AST")
    return {"kind": kind, "layers": int(model["encoder_layers"]), "layer_norm_first": bool(model["layer_norm_first"]),
            "enc_sine_pos": bool(model["enc_sine_pos"])}


def required_keys(layers: int, layer_norm_first: bool, enc_sine_pos: bool) -> List[str]:
    """The state-dict tensors the forward reads."""
    keys = ["post_extract_proj.weight", "post_extract_proj.bias", "batch_norm.running_mean", "batch_norm.running_var"]
    if enc_sine_pos:
        keys.append("enc_sine_pos_embed.pe")
    if not layer_norm_first:
        keys += ["encoder.layer_norm.weight", "encoder.layer_norm.bias"]
    for l in range(layers):
        p = f"encoder.layers.{l}."
        for n in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj",
                  "self_attn_layer_norm", "fc1", "fc2", "final_layer_norm"):
            keys += [p + n + ".weight", p + n + ".bias"]
    return keys


def prepare_mae_ast_tensors(ckpt: Dict, kind: str, where: str = "checkpoint") -> Tuple[Dict, Dict[str, torch.Tensor]]:
    """``(served config, tensors the library reads)`` of a reference checkpoint dict."""
    if not isinstance(ckpt, dict) or "cfg" not in ckpt or "model" not in ckpt:
        raise ValueError(f"{where}: not an MAE-AST checkpoint (expected a dict with 'cfg' and 'model')")
    cfg = served_config(ckpt["cfg"], kind, where)
    sd = ckpt["model"]
    keys = required_keys(cfg["layers"], cfg["layer_norm_first"], cfg["enc_sine_pos"])
    missing = [k for k in keys if k not in sd]
    if missing:
        raise KeyError(f"{where}: MAE-AST checkpoint lacks {len(missing)} required tensor(s), first '{missing[0]}'")
    kt, kc = KINDS[kind]
    if tuple(sd["post_extract_proj.weight"].shape) != (EMBED, kt * kc):
        raise ValueError(f"{where}: post_extract_proj.weight has shape {tuple(sd['post_extract_proj.weight'].shape)}, "
                         f"the {kind} model needs ({EMBED}, {kt * kc})")
    if cfg["enc_sine_pos"]:
        pe = sd["enc_sine_pos_embed.pe"]
        if pe.dim() != 3 or pe.shape[0] != 1 or pe.shape[2] != EMBED or pe.shape[1] < 1:
            raise ValueError(f"{where}: enc_sine_pos_embed.pe has shape {tuple(pe.shape)}, expected [1, rows, {EMBED}]")
    out = {k: sd[k].detach().to("cpu", torch.float32).contiguous() for k in keys}
    return cfg, out


def load_mae_ast_checkpoint(path: str) -> Dict:
    """The ``{"cfg", "model"}`` dict of a reference MAE-AST checkpoint file."""
    return torch.load(path, map_location="cpu", weights_only=False)


class MaeAstExpert(NativeExpert):
    """``UpstreamExpert`` of MAE-AST: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms of at least 400 samples
    returns the reference's ``{"hidden_states": [layer 1, ..., layer L]}``, L tensors [B, T', nv * 768] (frame model
    nv = 1, patch model nv = 8) at a downsample rate of 320 or 2560. The longest utterance needs 560 (frame) or 2800
    (patch) samples. ``lanes``, ``global_max_len``, the inference-only refusal, the training-mode warning and
    ``forward_host`` are those of every expert (``NativeExpert``)."""

    model_label = "MAE-AST"
    min_samples = MIN_SAMPLES

    def __init__(self, ckpt: Optional[str] = None, name: str = "mae_ast_frame", kind: Optional[str] = "frame",
                 seed: int = 0, randomize_seed: Optional[int] = None, hooks=None, feature_selection=None, **kwargs):
        if hooks or feature_selection is not None:
            raise TypeError("hooks and feature_selection are not available for MAE-AST: the reference expert registers "
                            "none (mae_ast/expert.py); use the default hidden_states")
        if ckpt is not None:
            data, where = load_mae_ast_checkpoint(ckpt), ckpt
        else:
            data, where = None, name
        if kind is None:  # mae_ast_local / mae_ast_url: the file's own patch shape
            if data is None:
                raise ValueError(f"{name}: a checkpoint file is required")
            kind = kind_of(data, where)
        if kind not in KINDS:
            raise ValueError(f"kind={kind!r} is not served (served: 'frame', 'patch')")
        if data is None or randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights, same shapes
            data = fabricate_mae_ast_state_dict(seed if randomize_seed is None else randomize_seed, kind)
        self.cfg, tensors = prepare_mae_ast_tensors(data, kind, where)
        super().__init__(tensors)
        self.name = name
        self.kind = kind
        self.num_layers = self.num_outputs = self.cfg["layers"]
        self.min_batch_samples = min_batch_samples(kind)
        self.pe_rows = int(tensors["enc_sine_pos_embed.pe"].shape[1]) if self.cfg["enc_sine_pos"] else 0

    def _native_args(self):
        c = self.cfg
        cfg = _lib.S3BMaeAstConfig(patch=int(self.kind == "patch"), embed_dim=EMBED, num_heads=HEADS, ffn_dim=FFN,
                                   num_layers=c["layers"], layer_norm_first=int(c["layer_norm_first"]),
                                   sine_pos=int(c["enc_sine_pos"]), max_tokens=self.pe_rows)
        return "s3b_mae_ast_model_create", cfg, self._state_dict_host

    def get_downsample_rates(self, key: str = None) -> int:
        return KINDS[self.kind][0] * FBANK_STRIDE

    @property
    def hidden_size(self) -> int:
        return (NUM_BINS // KINDS[self.kind][1]) * EMBED

    def num_frames(self, max_len: int) -> int:
        return num_frames(self.kind, max_len)

    def forward(self, wavs: List[torch.Tensor]) -> Dict:
        native, wavs, lens, max_len, T = self._prepare(wavs)
        nv = NUM_BINS // KINDS[self.kind][1]
        if self.cfg["enc_sine_pos"] and T * nv > self.pe_rows:
            raise ValueError(f"{T * nv} tokens ({max_len} samples) exceed enc_sine_pos_embed.pe's {self.pe_rows} rows "
                             "(max_token_length)")
        out = self._forward_ex(native, wavs, lens, max_len, T)
        return {"hidden_states": [out[i] for i in range(self.num_outputs)]}
