"""NPC (``npc``, ``npc_360hr``, ``npc_960hr`` and their hub variants) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/npc/{expert,npc,audio}.py) runs APC's front end per utterance (kaldi fbank with a
hamming window, 80 bins, CMVN over all frames with the unbiased std), pads the features to T = max m with zeros, and
feeds them through ``n_blocks`` blocks. ConvBlock i is ``act(bn2(linear(act(bn1(conv(x))))) + x)`` (the residual from
block 1 on, when ``residual`` is set), with a k = 3 same-padded conv and a 1x1 linear; masked conv i is
``tanh(conv1d(x, W * conv_mask))`` on block i's output, with a centred band of ``mask_size + 2 (i + 1)`` of its
``kernel_size`` taps masked out. ``feat`` is the sum of the masked convs. The expert's hooks record, in firing order,
block 0, masked conv 0, block 1, ..., masked conv n-1 and ``feat``: 2 n + 1 hidden states [B, T, 512].

Frames t >= m_b are not zero: they hold the model's response to the zero padding features, and valid frames near m_b
read them, so an utterance's result depends on T. ``global_max_len`` fixes T across shards, as for every expert.

Here the whole forward is one ``s3b_forward`` of a model made by ``s3b_npc_model_create``: the fbank and CMVN kernels,
then three GEMMs per block (conv, linear, masked conv), with each BatchNorm folded into the conv before it and the
masked taps left out of the contraction.

Checkpoint: the reference's ``{"config": {...}, "model": NPC.state_dict()}`` file (npc/expert.py:22-26). Served:
APC's audio settings, ``hidden_size`` 512, any ``n_blocks`` >= 1, odd ``kernel_size`` and ``mask_size`` with
``kernel_size > mask_size + 2 n_blocks``, ``activate`` relu or tanh, ``batch_norm`` and ``residual`` either way.
``disable_cross_layer`` and ``dim_bottleneck`` are refused; ``vq`` (which acts after ``feat``) is read and ignored.
The released checkpoints (npc_360hr, npc_960hr) are not reachable offline, and their configs were not checked; the
config believed to be released (hidden 512, 4 blocks, kernel 15, mask 5, batch_norm, relu, residual) is what
``npc_config()`` returns, and without a file the experts use a fabricated checkpoint of that shape.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from .. import lib as _lib
from .apc import DOWNSAMPLE_RATE, MIN_SAMPLES, NUM_MEL_BINS, num_frames, validate_audio
from .expert import NativeExpert

HIDDEN = 512
# the config believed to be that of the released checkpoints (not checked: the files are unreachable offline)
DEFAULTS = {"n_blocks": 4, "kernel_size": 15, "mask_size": 5, "residual": True, "batch_norm": True,
            "activate": "relu"}


def hidden_states_info(n_blocks: int) -> Tuple[str, ...]:
    """The expert's hook names in firing order (npc/expert.py:28-41)."""
    names = []
    for i in range(n_blocks):
        names += [f"self.model.blocks[{i}]", f"self.model.masked_convs[{i}]"]
    return tuple(names) + ("self.model",)


HIDDEN_STATES_INFO = hidden_states_info(DEFAULTS["n_blocks"])


def mask_width(paras: dict, i: int) -> int:
    """Taps masked out of masked conv i (npc.py: cur_mask_size grows by 2 per block)."""
    return paras["mask_size"] + 2 * (i + 1)


def npc_config(**over) -> dict:
    """The ``config`` entry of a checkpoint (npc/expert.py:22-26); ``over`` replaces ``model.paras`` fields."""
    paras = {"hidden_size": HIDDEN, "dropout": 0.1, "vq": {"codebook_size": [64, 64, 64, 64],
                                                          "code_dim": [128, 128, 128, 128],
                                                          "gumbel_temperature": 1.0}}
    paras.update(DEFAULTS)
    paras.update(over)
    return {"data": {"audio": {"feat_type": "fbank", "feat_dim": NUM_MEL_BINS, "frame_length": 25, "frame_shift": 10,
                               "decode_wav": False, "cmvn": True}},
            "model": {"paras": paras}}


def validate_config(config: dict, where: str = "config") -> dict:
    """Checks that a checkpoint's config is served; returns ``model.paras`` with every served field. Anything else
    raises ``ValueError`` naming the field."""
    try:
        paras = dict(config["model"]["paras"])
    except (KeyError, TypeError) as e:
        raise ValueError(f"{where}: expected config['data']['audio'] and config['model']['paras'] ({e!r} missing)")
    validate_audio(config, where)
    if paras.pop("hidden_size", None) != HIDDEN:
        raise ValueError(f"{where}: model.paras.hidden_size must be {HIDDEN}")
    out = {"hidden_size": HIDDEN}
    for key in ("n_blocks", "kernel_size", "mask_size", "residual"):
        if key not in paras:
            raise ValueError(f"{where}: model.paras.{key} is missing")
    out["n_blocks"] = n = paras.pop("n_blocks")
    out["kernel_size"] = k = paras.pop("kernel_size")
    out["mask_size"] = msk = paras.pop("mask_size")
    out["residual"] = bool(paras.pop("residual"))
    out["batch_norm"] = bool(paras.pop("batch_norm", True))
    out["activate"] = paras.pop("activate", "relu")
    if not isinstance(n, int) or not 1 <= n <= 32:
        raise ValueError(f"{where}: model.paras.n_blocks must be an integer in 1..32, not {n!r}")
    if not isinstance(k, int) or k % 2 != 1 or k > 127:
        raise ValueError(f"{where}: model.paras.kernel_size must be odd and <= 127, not {k!r}")
    if not isinstance(msk, int) or msk % 2 != 1 or msk < 1:
        raise ValueError(f"{where}: model.paras.mask_size must be odd, not {msk!r}")
    if k <= msk + 2 * n:
        raise ValueError(f"{where}: model.paras.kernel_size {k} must exceed mask_size + 2 n_blocks = {msk + 2 * n}")
    if out["activate"] not in ("relu", "tanh"):
        raise ValueError(f"{where}: model.paras.activate must be 'relu' or 'tanh', not {out['activate']!r}")
    if paras.pop("disable_cross_layer", False):
        raise ValueError(f"{where}: model.paras.disable_cross_layer=True is not served")
    if paras.pop("dim_bottleneck", None) is not None:
        raise ValueError(f"{where}: model.paras.dim_bottleneck is not served (it replaces feat)")
    paras.pop("dropout", None)  # inactive in eval
    paras.pop("vq", None)  # acts after feat is recorded
    if paras:
        raise ValueError(f"{where}: model.paras.{sorted(paras)[0]} is not an NPC parameter")
    return out


def required_keys(paras: dict) -> List[str]:
    keys = []
    for i in range(paras["n_blocks"]):
        for mod in ("conv", "linear"):
            keys += [f"blocks.{i}.{mod}.weight", f"blocks.{i}.{mod}.bias"]
        if paras["batch_norm"]:
            for bn in ("bn1", "bn2"):
                keys += [f"blocks.{i}.{bn}.{n}" for n in ("weight", "bias", "running_mean", "running_var")]
        keys += [f"masked_convs.{i}.conv.weight", f"masked_convs.{i}.conv.bias", f"masked_convs.{i}.conv_mask"]
    return keys


def fabricate_npc_state_dict(seed: int = 0, paras: Optional[dict] = None) -> Dict[str, torch.Tensor]:
    """Deterministic weights with the keys and shapes of ``NPC(80, **paras)`` (default ``npc_config()``'s).

    BatchNorm is not the identity: running means and variances away from 0 and 1, gammas away from 1. Conv weights are
    scaled by their fan-in (the masked convs' over their unmasked taps only), so that activations through the residual
    blocks stay in the range of a trained model instead of growing block by block."""
    p = dict(npc_config()["model"]["paras"])
    p.update(paras or {})
    g = torch.Generator().manual_seed(seed)
    H, k = HIDDEN, p["kernel_size"]
    sd: Dict[str, torch.Tensor] = {}
    for i in range(p["n_blocks"]):
        cin = NUM_MEL_BINS if i == 0 else H
        b = f"blocks.{i}."
        sd[b + "conv.weight"] = torch.randn(H, cin, 3, generator=g) / math.sqrt(3 * cin)
        sd[b + "conv.bias"] = torch.randn(H, generator=g) * 0.1
        sd[b + "linear.weight"] = torch.randn(H, H, 1, generator=g) / math.sqrt(H)
        sd[b + "linear.bias"] = torch.randn(H, generator=g) * 0.1
        if p["batch_norm"]:
            for bn in ("bn1", "bn2"):
                sd[b + f"{bn}.weight"] = 0.5 + torch.rand(H, generator=g)
                sd[b + f"{bn}.bias"] = torch.randn(H, generator=g) * 0.2
                sd[b + f"{bn}.running_mean"] = torch.randn(H, generator=g) * 0.3
                sd[b + f"{bn}.running_var"] = 0.4 + 1.2 * torch.rand(H, generator=g)
                sd[b + f"{bn}.num_batches_tracked"] = torch.tensor(1000)
        mw = mask_width(p, i)
        head = (k - mw) // 2
        mask = torch.ones(H, H, k)
        mask[:, :, head:head + mw] = 0
        sd[f"masked_convs.{i}.conv.weight"] = torch.randn(H, H, k, generator=g) / math.sqrt(H * (k - mw))
        sd[f"masked_convs.{i}.conv.bias"] = torch.randn(H, generator=g) * 0.1
        sd[f"masked_convs.{i}.conv_mask"] = mask
    if p.get("vq") is not None:
        for j, (cs, cd) in enumerate(zip(p["vq"]["codebook_size"], p["vq"]["code_dim"])):
            sd[f"vq_layers.{j}.vq_logits.weight"] = torch.randn(cs, cd, generator=g) / math.sqrt(cd)
            sd[f"vq_layers.{j}.vq_logits.bias"] = torch.randn(cs, generator=g) * 0.1
            sd[f"vq_layers.{j}.codebook_CxE.weight"] = torch.randn(cd, cs, generator=g) / math.sqrt(cs)
    sd["postnet.weight"] = torch.randn(NUM_MEL_BINS, H, generator=g) / math.sqrt(H)
    sd["postnet.bias"] = torch.randn(NUM_MEL_BINS, generator=g) * 0.1
    return sd


def load_npc_checkpoint(path: str) -> Tuple[dict, Dict[str, torch.Tensor]]:
    """``(paras, tensors)`` of a reference NPC checkpoint file; a missing weight raises ``KeyError`` and is named."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(state, dict) or "config" not in state or "model" not in state:
        raise ValueError(f"{path}: not an NPC checkpoint (expected a dict with the keys 'config' and 'model')")
    paras = validate_config(state["config"], path)
    weights = state["model"]
    missing = [k for k in required_keys(paras) if k not in weights]
    if missing:
        raise KeyError(f"{path}: NPC checkpoint lacks {len(missing)} required tensor(s), first '{missing[0]}'")
    k = paras["kernel_size"]
    for i in range(paras["n_blocks"]):
        w = weights[f"masked_convs.{i}.conv.weight"].float() * weights[f"masked_convs.{i}.conv_mask"].float()
        mw = mask_width(paras, i)
        head = (k - mw) // 2
        if w.shape[-1:] == (k,) and w[..., head:head + mw].abs().max().item() != 0.0:
            raise ValueError(f"{path}: masked_convs.{i}.conv_mask leaves weight on taps that kernel_size {k} and "
                             f"mask_size {paras['mask_size']} mask in block {i}: the checkpoint's mask is not the config's")
    return paras, {k: weights[k] for k in required_keys(paras)}


class NpcExpert(NativeExpert):
    """``UpstreamExpert`` of NPC: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms of at least 560 samples.
    ``lanes``, ``global_max_len``, the inference-only refusal, the training-mode warning and ``forward_host`` are
    those of every expert (``NativeExpert``). The result dict is the reference's: 2 n_blocks + 1 hidden states
    [B, T, 512], ``last_hidden_state`` (``feat``), ``hidden_state_{i}`` and ``_hidden_states_info``."""

    min_samples = MIN_SAMPLES
    model_label = "NPC"
    hidden_size = HIDDEN

    def __init__(self, ckpt: Optional[str] = None, name: str = "npc", seed: int = 0,
                 randomize_seed: Optional[int] = None, hooks=None, feature_selection=None, **kwargs):
        if hooks or feature_selection is not None:
            raise TypeError("hooks and feature_selection are not available for NPC: the reference expert registers "
                            "its hooks itself (npc/expert.py:28-41); use the default hidden_states")
        if ckpt is not None:
            paras, sd = load_npc_checkpoint(ckpt)
        else:
            paras = validate_config(npc_config())
            sd = fabricate_npc_state_dict(seed)
        if randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights of the same shape
            sd = fabricate_npc_state_dict(randomize_seed, paras)
        super().__init__(sd)
        self.name = name
        self.paras = paras
        self.num_layers = self.num_outputs = 2 * paras["n_blocks"] + 1

    def _native_args(self):
        p = self.paras
        cfg = _lib.S3BNpcConfig(n_blocks=p["n_blocks"], hidden=HIDDEN, kernel_size=p["kernel_size"],
                                mask_size=p["mask_size"], residual=int(p["residual"]),
                                batch_norm=int(p["batch_norm"]), act=0 if p["activate"] == "relu" else 1)
        return "s3b_npc_model_create", cfg, {k: self._state_dict_host[k] for k in required_keys(p)}

    def get_downsample_rates(self, key: str) -> int:
        return DOWNSAMPLE_RATE

    def num_frames(self, max_len: int) -> int:
        return num_frames(max_len)

    def forward(self, wavs: List[torch.Tensor]) -> Dict:
        out = self._forward_ex(*self._prepare(wavs))
        hidden = tuple(out[i] for i in range(self.num_outputs))
        result = {"_hidden_states_info": hidden_states_info(self.paras["n_blocks"]), "hidden_states": hidden,
                  "last_hidden_state": hidden[-1]}
        for i, h in enumerate(hidden):
            result[f"hidden_state_{i}"] = h
        return result
