"""Modified CPC (``modified_cpc``, ``cpc_local``, ``cpc_url``) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/cpc/{expert,model,feature_loader}.py) pads the raw waveforms with ``pad_sequence`` (no
normalisation, no length mask) and runs ``CPCModel``: the encoder is five ``Conv1d`` layers (1 -> 256 channels, then
256 -> 256; kernels 10, 8, 4, 4, 4; strides 5, 4, 2, 2, 2; paddings 3, 2, 1, 1, 1), each followed by ``ChannelNorm``
(per frame over the 256 channels, unbiased variance, ``rsqrt(var + 1e-5)``, affine) and ReLU; then
``nn.LSTM(256, 256, num_layers=nLevelsGRU, batch_first=True)`` over the whole padded batch from zero state. The
expert's hooks record the encoder output (transposed to [B, T, 256]) and the LSTM output: two hidden states.

Frames are not masked. The frames near and after an utterance's end hold the model's response to the zero samples:
only an utterance's last frame ``T(L_b) - 1`` (and the frames after it) depend on the padded length, so
``global_max_len`` fixes them across shards, as for every expert.

Here the whole forward is one ``s3b_forward`` of a model made by ``s3b_cpc_model_create``: conv 0 with its norm in
one kernel, conv 1..4 as implicit GEMMs over padded channels-last operands with a norm kernel each, and per LSTM layer
the input GEMM and a recurrence kernel that keeps W_hh resident in one thread-block cluster.

Checkpoint: the reference's ``torch.save({"config": vars(args), "weights": CPCModel.state_dict(), ...})`` file, whose
config is overlaid on ``cpc_default_config``'s defaults. Served: ``encoder_type`` "cpc", ``normMode`` "layerNorm",
``hiddenEncoder`` = ``hiddenGar`` = 256, ``arMode`` "LSTM", ``nLevelsGRU`` 1..8 and ``cpc_mode`` None or "none".
``samplingType`` "sequential" is refused: the reference then carries the LSTM state from one call to the next.
Training-only fields (``nPredicts``, ``rnnMode``, ``negativeSamplingExt``, ...) are ignored. Unlike the reference's
``load_state_dict(strict=False)``, which would silently keep random weights, a missing ``gEncoder.*`` or
``gAR.baseNet.*`` tensor raises ``KeyError`` naming it. The released checkpoint (``60k_epoch4-d0f474de.pt``) is not
reachable offline and its config was not checked; it is believed to use the default architecture, which is what
``cpc_config()`` returns, and without a file ``modified_cpc`` uses a fabricated checkpoint of that shape.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from .. import lib as _lib
from .expert import NativeExpert

HIDDEN = 256
DOWNSAMPLE_RATE = 160
STRIDES = (5, 4, 2, 2, 2)  # kernel = 2 * stride
PADDINGS = (3, 2, 1, 1, 1)
MIN_BATCH_SAMPLES = 159  # the shortest padded batch with one frame
HIDDEN_STATES_INFO = ("self.model.gEncoder", "self.model.gAR")

# cpc_default_config.get_default_cpc_config(): the fields a checkpoint's config is overlaid on
_DEFAULTS = {"hiddenEncoder": 256, "hiddenGar": 256, "nPredicts": 12, "negativeSamplingExt": 128,
             "learningRate": 2e-4, "schedulerStep": -1, "schedulerRamp": None, "beta1": 0.9, "beta2": 0.999,
             "epsilon": 1e-8, "sizeWindow": 20480, "nEpoch": 200, "samplingType": "samespeaker", "nLevelsPhone": 1,
             "cpc_mode": None, "encoder_type": "cpc", "normMode": "layerNorm", "onEncoder": False, "random_seed": None,
             "speakerEmbedding": 0, "arMode": "LSTM", "nLevelsGRU": 1, "rnnMode": "transformer", "dropout": False,
             "abspos": False}


def num_frames(max_len: int) -> int:
    """Frames of a batch padded to ``max_len`` samples: the conv chain ``(L + 2 p - 2 s) // s + 1`` (0: none)."""
    n = int(max_len)
    for s, p in zip(STRIDES, PADDINGS):
        n = (n + 2 * p - 2 * s) // s + 1 if n + 2 * p >= 2 * s else 0
    return n


def cpc_config(**over) -> dict:
    """The default ``config`` of a checkpoint (``vars(get_default_cpc_config())``); ``over`` replaces fields."""
    c = dict(_DEFAULTS)
    c.update(over)
    return c


def validate_config(config: dict, where: str = "config") -> dict:
    """Checks that a checkpoint's config, overlaid on the defaults, is served; returns ``{"num_layers": nLevelsGRU}``.
    Anything else raises ``ValueError`` naming the field."""
    if not isinstance(config, dict):
        raise ValueError(f"{where}: config must be a dict of the training arguments, not {type(config).__name__}")
    c = cpc_config(**config)
    served = {"encoder_type": ("cpc",), "normMode": ("layerNorm",), "arMode": ("LSTM",), "cpc_mode": (None, "none")}
    for key, ok in served.items():
        if c[key] not in ok:
            raise ValueError(f"{where}: {key}={c[key]!r} is not served (served: {', '.join(map(repr, ok))})")
    for key in ("hiddenEncoder", "hiddenGar"):
        if c[key] != HIDDEN:
            raise ValueError(f"{where}: {key}={c[key]!r} is not served (served: {HIDDEN})")
    if c["samplingType"] == "sequential":
        raise ValueError(f"{where}: samplingType='sequential' is not served: the reference then keeps the LSTM state "
                         "from one call to the next")
    n = c["nLevelsGRU"]
    if not isinstance(n, int) or isinstance(n, bool) or not 1 <= n <= 8:
        raise ValueError(f"{where}: nLevelsGRU must be an integer in 1..8, not {n!r}")
    return {"num_layers": n}


def required_keys(num_layers: int) -> List[str]:
    keys = []
    for i in range(len(STRIDES)):
        keys += [f"gEncoder.conv{i}.weight", f"gEncoder.conv{i}.bias", f"gEncoder.batchNorm{i}.weight",
                 f"gEncoder.batchNorm{i}.bias"]
    for k in range(num_layers):
        keys += [f"gAR.baseNet.{n}_l{k}" for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return keys


def fabricate_cpc_state_dict(seed: int = 0, num_layers: int = 1) -> Dict[str, torch.Tensor]:
    """Deterministic weights with the keys and shapes of the reference's ``CPCModel(CPCEncoder(256, "layerNorm"),
    CPCAR(256, 256, False, num_layers, "LSTM"))``.

    Conv weights are scaled by their fan-in; the ChannelNorm affines are away from (1, 0); LSTM weights are scaled by
    1 / sqrt(256), and the forget-gate biases are raised so that the cell keeps a long memory, which lets rounding
    errors accumulate over the 1000 steps of a 10 s utterance as they would in a trained model."""
    g = torch.Generator().manual_seed(seed)
    H = HIDDEN
    sd: Dict[str, torch.Tensor] = {}
    for i, s in enumerate(STRIDES):
        cin = 1 if i == 0 else H
        sd[f"gEncoder.conv{i}.weight"] = torch.randn(H, cin, 2 * s, generator=g) / math.sqrt(cin * 2 * s)
        sd[f"gEncoder.conv{i}.bias"] = torch.randn(H, generator=g) * 0.1
        sd[f"gEncoder.batchNorm{i}.weight"] = (0.5 + torch.rand(H, generator=g)).view(1, H, 1)
        sd[f"gEncoder.batchNorm{i}.bias"] = (torch.randn(H, generator=g) * 0.2).view(1, H, 1)
    for k in range(num_layers):
        sc = 1.0 / math.sqrt(H)
        sd[f"gAR.baseNet.weight_ih_l{k}"] = (torch.rand(4 * H, H, generator=g) * 2 - 1) * sc
        sd[f"gAR.baseNet.weight_hh_l{k}"] = (torch.rand(4 * H, H, generator=g) * 2 - 1) * sc
        bih = (torch.rand(4 * H, generator=g) * 2 - 1) * sc
        bhh = (torch.rand(4 * H, generator=g) * 2 - 1) * sc
        bhh[H:2 * H] += 2.0  # forget gate: sigmoid(~2) = 0.88, a memory of ~8 steps and more
        sd[f"gAR.baseNet.bias_ih_l{k}"] = bih
        sd[f"gAR.baseNet.bias_hh_l{k}"] = bhh
    return sd


def load_cpc_checkpoint(path: str) -> Tuple[dict, Dict[str, torch.Tensor]]:
    """``(served config, tensors)`` of a reference CPC checkpoint file. A missing encoder or LSTM weight raises
    ``KeyError`` naming it (the reference's ``strict=False`` would keep random weights instead)."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(state, dict) or "config" not in state or "weights" not in state:
        raise ValueError(f"{path}: not a CPC checkpoint (expected a dict with the keys 'config' and 'weights')")
    cfg = validate_config(state["config"], path)
    weights = state["weights"]
    keys = required_keys(cfg["num_layers"])
    missing = [k for k in keys if k not in weights]
    if missing:
        raise KeyError(f"{path}: CPC checkpoint lacks {len(missing)} required tensor(s), first '{missing[0]}'")
    return cfg, {k: weights[k] for k in keys}


class CpcExpert(NativeExpert):
    """``UpstreamExpert`` of modified CPC: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms whose longest has at
    least 159 samples (shorter ones are padded like the reference pads them). ``lanes``, ``global_max_len``, the
    inference-only refusal, the training-mode warning and ``forward_host`` are those of every expert
    (``NativeExpert``). The result dict is the reference's: two hidden states [B, T, 256] (the encoder's output, then
    the last LSTM layer's), ``last_hidden_state``, ``hidden_state_{i}`` and ``_hidden_states_info``."""

    model_label = "modified CPC"
    min_batch_samples = MIN_BATCH_SAMPLES
    hidden_size = HIDDEN
    num_outputs = 2

    def __init__(self, ckpt: Optional[str] = None, name: str = "modified_cpc", seed: int = 0,
                 randomize_seed: Optional[int] = None, hooks=None, feature_selection=None, **kwargs):
        if hooks or feature_selection is not None:
            raise TypeError("hooks and feature_selection are not available for modified CPC: the reference expert "
                            "registers its hooks itself (cpc/expert.py); use the default hidden_states")
        if ckpt is not None:
            cfg, sd = load_cpc_checkpoint(ckpt)
        else:
            cfg = validate_config(cpc_config())
            sd = fabricate_cpc_state_dict(seed, cfg["num_layers"])
        if randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights of the same shape
            sd = fabricate_cpc_state_dict(randomize_seed, cfg["num_layers"])
        super().__init__(sd)
        self.name = name
        self.cfg = cfg
        self.num_layers = self.num_outputs

    def _native_args(self):
        n = self.cfg["num_layers"]
        cfg = _lib.S3BCpcConfig(hidden=HIDDEN, num_layers=n)
        return "s3b_cpc_model_create", cfg, {k: self._state_dict_host[k] for k in required_keys(n)}

    def get_downsample_rates(self, key: str) -> int:
        return DOWNSAMPLE_RATE

    def num_frames(self, max_len: int) -> int:
        return num_frames(max_len)

    def forward(self, wavs: List[torch.Tensor]) -> Dict:
        out = self._forward_ex(*self._prepare(wavs))
        hidden = (out[0], out[1])
        result = {"_hidden_states_info": HIDDEN_STATES_INFO, "hidden_states": hidden, "last_hidden_state": hidden[-1]}
        for i, h in enumerate(hidden):
            result[f"hidden_state_{i}"] = h
        return result
