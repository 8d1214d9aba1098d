"""APC and VQ-APC (``apc``, ``vq_apc`` and their hub variants) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/apc/{expert,apc,audio}.py, vq_apc/expert.py) runs, per utterance, kaldi fbank with a
hamming window (80 bins) and CMVN over all frames with the unbiased std, pads the features to T = max m, and feeds the
packed sequences through three single-layer ``nn.GRU(512)``; from layer 1 on each layer adds its input when ``residual``
is set. Its fixed hooks expose the input of ``rnn_layers[1]``, the input of ``rnn_layers[2]`` and the model's feature
output, i.e. the outputs of layers 0, 1 and 2; frames t >= m_b are exactly zero. Here the whole forward is one
``s3b_forward`` of a model made by ``s3b_apc_model_create``: the fbank and CMVN kernels, one GEMM per layer for the
input projections, and a thread-block-cluster kernel for each recurrence.

VQ-APC uses the same expert. Its VQ layers quantise the last layer's output only after that output has been recorded
as a hidden state (apc.py:141-156), so they never change a hidden state: ``vq_layers.*`` and ``postnet.*`` are read
and ignored.

Checkpoint: the reference's ``{"config": {...}, "model": APC.state_dict()}`` file (apc/expert.py:20-26). Served:
fbank features with ``feat_dim`` 80 and CMVN, ``hidden_size`` 512, ``num_layers`` 3, ``residual`` true or false.
The released checkpoints (apc_360hr, apc_960hr, vq_apc_360hr, vq_apc_960hr) are not reachable offline; their configs
are believed to be hidden_size 512, num_layers 3, residual true, but that was not checked. Without a file the experts
use a fabricated checkpoint of that shape.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from .. import lib as _lib
from .expert import NativeExpert

HIDDEN = 512
NUM_LAYERS = 3
NUM_MEL_BINS = 80
# kaldi fbank frames m = 1 + (n - 400) // 160; the CMVN's unbiased std needs m >= 2
MIN_SAMPLES = 560
DOWNSAMPLE_RATE = 160  # apc/expert.py:44-45
HIDDEN_STATES_INFO = ("self.model.rnn_layers[1]", "self.model.rnn_layers[2]", "self.model")
# audio kwargs of config["data"]["audio"] that reach kaldi.fbank, accepted at their default value only
_FBANK_DEFAULTS = {"frame_length": 25.0, "frame_shift": 10.0}


def num_frames(n: int) -> int:
    """Frames of one utterance of n samples (or of a batch padded to n): ``len(FeatureExtractor()(wav))``."""
    return 0 if n < 400 else 1 + (n - 400) // 160


def apc_config(residual: bool = True, vq: bool = False) -> dict:
    """The ``config`` entry of a checkpoint of the served shape (apc/expert.py:22-25)."""
    paras = {"hidden_size": HIDDEN, "num_layers": NUM_LAYERS, "dropout": 0.1, "residual": residual}
    if vq:
        paras["vq"] = {"codebook_size": [128], "code_dim": [HIDDEN], "gumbel_temperature": 0.5}
    return {"data": {"audio": {"feat_type": "fbank", "feat_dim": NUM_MEL_BINS, "frame_length": 25, "frame_shift": 10,
                               "decode_wav": False, "cmvn": True}},
            "model": {"paras": paras}}


def fabricate_apc_state_dict(seed: int = 0, vq: bool = False) -> Dict[str, torch.Tensor]:
    """Deterministic weights with the keys and shapes of ``APC(80, **apc_config(vq=vq)["model"]["paras"])``.

    PyTorch's default GRU initialisation forgets within a few frames. These weights keep a long memory instead: the
    update gate's bias is drawn per unit from [2, 7] (z between 0.88 and 0.999), so that what the first frames write
    is still visible hundreds of frames later, as in a trained model."""
    g = torch.Generator().manual_seed(seed)
    H = HIDDEN
    sd: Dict[str, torch.Tensor] = {}
    for l in range(NUM_LAYERS):
        k = NUM_MEL_BINS if l == 0 else H
        p = f"rnn_layers.{l}."
        sd[p + "weight_ih_l0"] = torch.randn(3 * H, k, generator=g) / math.sqrt(k)
        sd[p + "weight_hh_l0"] = torch.randn(3 * H, H, generator=g) / math.sqrt(H)
        b_ih = torch.randn(3 * H, generator=g) * 0.1
        b_ih[H:2 * H] += 2.0 + 5.0 * torch.rand(H, generator=g)
        sd[p + "bias_ih_l0"] = b_ih
        sd[p + "bias_hh_l0"] = torch.randn(3 * H, generator=g) * 0.1
    if vq:
        cs = 128
        sd["vq_layers.0.vq_logits.weight"] = torch.randn(cs, H, generator=g) / math.sqrt(H)
        sd["vq_layers.0.vq_logits.bias"] = torch.randn(cs, generator=g) * 0.1
        sd["vq_layers.0.codebook_CxE.weight"] = torch.randn(H, cs, generator=g) / math.sqrt(cs)
    sd["postnet.weight"] = torch.randn(NUM_MEL_BINS, H, generator=g) / math.sqrt(H)
    sd["postnet.bias"] = torch.randn(NUM_MEL_BINS, generator=g) * 0.1
    return sd


def required_keys() -> List[str]:
    return [f"rnn_layers.{l}.{n}" for l in range(NUM_LAYERS)
            for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")]


def validate_audio(config: dict, where: str = "config") -> None:
    """Checks that a checkpoint's ``data.audio`` is the served front end (shared by APC and NPC, whose audio.py is
    APC's); anything else raises ``ValueError`` naming the field."""
    try:
        audio = dict(config["data"]["audio"])
    except (KeyError, TypeError) as e:
        raise ValueError(f"{where}: expected config['data']['audio'] and config['model']['paras'] ({e!r} missing)")
    if audio.pop("feat_type", None) != "fbank":
        raise ValueError(f"{where}: data.audio.feat_type must be 'fbank'")
    if audio.pop("feat_dim", None) != NUM_MEL_BINS:
        raise ValueError(f"{where}: data.audio.feat_dim must be {NUM_MEL_BINS}")
    if not audio.pop("cmvn", True):
        raise ValueError(f"{where}: data.audio.cmvn=False is not served (CMVN is part of the front-end kernel)")
    audio.pop("decode_wav", None)  # file decoding only; the expert takes waveforms
    for key, default in _FBANK_DEFAULTS.items():
        if key in audio and float(audio.pop(key)) != default:
            raise ValueError(f"{where}: data.audio.{key} must be {default:g} (the served fbank)")
    if audio:
        raise ValueError(f"{where}: data.audio.{sorted(audio)[0]} is not served (fbank kwargs other than "
                         "frame_length / frame_shift at their defaults)")


def validate_config(config: dict, where: str = "config") -> bool:
    """Checks that a checkpoint's config is of the served shape; returns ``residual``. Anything else raises
    ``ValueError`` naming the field."""
    try:
        config["data"]["audio"]
        paras = dict(config["model"]["paras"])
    except (KeyError, TypeError) as e:
        raise ValueError(f"{where}: expected config['data']['audio'] and config['model']['paras'] ({e!r} missing)")
    validate_audio(config, where)
    if paras.pop("hidden_size", None) != HIDDEN:
        raise ValueError(f"{where}: model.paras.hidden_size must be {HIDDEN}")
    if paras.pop("num_layers", None) != NUM_LAYERS:
        raise ValueError(f"{where}: model.paras.num_layers must be {NUM_LAYERS}")
    if "residual" not in paras:
        raise ValueError(f"{where}: model.paras.residual is missing")
    residual = bool(paras.pop("residual"))
    paras.pop("dropout", None)  # inactive in eval
    paras.pop("vq", None)  # acts after the last hidden state is recorded
    if paras:
        raise ValueError(f"{where}: model.paras.{sorted(paras)[0]} is not an APC parameter")
    return residual


def load_apc_checkpoint(path: str) -> Tuple[bool, Dict[str, torch.Tensor]]:
    """``(residual, tensors)`` of a reference APC / VQ-APC checkpoint file; a missing weight raises and is named."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(state, dict) or "config" not in state or "model" not in state:
        raise ValueError(f"{path}: not an APC checkpoint (expected a dict with the keys 'config' and 'model')")
    residual = validate_config(state["config"], path)
    weights = state["model"]
    missing = [k for k in required_keys() if k not in weights]
    if missing:
        raise KeyError(f"{path}: APC checkpoint lacks {len(missing)} required tensor(s), first '{missing[0]}'")
    return residual, {k: weights[k] for k in required_keys()}


class ApcExpert(NativeExpert):
    """``UpstreamExpert`` of APC / VQ-APC: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms of at least 560
    samples. ``lanes``, ``global_max_len`` (sharding), the inference-only refusal, the training-mode warning and
    ``forward_host`` (its pinned result reused across calls of the same shape) are those of every expert
    (``NativeExpert``). The result dict is the reference's: three hidden states [B, T, 512], ``last_hidden_state``,
    ``hidden_state_{i}`` and ``_hidden_states_info``."""

    min_samples = MIN_SAMPLES
    model_label = "APC"
    num_layers = num_outputs = NUM_LAYERS  # the output of every GRU layer is a hidden state
    hidden_size = HIDDEN

    def __init__(self, ckpt: Optional[str] = None, name: str = "apc", vq: bool = False, seed: int = 0,
                 randomize_seed: Optional[int] = None, hooks=None, feature_selection=None, **kwargs):
        if hooks or feature_selection is not None:
            raise TypeError("hooks and feature_selection are not available for APC: the reference expert registers "
                            "its three hooks itself (apc/expert.py:27-42); use the default hidden_states")
        if ckpt is not None:
            residual, sd = load_apc_checkpoint(ckpt)
        else:
            residual, sd = True, fabricate_apc_state_dict(seed, vq)
        if randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights of the same shape
            sd = fabricate_apc_state_dict(randomize_seed, vq)
        super().__init__(sd)
        self.name = name
        self.residual = residual

    def _native_args(self):
        cfg = _lib.S3BApcConfig(num_layers=NUM_LAYERS, hidden=HIDDEN, residual=int(self.residual))
        return "s3b_apc_model_create", cfg, {k: self._state_dict_host[k] for k in required_keys()}

    def get_downsample_rates(self, key: str) -> int:
        return DOWNSAMPLE_RATE

    def num_frames(self, max_len: int) -> int:
        return num_frames(max_len)

    def forward(self, wavs: List[torch.Tensor]) -> Dict:
        out = self._forward_ex(*self._prepare(wavs))
        hidden = tuple(out[i] for i in range(NUM_LAYERS))
        result = {"_hidden_states_info": HIDDEN_STATES_INFO, "hidden_states": hidden, "last_hidden_state": hidden[-1]}
        for i, h in enumerate(hidden):
            result[f"hidden_state_{i}"] = h
        return result
