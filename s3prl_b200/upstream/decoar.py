"""DeCoAR (``decoar``, ``decoar_layers`` and their hub variants) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/decoar/{expert,decoar,audio}.py, decoar_layers/{expert,decoar}.py) runs, per utterance,
kaldi fbank with a hamming window (80 bins) and CMVN over all frames with the unbiased std, pads the features to
T = max m, projects them with ``post_extract_proj = Linear(80, 1024)`` and feeds the packed sequences through two
4-layer ``nn.LSTM(1024, 1024)`` stacks: ``forward_lstm`` in time order and ``backward_lstm`` over each utterance
reversed within its own length, its output flipped back. Each layer's output is ``cat(forward, backward)``
[B, T, 2048], zero at frames t >= m_b. ``decoar`` returns the last layer, ``decoar_layers`` all four. Here the whole
forward is one ``s3b_forward`` of a model made by ``s3b_decoar_model_create``: the fbank and CMVN kernels, GEMMs for
post_extract_proj and every layer's input projections, and a grid-resident kernel for each recurrence. That kernel
needs the whole device, so a forward always runs as one lane.

Checkpoint: the reference's ``{"model": state_dict}`` file (decoar/expert.py). Both experts read the same keys
(``decoar_layers`` only renames them into its ModuleList). The reference loads with ``strict=False``, which keeps
random weights for a missing key; here a missing key raises and is named. Other keys are ignored. The released
checkpoint is not reachable offline; without a file the experts use a fabricated checkpoint of the same shape.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from .. import lib as _lib
from .expert import NativeExpert

HIDDEN = 1024
NUM_LAYERS = 4
NUM_MEL_BINS = 80
OUTPUT_DIM = 2 * HIDDEN
# kaldi fbank frames m = 1 + (n - 400) // 160; the CMVN's unbiased std needs m >= 2
MIN_SAMPLES = 560
DOWNSAMPLE_RATE = 160  # decoar/expert.py get_downsample_rates


def num_frames(n: int) -> int:
    """Frames of one utterance of n samples (or of a batch padded to n)."""
    return 0 if n < 400 else 1 + (n - 400) // 160


def required_keys() -> List[str]:
    keys = ["post_extract_proj.weight", "post_extract_proj.bias"]
    for d in ("forward", "backward"):
        for k in range(NUM_LAYERS):
            keys += [f"{d}_lstm.{n}_l{k}" for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return keys


def fabricate_decoar_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic weights with the keys and shapes of the reference's ``Decoar().state_dict()``.

    PyTorch's default LSTM initialisation forgets within a few frames. These weights keep a long memory instead: the
    forget gate's bias (rows 1024..2047 of ``bias_ih``) is drawn per unit from [2, 7] (f between 0.88 and 0.999), so
    that what the first frames write is still visible hundreds of frames later, as in a trained model. W_ih and W_hh
    are drawn at 0.7 / sqrt(H) and 0.2 / sqrt(H). With both at 1 / sqrt(H) the 4-layer stacks amplify rounding (fp32
    against fp64 differs by 2.5e-3 in the last layer of a 10 s utterance); with these scales a relative perturbation
    of 1e-5 in the features moves the last layer by 3.5e-5, so that a parity test measures the implementation rather
    than the amplification."""
    g = torch.Generator().manual_seed(seed)
    H = HIDDEN
    sd: Dict[str, torch.Tensor] = {
        "post_extract_proj.weight": torch.randn(H, NUM_MEL_BINS, generator=g) / math.sqrt(NUM_MEL_BINS),
        "post_extract_proj.bias": torch.randn(H, generator=g) * 0.1,
    }
    for d in ("forward", "backward"):
        for k in range(NUM_LAYERS):
            p = f"{d}_lstm."
            sd[p + f"weight_ih_l{k}"] = torch.randn(4 * H, H, generator=g) * (0.7 / math.sqrt(H))
            sd[p + f"weight_hh_l{k}"] = torch.randn(4 * H, H, generator=g) * (0.2 / math.sqrt(H))
            b_ih = torch.randn(4 * H, generator=g) * 0.1
            b_ih[H:2 * H] += 2.0 + 5.0 * torch.rand(H, generator=g)
            sd[p + f"bias_ih_l{k}"] = b_ih
            sd[p + f"bias_hh_l{k}"] = torch.randn(4 * H, generator=g) * 0.1
    return sd


def load_decoar_checkpoint(path: str) -> Dict[str, torch.Tensor]:
    """The served tensors of a reference DeCoAR checkpoint file; a missing key raises ``KeyError`` naming it."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(state, dict) or "model" not in state:
        raise ValueError(f"{path}: not a DeCoAR checkpoint (expected a dict with the key 'model')")
    weights = state["model"]
    missing = [k for k in required_keys() if k not in weights]
    if missing:
        raise KeyError(f"{path}: DeCoAR checkpoint lacks {len(missing)} required tensor(s), first '{missing[0]}'")
    return {k: weights[k] for k in required_keys()}


class DecoarExpert(NativeExpert):
    """``UpstreamExpert`` of DeCoAR: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms of at least 560 samples.
    ``global_max_len`` (sharding), the inference-only refusal, the training-mode warning and ``forward_host`` (its
    pinned result reused across calls of the same shape) are those of every expert (``NativeExpert``); ``lanes`` is
    accepted but a forward always runs as one lane. The result dict is the reference's: ``hidden_states``
    (``decoar``: the last layer; ``decoar_layers`` with ``all_layers``: all four) of shape [B, T, 2048] and
    ``last_hidden_state``."""

    min_samples = MIN_SAMPLES
    model_label = "DeCoAR"
    hidden_size = OUTPUT_DIM

    def __init__(self, ckpt: Optional[str] = None, all_layers: bool = False, name: Optional[str] = None,
                 seed: int = 0, randomize_seed: Optional[int] = None, hooks=None, feature_selection=None, **kwargs):
        if hooks or feature_selection is not None:
            raise TypeError("hooks and feature_selection are not available for DeCoAR: use the default hidden_states")
        sd = load_decoar_checkpoint(ckpt) if ckpt is not None else fabricate_decoar_state_dict(seed)
        if randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights of the same shape
            sd = fabricate_decoar_state_dict(randomize_seed)
        super().__init__(sd)
        self.name = name or ("decoar_layers" if all_layers else "decoar")
        self.all_layers = bool(all_layers)

    def _native_args(self):
        cfg = _lib.S3BDecoarConfig(num_layers=NUM_LAYERS, hidden=HIDDEN, all_layers=int(self.all_layers))
        return "s3b_decoar_model_create", cfg, {k: self._state_dict_host[k] for k in required_keys()}

    def get_downsample_rates(self, key: str) -> int:
        return DOWNSAMPLE_RATE

    @property
    def num_outputs(self) -> int:
        return NUM_LAYERS if self.all_layers else 1

    def num_frames(self, max_len: int) -> int:
        return num_frames(max_len)

    def forward(self, wavs: List[torch.Tensor]) -> Dict:
        out = self._forward_ex(*self._prepare(wavs))
        return {"hidden_states": [out[i] for i in range(self.num_outputs)], "last_hidden_state": out[-1]}
