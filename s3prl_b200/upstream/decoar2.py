"""DeCoAR 2.0 (``decoar2``) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/decoar2/{expert,decoar2,audio}.py) runs, per utterance, kaldi fbank with a hamming
window, CMVN over all frames and keeps every second frame; the padded batch goes through ``post_extract_proj``
(Linear(80, 768)) and the wav2vec 2.0 ``TransformerEncoder`` of ``wav2vec2_base_960`` (12 post-LN layers, pos_conv
128 / 16). Here the whole forward is one ``s3b_forward`` of a model created with ``frontend = 1``. The result dict is
the reference's: 13 hidden states (the input of every encoder layer and the encoder output), ``last_hidden_state``,
``hidden_state_{i}`` and ``_hidden_states_info``.

Checkpoint: the reference's ``{"model": Decoar2().state_dict()}`` file (decoar2/expert.py:19-26). Only
``post_extract_proj.*`` and ``encoder.*`` are read; other keys are ignored. Where the reference's
``load_state_dict(strict=False)`` would silently keep a random initialisation for a missing key, this expert raises.
The key layout of the released ``checkpoint_decoar2.pt`` was not checked (the file is not reachable offline); it is
assumed to be the reference model's own.
"""
from __future__ import annotations

import math
from dataclasses import replace
from typing import Dict, List, Optional

import torch

from .configs import ARCHS
from .expert import UpstreamExpert
from .weights import fabricate_state_dict

# decoar2/decoar2.py:9-24: the wav2vec2_base_960 encoder behind Linear(80, 768). Not an ARCHS entry: ARCHS is the table
# of conv-stack models (oracle, goldens and reference runtime iterate over it).
DECOAR2 = replace(ARCHS["wav2vec2_base_960"], frontend="fbank")
NUM_MEL_BINS = 80
# kaldi fbank frames m = 1 + (n - 400) // 160; the CMVN's unbiased std needs m >= 2
MIN_SAMPLES = 560
DOWNSAMPLE_RATE = 320  # decoar2/expert.py:64-65


def num_frames(n: int) -> int:
    """Frames of one utterance of n samples (or of a batch padded to n): ``len(FeatureExtractor()(wav))``."""
    return 0 if n < 400 else (1 + (n - 400) // 160 + 1) // 2


def fabricate_decoar2_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic weights with the keys and shapes of ``Decoar2().state_dict()``: the encoder of the fabricated
    wav2vec2_base_960 checkpoint and a Linear(80, 768) sized for unit-variance (CMVN'd) inputs."""
    sd = {k: v for k, v in fabricate_state_dict(DECOAR2, seed).items() if k.startswith("encoder.")}
    g = torch.Generator().manual_seed(seed)
    D = DECOAR2.encoder_embed_dim
    sd["post_extract_proj.weight"] = torch.randn(D, NUM_MEL_BINS, generator=g) / math.sqrt(NUM_MEL_BINS)
    sd["post_extract_proj.bias"] = torch.randn(D, generator=g) * 0.05
    return sd


def required_keys() -> List[str]:
    return sorted(fabricate_decoar2_state_dict(0))


def load_decoar2_checkpoint(path: str) -> Dict[str, torch.Tensor]:
    """The tensors the model needs from a ``{"model": state_dict}`` file; a missing one raises and is named."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(state, dict) or "model" not in state:
        raise ValueError(f"{path}: not a DeCoAR 2.0 checkpoint (expected a dict with the key 'model')")
    weights = state["model"]
    missing = [k for k in required_keys() if k not in weights]
    if missing:
        raise KeyError(f"{path}: DeCoAR 2.0 checkpoint lacks {len(missing)} required tensor(s), first '{missing[0]}'")
    return {k: weights[k] for k in required_keys()}


class Decoar2Expert(UpstreamExpert):
    """``UpstreamExpert`` of DeCoAR 2.0: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms of at least 560
    samples. ``lanes``, ``global_max_len`` (sharding) and ``forward_host`` work as for the wav2vec 2.0 experts."""

    min_samples = MIN_SAMPLES
    model_label = "DeCoAR 2.0"

    def __init__(self, ckpt: Optional[str] = None, randomize_seed: Optional[int] = None, seed: int = 0, **kwargs):
        # the reference's expert swallows every other keyword (decoar2/expert.py:19); so does this one
        if randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights of the same architecture
            sd = fabricate_decoar2_state_dict(randomize_seed)
        elif ckpt is not None:
            sd = load_decoar2_checkpoint(ckpt)
        else:
            sd = fabricate_decoar2_state_dict(seed)
        super().__init__(name="decoar2", arch=DECOAR2, state_dict=sd)

    def get_downsample_rates(self, key: str) -> int:
        return DOWNSAMPLE_RATE

    def num_frames(self, max_len: int) -> int:
        return num_frames(max_len)
