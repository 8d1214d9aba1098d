"""SSAST (``ssast_frame_base``, ``ssast_patch_base``) backed by the sm_90a C-ABI library.

The reference (s3prl/upstream/ssast/{expert,audio,ast_models}.py) cuts every utterance, zero-padded, into
``nseg = len(range(0, max_len, S))`` windows of ``S = int(window_secs * 16000)`` samples and runs each window alone:
kaldi fbank (128 mel bins, hanning window), ``(y + 4.2677393) / (4.5689974 * 2)``, zero rows up to ``target_length =
int(window_secs * 16000 / 160)``, then the fine-tuning ``ASTModel``: a patch-embedding Conv2d over the [128, target_length]
spectrogram (frame model ``base_f``: kernel (128, 2), stride (128, 1); patch model ``base_p``: kernel (16, 16), stride
(10, 10)), ``[cls_token, dist_token, patches] + pos_embed`` and 12 pre-LN DeiT blocks (LayerNorm eps 1e-6). The 12
hidden states are the block outputs without the class tokens and without the final ``v.norm``; the patch model folds
its 12 frequency patches into channels. The time axis is trimmed to ``len(range(0, max_len, rate))``, rate 160 (frame)
or 1600 (patch).

Checkpoint: the reference's DataParallel ``state_dict`` (``module.v.*``, ``module.p_input_fdim``,
``module.p_input_tdim``). ``cpredlayer``, ``gpredlayer``, ``mask_embed``, ``v.norm``, ``v.head`` and ``v.head_dist`` are
ignored. The positional table is re-gridded once at load, with the branches of ``ASTModel.__init__`` (fine-tuning): the
checkpoint's [p_f_dim, p_t_dim] patch table is centre-cropped in time when the window has fewer time patches, else
bilinearly interpolated to (8, t_dim); then interpolated to (f_dim, t_dim). A missing tensor raises ``KeyError`` naming
it; a patch shape other than (128, 2) / (16, 16) or not the entry's, an embedding width other than 768, and a window
too short for one patch (or longer than 10 s) raise ``ValueError`` naming the field. The released files
(SSAST-Base-Frame-400.pth, SSAST-Base-Patch-400.pth) are not reachable offline: ``fabricate_ssast_state_dict`` writes
their believed format (frame: 128 x 2 patches at pretraining stride (128, 2), ``p_input_tdim`` 1024; patch: 16 x 16 at
stride 16, 1024), which was not checked against them.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from .. import lib as _lib
from .expert import NativeExpert

SAMPLE_RATE = 16000
FBANK_STRIDE = 160
EMBED, HEADS, LAYERS, FFN = 768, 12, 12, 3072
NUM_BINS = 128
# kind -> (patch shape (fshape, tshape), fine-tuning stride (fstride, tstride))
KINDS = {"frame": ((128, 2), (128, 1)), "patch": ((16, 16), (10, 10))}
MAX_WINDOW_SAMPLES = 160000


def geometry(kind: str, window_secs: float) -> Dict[str, int]:
    """The window's sizes as the reference derives them: S samples, TL feature rows, f_dim x t_dim patches (P of them)
    and the output frame rate. Refuses a window the model cannot run with a ``ValueError`` naming window_secs."""
    if kind not in KINDS:
        raise ValueError(f"kind={kind!r} is not served (served: 'frame', 'patch')")
    (fs, ts), (fst, tst) = KINDS[kind]
    S = int(window_secs * SAMPLE_RATE)
    TL = int(window_secs * SAMPLE_RATE / FBANK_STRIDE)
    if TL != S // FBANK_STRIDE:
        raise ValueError(f"window_secs={window_secs!r}: target_length {TL} is not the window's {S} samples // 160")
    if TL < ts or S < 400:
        raise ValueError(f"window_secs={window_secs!r} is too short for one {fs} x {ts} patch (needs >= "
                         f"{max(ts * FBANK_STRIDE, 400) / SAMPLE_RATE} s)")
    if S > MAX_WINDOW_SAMPLES:
        raise ValueError(f"window_secs={window_secs!r}: windows up to {MAX_WINDOW_SAMPLES / SAMPLE_RATE:g} s are served")
    f_dim = (NUM_BINS - fs) // fst + 1
    t_dim = (TL - ts) // tst + 1
    return {"S": S, "TL": TL, "f_dim": f_dim, "t_dim": t_dim, "P": f_dim * t_dim, "rate": FBANK_STRIDE * tst}


def num_segments(window_samples: int, max_len: int) -> int:
    return len(range(0, max_len, window_samples))


def num_frames(kind: str, window_secs: float, max_len: int) -> int:
    """Frames of a batch padded to max_len: the windows' time patches, trimmed to len(range(0, max_len, rate))."""
    g = geometry(kind, window_secs)
    return min(num_segments(g["S"], max_len) * g["t_dim"], len(range(0, max_len, g["rate"])))


def fabricate_ssast_state_dict(seed: int = 0, kind: str = "frame") -> Dict[str, torch.Tensor]:
    """Deterministic weights in the believed format of the released pretraining checkpoints: the DataParallel
    ``state_dict`` of a pretraining ``ASTModel`` (``vit_deit_base_distilled_patch16_384`` blocks), patch shape
    (128, 2) or (16, 16) at a stride equal to it, ``p_input_fdim`` 128 and ``p_input_tdim`` 1024, with the
    pretraining heads. Scales keep activations in the range of a trained ViT: LayerNorm gains near 1, linear weights
    of fan-in variance, positional and class tokens of std 0.02 like ``trunc_normal_``."""
    (fs, ts), _ = KINDS[kind]
    g = torch.Generator().manual_seed(seed)
    D = EMBED
    p_f, p_t = (NUM_BINS - fs) // fs + 1, (1024 - ts) // ts + 1

    def lin(n, k):
        return torch.randn(n, k, generator=g) / math.sqrt(k), torch.randn(n, generator=g) * 0.02

    sd: Dict[str, torch.Tensor] = {}
    v = "module.v."
    sd[v + "cls_token"] = torch.randn(1, 1, D, generator=g) * 0.02
    sd[v + "dist_token"] = torch.randn(1, 1, D, generator=g) * 0.02
    sd[v + "pos_embed"] = torch.randn(1, 2 + p_f * p_t, D, generator=g) * 0.02
    sd[v + "patch_embed.proj.weight"] = torch.randn(D, 1, fs, ts, generator=g) / math.sqrt(fs * ts)
    sd[v + "patch_embed.proj.bias"] = torch.randn(D, generator=g) * 0.02
    for l in range(LAYERS):
        p = f"{v}blocks.{l}."
        for n in ("norm1", "norm2"):
            sd[p + n + ".weight"] = 1.0 + 0.1 * torch.randn(D, generator=g)
            sd[p + n + ".bias"] = 0.05 * torch.randn(D, generator=g)
        for n, (o, i) in (("attn.qkv", (3 * D, D)), ("attn.proj", (D, D)), ("mlp.fc1", (FFN, D)), ("mlp.fc2", (D, FFN))):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = lin(o, i)
    sd[v + "norm.weight"] = 1.0 + 0.1 * torch.randn(D, generator=g)
    sd[v + "norm.bias"] = 0.05 * torch.randn(D, generator=g)
    sd[v + "head.weight"], sd[v + "head.bias"] = lin(1000, D)
    sd[v + "head_dist.weight"], sd[v + "head_dist.bias"] = lin(1000, D)
    for head in ("cpredlayer", "gpredlayer"):
        sd[f"module.{head}.0.weight"], sd[f"module.{head}.0.bias"] = lin(D, D)
        sd[f"module.{head}.2.weight"], sd[f"module.{head}.2.bias"] = lin(256, D)
    sd["module.mask_embed"] = torch.randn(1, 1, D, generator=g) * 0.02
    sd["module.p_input_fdim"] = torch.tensor(NUM_BINS)
    sd["module.p_input_tdim"] = torch.tensor(1024)
    return sd


def required_keys() -> List[str]:
    """The checkpoint tensors the forward reads (``module.``-prefixed, as the reference's DataParallel file)."""
    v = "module.v."
    keys = ["module.p_input_fdim", "module.p_input_tdim"]
    keys += [v + k for k in ("cls_token", "dist_token", "pos_embed", "patch_embed.proj.weight", "patch_embed.proj.bias")]
    for l in range(LAYERS):
        for n in ("norm1", "norm2", "attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"):
            keys += [f"{v}blocks.{l}.{n}.weight", f"{v}blocks.{l}.{n}.bias"]
    return keys


def regrid_pos_embed(pos: torch.Tensor, p_f_dim: int, p_t_dim: int, f_dim: int, t_dim: int) -> torch.Tensor:
    """The fine-tuning positional table [1, 2 + f_dim * t_dim, D] from the checkpoint's [1, 2 + p_f_dim * p_t_dim, D],
    by the branches of ``ASTModel.__init__`` (pretrain_stage=False). Its ``f_dim < p_f_dim`` branch cannot occur with
    128 bins and either served patch shape, and is refused rather than mirrored."""
    D = pos.shape[-1]
    if f_dim < p_f_dim:
        raise ValueError(f"f_dim={f_dim} < p_f_dim={p_f_dim}: a frequency crop of the positional table is not served")
    pos = pos.detach().float()
    new = pos[:, 2:, :].reshape(1, p_f_dim * p_t_dim, D).transpose(1, 2).reshape(1, D, p_f_dim, p_t_dim)
    if t_dim < p_t_dim:
        lo = int(p_t_dim / 2) - int(t_dim / 2)
        new = new[:, :, :, lo:lo + t_dim]
    else:
        new = F.interpolate(new, size=(8, t_dim), mode="bilinear")
    new = F.interpolate(new, size=(f_dim, t_dim), mode="bilinear")
    new = new.reshape(1, D, f_dim * t_dim).transpose(1, 2)
    return torch.cat([pos[:, :2, :], new], dim=1).contiguous()


def prepare_ssast_tensors(sd: Dict[str, torch.Tensor], kind: str, window_secs: float,
                          where: str = "checkpoint") -> Dict[str, torch.Tensor]:
    """The tensors the library reads (timm names of ``ASTModel.v``, the positional table re-gridded to the window)
    from a reference checkpoint's ``state_dict``. Refuses a missing tensor (``KeyError``) and an unserved checkpoint or
    window (``ValueError``), naming them."""
    missing = [k for k in required_keys() if k not in sd]
    if missing:
        raise KeyError(f"{where}: SSAST checkpoint lacks {len(missing)} required tensor(s), first '{missing[0]}'")
    g = geometry(kind, window_secs)
    (fs, ts), _ = KINDS[kind]
    w = sd["module.v.patch_embed.proj.weight"]
    if w.dim() != 4 or tuple(w.shape[2:]) not in [s for s, _ in KINDS.values()]:
        raise ValueError(f"{where}: module.v.patch_embed.proj.weight has shape {tuple(w.shape)}: patch shapes (128, 2) "
                         "and (16, 16) are served")
    if tuple(w.shape[2:]) != (fs, ts):
        raise ValueError(f"{where}: module.v.patch_embed.proj.weight has patch shape {tuple(w.shape[2:])}, the {kind} "
                         f"model needs ({fs}, {ts})")
    if w.shape[0] != EMBED or w.shape[1] != 1:
        raise ValueError(f"{where}: module.v.patch_embed.proj.weight has shape {tuple(w.shape)}: embed width {EMBED} "
                         "and one input channel are served (base only)")
    for k in ("cls_token", "dist_token", "pos_embed"):
        t = sd["module.v." + k]
        if t.dim() != 3 or t.shape[0] != 1 or t.shape[-1] != EMBED:
            raise ValueError(f"{where}: module.v.{k} has shape {tuple(t.shape)}: embed width {EMBED} is served")
    p_fdim, p_tdim = int(sd["module.p_input_fdim"]), int(sd["module.p_input_tdim"])
    p_f_dim, p_t_dim = (p_fdim - fs) // fs + 1, (p_tdim - ts) // ts + 1
    pos = sd["module.v.pos_embed"]
    if pos.shape[1] != 2 + p_f_dim * p_t_dim:
        raise ValueError(f"{where}: module.v.pos_embed has {pos.shape[1]} rows; module.p_input_fdim / p_input_tdim "
                         f"({p_fdim}, {p_tdim}) give 2 + {p_f_dim} x {p_t_dim}")
    out = {"pos_embed": regrid_pos_embed(pos, p_f_dim, p_t_dim, g["f_dim"], g["t_dim"])}
    for k in required_keys():
        if k.startswith("module.v.") and k != "module.v.pos_embed":
            out[k[len("module.v."):]] = sd[k].detach().to("cpu", torch.float32).contiguous()
    return out


def load_ssast_checkpoint(path: str) -> Dict[str, torch.Tensor]:
    """The ``state_dict`` of a reference SSAST checkpoint file (DataParallel keys)."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    if not isinstance(state, dict) or "module.v.patch_embed.proj.weight" not in state:
        raise ValueError(f"{path}: not an SSAST checkpoint (expected the DataParallel state_dict of an ASTModel, "
                         "with module.v.patch_embed.proj.weight)")
    return state


class SsastExpert(NativeExpert):
    """``UpstreamExpert`` of SSAST: ``expert(wavs)`` on a list of 1-D fp32 CUDA waveforms returns the reference's
    ``{"hidden_states": [block 1, ..., block 12]}``, 12 tensors [B, T, 768] (frame model) or [B, T, 12 * 768] (patch
    model), at a downsample rate of 160 or 1600. ``lanes``, ``global_max_len``, the inference-only refusal, the
    training-mode warning and ``forward_host`` are those of every expert (``NativeExpert``)."""

    model_label = "SSAST"
    min_batch_samples = 1
    num_outputs = LAYERS

    def __init__(self, ckpt: Optional[str] = None, name: str = "ssast_frame_base", kind: str = "frame",
                 window_secs: float = 1.0, seed: int = 0, randomize_seed: Optional[int] = None, hooks=None,
                 feature_selection=None, **kwargs):
        if hooks or feature_selection is not None:
            raise TypeError("hooks and feature_selection are not available for SSAST: the reference expert registers "
                            "none (ssast/expert.py); use the default hidden_states")
        self.geom = geometry(kind, window_secs)
        if ckpt is not None:
            sd, where = load_ssast_checkpoint(ckpt), ckpt
        else:
            sd, where = None, name
        if sd is None or randomize_seed is not None:  # S3PRLUpstream(randomize=True): fresh weights, same shapes
            sd = fabricate_ssast_state_dict(seed if randomize_seed is None else randomize_seed, kind)
        super().__init__(prepare_ssast_tensors(sd, kind, window_secs, where))
        self.name = name
        self.kind = kind
        self.window_secs = window_secs
        self.num_layers = LAYERS

    def _native_args(self):
        cfg = _lib.S3BSsastConfig(patch=int(self.kind == "patch"), window_samples=self.geom["S"], embed_dim=EMBED,
                                  num_heads=HEADS, num_layers=LAYERS)
        return "s3b_ssast_model_create", cfg, self._state_dict_host

    def get_downsample_rates(self, key: str = None) -> int:
        return self.geom["rate"]

    @property
    def hidden_size(self) -> int:
        return self.geom["f_dim"] * EMBED

    def num_frames(self, max_len: int) -> int:
        return num_frames(self.kind, self.window_secs, max_len)

    def forward(self, wavs: List[torch.Tensor]) -> Dict:
        out = self._forward_ex(*self._prepare(wavs))
        return {"hidden_states": [out[i] for i in range(self.num_outputs)]}
