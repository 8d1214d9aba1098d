"""``UpstreamExpert`` for wav2vec 2.0 / HuBERT / WavLM backed by the sm_90a C-ABI library.

Mirrors the reference interface (s3prl/upstream/hubert/expert.py:26-72, wav2vec2/expert.py:20-97,
wavlm/expert.py:33-87 and the UpstreamBase result dict, s3prl/upstream/interfaces.py:100-131):

    expert = UpstreamExpert(ckpt=None, name="hubert_base")
    result = expert([wav_0, wav_1, ...])          # list of 1-D fp32 CUDA tensors, un-padded
    result["hidden_states"]                        # tuple of NL+1 tensors [B, T, D] (fp32)
    result["last_hidden_state"], result["hidden_state_{i}"]
    expert.get_downsample_rates("hidden_states")   # 320

``NativeExpert`` is the host side shared with the APC, DeCoAR and DeCoAR 2.0 experts (upstream/{apc,decoar,
decoar2}.py): the model handle, the checks, the native forward calls.

Factory kwargs of the reference experts that are honoured: ``feature_selection`` in {None, "fairseq_layers",
"fairseq_layers_before_residual"} (wav2vec2/expert.py:35-39,81-93) and ``hooks=[(module_path, transform), ...]`` /
``hook_postprocess`` of ``UpstreamBase`` (interfaces.py:74-98) for the module paths ``self.model.encoder.layers[i]``
and ``self.model.encoder`` (the ones the reference experts themselves register).
"""
from __future__ import annotations

import ctypes as C
import re
import warnings
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn

from .. import lib as _lib
from .configs import ALIASES, ARCHS, DOWNSAMPLE_RATE, ArchConfig, get_arch
from .weights import fabricate_state_dict, load_reference_checkpoint

SAMPLE_RATE = 16000


def _c_config(cfg: ArchConfig) -> _lib.S3BConfig:
    c = _lib.S3BConfig()
    c.family = cfg.family_id
    c.extractor_layer_norm = int(cfg.extractor_mode == "layer_norm")
    c.conv_bias = int(cfg.conv_bias)
    c.layer_norm_first = int(cfg.layer_norm_first)
    c.normalize_wav = int(cfg.normalize)
    c.num_layers = cfg.encoder_layers
    c.embed_dim = cfg.encoder_embed_dim
    c.ffn_dim = cfg.encoder_ffn_embed_dim
    c.num_heads = cfg.encoder_attention_heads
    c.pos_conv_kernel = cfg.conv_pos
    c.pos_conv_groups = cfg.conv_pos_groups
    c.relative_position = int(cfg.relative_position_embedding)
    c.num_buckets = cfg.num_buckets
    c.max_distance = cfg.max_distance
    c.gru_rel_pos = int(cfg.gru_rel_pos)
    c.no_feature_layer_norm = int(not cfg.feature_layer_norm)
    c.pred_heads = int(cfg.pred_heads)
    c.pos_conv_depth = int(cfg.pos_conv_depth)
    if cfg.conformer:
        c.conformer = 1
        c.depthwise_kernel = int(cfg.depthwise_conv_kernel_size)
    c.frontend = {"conv": _lib.FRONTEND_CONV, "fbank": _lib.FRONTEND_DECOAR2}[cfg.frontend]
    return c


def _rotary_inv_freq() -> torch.Tensor:
    """RotaryPositionalEmbedding's buffer for 64-wide heads, computed as the reference computes it
    (wav2vec2_model.py:51): a checkpoint without the buffer gets the value the reference model would hold."""
    return 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))


class _NativeModel:
    """Owner of one ``s3b_model`` handle (weights resident on one CUDA device). ``create`` names the library's create
    function (``s3b_model_create``, ``s3b_apc_model_create`` or ``s3b_decoar_model_create``), ``config`` is its
    ctypes config, and every tensor of ``tensors`` is sent before the model is finalized on ``device``."""

    def __init__(self, create: str, config, tensors: Dict[str, torch.Tensor], device: torch.device):
        self.lib = _lib.load()
        _lib.require_gpu()
        self.device = device
        self.handle = C.c_void_p()
        _lib.check(getattr(self.lib, create)(C.byref(config), C.byref(self.handle)))
        try:
            for name, t in tensors.items():
                t = t.detach().to("cpu", torch.float32).contiguous()
                shape = (C.c_int64 * max(t.dim(), 1))(*t.shape)
                _lib.check(
                    self.lib.s3b_model_set_tensor(self.handle, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim())
                )
            with torch.cuda.device(device):
                _lib.check(self.lib.s3b_model_finalize(self.handle))
        except Exception:
            self.close()
            raise

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle:
            self.lib.s3b_model_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class NativeExpert(nn.Module):
    """What every expert backed by one ``s3b_model`` shares. A subclass gives ``_native_args``, ``num_outputs`` (the
    hidden states a forward returns), ``hidden_size`` and ``num_frames``, and ``min_samples`` / ``model_label`` when its
    front end needs a minimum utterance length.

    The forward is inference-only (frozen upstream, the configuration SUPERB uses). The module has no trainable
    parameters: a waveform that requires grad raises, a forward in training mode with autograd enabled warns once
    (``Runner`` calls ``.train()`` on the upstream only under ``-f/--upstream_trainable``, which the launcher
    ``python -m s3prl_b200.run_downstream`` rejects up front). An empty batch, an utterance shorter than
    ``min_samples`` and a batch too short for one frame raise ``ValueError`` before any device work.
    ``lanes`` picks the utterance micro-batches of a device forward, ``global_max_len`` pads every batch to a length
    shared across ranks."""

    min_samples = 0  # per-utterance minimum length (0: none beyond the library's own rules)
    min_batch_samples = 400  # the shortest padded batch the front end makes one frame of
    model_label = ""  # the model's name in the minimum-length message

    def __init__(self, state_dict: Dict[str, torch.Tensor]):
        super().__init__()
        self._state_dict_host = state_dict  # kept on the host until the first device placement
        self._native: Optional[_NativeModel] = None
        self._warned_grad = False
        self.lanes = 0  # 0 = library default; 1 / 2 = utterance micro-batches on that many streams
        self.global_max_len: Optional[int] = None  # set when a batch is sharded across ranks
        # a buffer so that .to(device) / .cuda() tell us where to live, like any nn.Module
        self.register_buffer("_device_anchor", torch.zeros(1), persistent=False)

    def _native_args(self) -> Tuple[str, object, Dict[str, torch.Tensor]]:
        """``(create function, its ctypes config, tensors to send)`` of this expert's model (``_NativeModel``)."""
        raise NotImplementedError

    def _ensure_native(self, device: torch.device) -> _NativeModel:
        if device.type != "cuda":
            raise _lib.S3BError(
                "s3prl_b200 runs on CUDA devices only (sm_90a); there is no CPU fallback. "
                "Move the expert and the waveforms to an H100: expert.to('cuda')."
            )
        if self._native is None or self._native.device != device:
            if self._native is not None:
                self._native.close()
            self._native = _NativeModel(*self._native_args(), device)
        return self._native

    def _batch(self, wavs: Sequence[torch.Tensor]) -> Tuple[List[int], int, int]:
        """``(lens, max_len, T)`` of a batch; refuses what no forward can run."""
        if len(wavs) == 0:
            raise ValueError("empty batch")
        lens = [int(w.numel()) for w in wavs]
        for i, n in enumerate(lens):
            if n < self.min_samples:
                raise ValueError(f"utterance {i} has {n} samples: {self.model_label} needs >= {self.min_samples} (two "
                                 "fbank frames; the reference's CMVN std of a single frame is NaN)")
        max_len = self.global_max_len or max(lens)
        T = self.num_frames(max_len)
        if T < 1:
            raise ValueError(f"waveforms too short ({max_len} samples): the front end needs >= "
                             f"{self.min_batch_samples} samples")
        return lens, max_len, T

    def _prepare(self, wavs: List[torch.Tensor]):
        """The checks of a device forward, then ``(native, fp32 contiguous wavs, lens, max_len, T)``."""
        lens, max_len, T = self._batch(wavs)
        if any(w.requires_grad for w in wavs):
            raise _lib.S3BError(
                "s3prl_b200 upstreams are inference-only (frozen upstream); gradients w.r.t. the waveform "
                "or upstream weights are not available. Do not pass -f/--upstream_trainable."
            )
        if self.training and torch.is_grad_enabled() and not self._warned_grad:
            self._warned_grad = True
            warnings.warn(
                "s3prl_b200 upstream called in training mode with autograd enabled: it has no trainable parameters, "
                "its outputs are constants for autograd (frozen upstream). Fine-tuning the upstream "
                "(-f/--upstream_trainable) is not supported.",
                RuntimeWarning,
                stacklevel=3,
            )
        native = self._ensure_native(wavs[0].device)
        wavs = [w.detach().to(torch.float32).contiguous() for w in wavs]
        return native, wavs, lens, max_len, T

    def _forward_ex(self, native: _NativeModel, wavs: List[torch.Tensor], lens: List[int], max_len: int, T: int,
                    ffn_out: Optional[torch.Tensor] = None, last_residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``s3b_forward_ex`` of a prepared batch into a new [num_outputs, B, T, hidden_size] device tensor;
        ``ffn_out`` / ``last_residual`` are the optional outputs of those names."""
        device, B = wavs[0].device, len(wavs)
        with torch.cuda.device(device):
            out = torch.empty((self.num_outputs, B, T, self.hidden_size), dtype=torch.float32, device=device)
            ptrs = (C.c_void_p * B)(*[w.data_ptr() for w in wavs])
            lens_c = (C.c_int64 * B)(*lens)
            opts = _lib.S3BForwardOpts(lanes=int(self.lanes))
            if ffn_out is not None:
                opts.ffn_out = ffn_out.data_ptr()
            if last_residual is not None:
                opts.last_residual = last_residual.data_ptr()
            _lib.check(
                native.lib.s3b_forward_ex(
                    native.handle, ptrs, lens_c, B, max_len, C.c_void_p(out.data_ptr()),
                    C.c_void_p(torch.cuda.current_stream(device).cuda_stream), C.byref(opts),
                )
            )
        return out

    def forward_host(self, wavs_host: List[torch.Tensor], keep_device: bool = False):
        """End-to-end from HOST buffers through ``s3b_forward_host[_ex]`` (H2D and D2H inside the call).
        Returns a pinned host tensor [num_outputs, B, T, hidden_size], reused across calls of the same shape: it is
        valid until the next ``forward_host``. With ``keep_device`` also the device-resident copy (a torch tensor of
        the same shape) for device-side consumers such as the Featurizer."""
        lens, max_len, T = self._batch(wavs_host)
        native = self._ensure_native(self._device_anchor.device)
        wavs = [w.detach().to("cpu", torch.float32).contiguous() for w in wavs_host]
        B = len(wavs)
        shape = (self.num_outputs, B, T, self.hidden_size)
        out = getattr(self, "_host_out", None)
        if out is None or tuple(out.shape) != shape:
            out = torch.empty(shape, dtype=torch.float32).pin_memory()
            self._host_out = out
        ptrs = (C.c_void_p * B)(*[w.data_ptr() for w in wavs])
        lens_c = (C.c_int64 * B)(*lens)
        with torch.cuda.device(native.device):
            if keep_device:
                dev = torch.empty(shape, dtype=torch.float32, device=native.device)
                torch.cuda.current_stream(native.device).synchronize()  # the call runs on the library's own streams
                _lib.check(native.lib.s3b_forward_host_ex(native.handle, ptrs, lens_c, B, max_len,
                                                          C.c_void_p(out.data_ptr()), C.c_void_p(dev.data_ptr())))
                return out, dev
            _lib.check(native.lib.s3b_forward_host(native.handle, ptrs, lens_c, B, max_len, C.c_void_p(out.data_ptr())))
        return out


_LAYER_PATH = re.compile(r"^self\.model\.encoder\.layers\[(\d+)\]$")
_FEATURE_SELECTIONS = (None, "fairseq_layers", "fairseq_layers_before_residual")


class UpstreamExpert(NativeExpert):
    def __init__(
        self,
        ckpt: Optional[str] = None,
        name: str = "hubert_base",
        model_config: Optional[str] = None,
        seed: int = 0,
        state_dict: Optional[Dict[str, torch.Tensor]] = None,
        arch: Optional[ArchConfig] = None,
        feature_selection: Optional[str] = None,
        hooks: Optional[Sequence[Tuple[str, Callable]]] = None,
        hook_postprocess: Optional[Callable] = None,
        randomize_seed: Optional[int] = None,
        **kwargs,
    ):
        family = (arch or get_arch(name)).family if (arch is not None or ckpt is None) else _family_of(name)
        if ckpt is not None:
            arch, sd = load_reference_checkpoint(ckpt, family)
            if randomize_seed is not None:  # S3PRLUpstream(randomize=True): the ckpt's architecture, fresh weights
                sd = fabricate_state_dict(arch, randomize_seed)
        else:
            arch = arch or get_arch(name)
            if randomize_seed is not None:
                seed = randomize_seed
            sd = state_dict if state_dict is not None else fabricate_state_dict(arch, seed)
        super().__init__(sd)
        self.name = name
        self.arch = arch
        # wav2vec2/expert.py:35-39: only the wav2vec 2.0 expert takes feature_selection
        if feature_selection not in _FEATURE_SELECTIONS:
            raise AssertionError(f"feature_selection must be one of {_FEATURE_SELECTIONS}, got {feature_selection!r}")
        if self.arch.family == "distiller" and (hooks or feature_selection is not None):
            raise TypeError("the Distiller expert takes neither hooks nor feature_selection (distiller/expert.py:18-40)")
        if self.arch.conformer and (hooks or feature_selection is not None):
            raise TypeError(
                "feature_selection and hooks are not available for a Conformer model: its encoder collects no layer "
                "results (wav2vec2_model.py:3199-3200); use the default hidden_states"
            )
        if feature_selection is not None and self.arch.family != "wav2vec2":
            raise TypeError(f"feature_selection is an option of the wav2vec2 experts only (got family {self.arch.family})")
        self.feature_selection = feature_selection
        # UpstreamBase hooks (interfaces.py:74-98): (module_path, transform(input, output)); supported module paths
        # are the ones the reference experts register themselves
        self.hooks: List[Tuple[str, Callable]] = []
        for path, transform in hooks or []:
            if not (_LAYER_PATH.match(path) or path == "self.model.encoder"):
                raise ValueError(
                    f"hook on '{path}' is not available: the native model exposes self.model.encoder.layers[i] "
                    "and self.model.encoder"
                )
            m_ = _LAYER_PATH.match(path)
            if m_ and int(m_.group(1)) >= self.arch.encoder_layers:
                raise ValueError(f"hook on '{path}': the model has {self.arch.encoder_layers} layers")
            self.hooks.append((path, transform))
        self.hook_postprocess = hook_postprocess

    def _native_args(self):
        tensors = {k: t for k, t in self._state_dict_host.items() if torch.is_tensor(t) and t.is_floating_point()}
        if self.arch.conformer:
            for l in range(self.arch.encoder_layers):
                tensors.setdefault(f"encoder.layers.{l}.self_attn.rotary_emb.inv_freq", _rotary_inv_freq())
        return "s3b_model_create", _c_config(self.arch), tensors

    def get_downsample_rates(self, key: str) -> int:
        return DOWNSAMPLE_RATE

    @property
    def num_layers(self) -> int:
        return self.arch.encoder_layers

    @property
    def num_outputs(self) -> int:
        return self.arch.num_outputs

    @property
    def hidden_size(self) -> int:
        return self.arch.encoder_embed_dim

    def num_frames(self, max_len: int) -> int:
        n = max_len
        for k, s in ((10, 5), (3, 2), (3, 2), (3, 2), (3, 2), (2, 2), (2, 2)):
            n = (n - k) // s + 1 if n >= k else 0
        return n

    def valid_frames(self, lens: List[int], max_len: Optional[int] = None) -> List[int]:
        """Number of un-padded frames per utterance (the frame padding mask is ``t >= valid_frames[b]``)."""
        lib = _lib.load()
        B = len(lens)
        max_len = max_len or max(lens)
        arr = (C.c_int64 * B)(*lens)
        out = (C.c_int32 * B)()
        native = self._native
        if native is None:
            # bookkeeping only needs the config: use a throw-away, un-finalized handle (no GPU work)
            h = C.c_void_p()
            cc = _c_config(self.arch)
            _lib.check(lib.s3b_model_create(C.byref(cc), C.byref(h)))
            try:
                _lib.check(lib.s3b_valid_frames(h, arr, B, max_len, out))
            finally:
                lib.s3b_model_destroy(h)
        else:
            _lib.check(lib.s3b_valid_frames(native.handle, arr, B, max_len, out))
        return list(out)

    # ---- the hot path ------------------------------------------------------------------------------
    def forward(self, wavs: List[torch.Tensor]) -> Dict[str, Union[torch.Tensor, tuple]]:
        native, wavs, lens, max_len, T = self._prepare(wavs)
        device, B = wavs[0].device, len(wavs)
        NL, D = self.arch.encoder_layers, self.arch.encoder_embed_dim
        need_ffn = self.feature_selection == "fairseq_layers_before_residual" or bool(self.hooks)
        need_last = self.arch.layer_norm_first and (self.feature_selection == "fairseq_layers" or bool(self.hooks))
        ffn = torch.empty((NL, B, T, D), dtype=torch.float32, device=device) if need_ffn else None
        last = torch.empty((B, T, D), dtype=torch.float32, device=device) if need_last else None
        out = self._forward_ex(native, wavs, lens, max_len, T, ffn, last)
        if self.arch.family == "distiller":
            return self._distiller_result(out, lens, max_len, T)
        hidden_states = tuple(out[i] for i in range(NL + 1))
        # layer outputs as the reference's layer_results[i][0]: identical to hidden state i+1 except that a pre-LN
        # model's last entry is the stream BEFORE encoder.layer_norm (wav2vec2_model.py:3049-3050, 3095-3099)
        layer_out = [out[i + 1] for i in range(NL)]
        if last is not None:
            layer_out[-1] = last
        if self.feature_selection == "fairseq_layers":  # wav2vec2/expert.py:81-86
            return {"hidden_states": layer_out}
        if self.feature_selection == "fairseq_layers_before_residual":  # wav2vec2/expert.py:87-93
            return {"hidden_states": [ffn[i] for i in range(NL)]}
        if self.hooks:
            return self._run_hooks(out, layer_out, ffn)
        result: Dict[str, Union[torch.Tensor, tuple]] = {
            "_hidden_states_info": tuple([f"self.model.encoder.layers[{i}]" for i in range(NL)] + ["self.model.encoder"]),
            "hidden_states": hidden_states,
            "last_hidden_state": hidden_states[-1],
        }
        for i, h in enumerate(hidden_states):
            result[f"hidden_state_{i}"] = h
        return result

    def _distiller_result(self, out: torch.Tensor, lens: List[int], max_len: int, T: int) -> Dict:
        """The Distiller expert's result dict (s3prl/upstream/distiller/expert.py:44-63): hidden_states =
        [feat_final] + layer outputs + prediction heads, "paper" = the last layer output, "pad_mask" = frame validity."""
        device = out.device
        hidden = [out[i] for i in range(self.num_outputs)]
        valid = torch.tensor(self.valid_frames(lens, max_len), device=device)
        pad_mask = (torch.arange(T, device=device).unsqueeze(0) < valid.unsqueeze(1)).to(torch.float32)  # 1 = valid frame
        result = {"last_hidden_state": hidden[-1], "hidden_states": hidden, "pad_mask": pad_mask,
                  "paper": hidden[self.arch.encoder_layers]}
        for i, h in enumerate(hidden):
            result[f"hidden_state_{i}"] = h
        return result

    def _run_hooks(self, out: torch.Tensor, layer_out: List[torch.Tensor], ffn: torch.Tensor) -> Dict:
        """Custom ``hooks=`` (interfaces.py:74-131): every transform sees the (input, output) pair the reference's
        forward hook on that module would see — time-major [T, B, D] tensors for the encoder layers
        (wav2vec2_model.py:3260-3322 returns ``x, (attn, layer_result)``), batch-major for the encoder itself."""
        NL = self.arch.encoder_layers
        hiddens = []
        for path, transform in self.hooks:
            m_ = _LAYER_PATH.match(path)
            if m_:
                i = int(m_.group(1))
                inp = (out[i].transpose(0, 1),)
                outp = (layer_out[i].transpose(0, 1), (None, ffn[i].transpose(0, 1)))
            else:  # TransformerEncoder.forward -> (x, layer_results) (wav2vec2_model.py:3046-3052)
                inp = (None,)
                results = [(layer_out[i].transpose(0, 1), None, ffn[i].transpose(0, 1)) for i in range(NL)]
                outp = (out[NL], results)
            hiddens.append((path, transform(inp, outp)))
        if callable(self.hook_postprocess):
            hiddens = self.hook_postprocess(hiddens)
        names, hs = zip(*hiddens)
        result = {"_hidden_states_info": names, "hidden_states": hs, "last_hidden_state": hs[-1]}
        for i, h in enumerate(hs):
            result[f"hidden_state_{i}"] = h
        return result


def _family_of(name: str) -> str:
    if name in ARCHS or name in ALIASES:
        return get_arch(name).family
    if name.startswith("unispeech_sat"):  # the WavLM model class (s3prl/upstream/unispeech_sat/expert.py:20)
        return "wavlm"
    if name.startswith("distil"):
        return "distiller"
    for fam in ("hubert", "wav2vec2", "wavlm", "data2vec"):
        if name.startswith(fam):
            return fam
    raise KeyError(f"cannot infer the model family from '{name}'")
