"""Hub entries with the reference's factory contract.

The reference resolves an upstream as ``getattr(s3prl.hub, NAME)(ckpt=..., model_config=..., refresh=...)``
(s3prl/downstream/runner.py:141-153, s3prl/nn/upstream.py:113-117); the entries of ``s3prl/upstream/*/hubconf.py``
download a pretrained file first (e.g. hubert/hubconf.py:85-95). Here every entry returns the H100-native
``UpstreamExpert``; without ``ckpt`` (no network on this box) it uses the deterministic fabricated checkpoint of
that architecture, with ``ckpt`` it reads a converted reference checkpoint (``*_local`` entries,
hubert/hubconf.py:69-70, wav2vec2/hubconf.py:68-69, wavlm/hubconf.py:19-25, data2vec/hubconf.py:17-18).

``install(hub_module)`` injects the entries into ``s3prl.hub`` so that ``run_downstream.py -u hubert_base`` uses
this implementation with the reference tree untouched (see INTEGRATION.md).
"""
from __future__ import annotations

from functools import partial
from typing import Callable, Dict, List, Optional

from .upstream.apc import ApcExpert
from .upstream.configs import ALIASES, ARCHS
from .upstream.cpc import CpcExpert
from .upstream.decoar import DecoarExpert
from .upstream.decoar2 import Decoar2Expert
from .upstream.expert import UpstreamExpert
from .upstream.lighthubert import LighthubertExpert
from .upstream.npc import NpcExpert
from .upstream.ssast import SsastExpert


def _entry(name: str, make: Callable, ckpt_required: bool = False, refuse_legacy: bool = False,
           url_hint: Optional[str] = None) -> Callable:
    """The hub entry ``name``: ``entry(ckpt, **kwargs)`` returns ``make(ckpt=ckpt, **kwargs)``. A URL is refused (the
    reference downloads it; remote checkpoints are not reachable here) and the reference's download options
    ``refresh`` / ``model_config`` are dropped. ``ckpt_required``: a path must be given (``*_local``, ``*_url``,
    ``*_custom``). ``refuse_legacy``: the entry reads converted fairseq checkpoints of a conv-stack family, and
    ``legacy=True`` (``hubert_custom``'s un-converted fairseq file, which needs fairseq itself) is refused."""

    def entry(ckpt=None, *args, **kwargs):
        if ckpt_required:
            assert isinstance(ckpt, str), f"a {'converted ' if refuse_legacy else ''}checkpoint path is required"
        if isinstance(ckpt, str) and ckpt.startswith("http"):
            hint = url_hint or f"download {ckpt} and pass the file"
            raise ValueError(f"{name}: remote checkpoints are not reachable here; {hint}")
        kwargs.pop("refresh", None)
        kwargs.pop("model_config", None)
        if refuse_legacy and kwargs.pop("legacy", False):
            raise ValueError(f"{name}: legacy fairseq checkpoints are not supported; convert first "
                             "(s3prl_b200.upstream.convert.convert_fairseq_checkpoint)")
        return make(ckpt=ckpt, **kwargs)

    entry.__name__ = name
    entry.__doc__ = f"H100-native {name} upstream (s3prl_b200)."
    return entry


ENTRIES: Dict[str, Callable] = {}
for _name in list(ARCHS) + list(ALIASES):
    ENTRIES[_name] = _entry(_name, partial(UpstreamExpert, name=_name), url_hint="pass a local converted ckpt")
# *_local / *_url / *_custom (hubert/hubconf.py:57-78 and its siblings): in the reference the latter two download
# ckpt when it is a URL and then behave like *_local; here a path is read as the converted checkpoint it must be
for _family in ("hubert", "wav2vec2", "wavlm", "unispeech_sat", "distiller", "data2vec"):
    _suffixes = ("local", "url", "custom") if _family in ("hubert", "wav2vec2", "data2vec") else ("local", "url")
    for _suffix in _suffixes:
        ENTRIES[f"{_family}_{_suffix}"] = _entry(f"{_family}_{_suffix}", partial(UpstreamExpert, name=f"{_family}_local"),
                                                 ckpt_required=True, refuse_legacy=True)
# DeCoAR 2.0 (decoar2/hubconf.py:10-42): the fabricated checkpoint without ckpt, else the local {"model": ...} file
ENTRIES["decoar2"] = _entry("decoar2", Decoar2Expert, url_hint="pass a local checkpoint file")
for _suffix in ("local", "url", "custom"):
    ENTRIES[f"decoar2_{_suffix}"] = _entry(f"decoar2_{_suffix}", Decoar2Expert, ckpt_required=True)
# APC / VQ-APC (apc/hubconf.py, vq_apc/hubconf.py): the fabricated checkpoint without ckpt, else the local
# {"config", "model"} file
for _name, _vq, _required in (("apc", False, False), ("apc_360hr", False, False), ("apc_960hr", False, False),
                              ("vq_apc", True, False), ("vq_apc_360hr", True, False), ("vq_apc_960hr", True, False),
                              ("apc_local", False, True), ("apc_url", False, True), ("vq_apc_url", True, True)):
    ENTRIES[_name] = _entry(_name, partial(ApcExpert, name=_name, vq=_vq), ckpt_required=_required)
# DeCoAR (decoar/hubconf.py, decoar_layers/hubconf.py): the fabricated checkpoint without ckpt, else the local
# {"model"} file
for _family, _all in (("decoar", False), ("decoar_layers", True)):
    for _name in (_family, f"{_family}_local", f"{_family}_url", f"{_family}_custom"):
        ENTRIES[_name] = _entry(_name, partial(DecoarExpert, all_layers=_all, name=_name), ckpt_required=_name != _family)
# NPC (npc/hubconf.py): the fabricated checkpoint without ckpt, else the local {"config", "model"} file
for _name, _required in (("npc", False), ("npc_360hr", False), ("npc_960hr", False), ("npc_local", True),
                         ("npc_url", True)):
    ENTRIES[_name] = _entry(_name, partial(NpcExpert, name=_name), ckpt_required=_required)
# modified CPC (cpc/hubconf.py): the fabricated checkpoint without ckpt, else the local {"config", "weights"} file
for _name, _required in (("modified_cpc", False), ("cpc_local", True), ("cpc_url", True)):
    ENTRIES[_name] = _entry(_name, partial(CpcExpert, name=_name), ckpt_required=_required)
# LightHuBERT (lighthubert/hubconf.py): the fabricated supernet of each released subnet without ckpt, else the local
# {"cfg", "model"} file; lighthubert is lighthubert_small
for _name, _kind, _required in (("lighthubert", "small", False), ("lighthubert_small", "small", False),
                                ("lighthubert_base", "base", False), ("lighthubert_stage1", "stage1", False),
                                ("lighthubert_local", "small", True), ("lighthubert_url", "small", True)):
    ENTRIES[_name] = _entry(_name, partial(LighthubertExpert, name=_name, kind=_kind), ckpt_required=_required)
# SSAST (ssast/hubconf.py): the fabricated checkpoint of each model without ckpt, else the local DataParallel file;
# window_secs as in the reference (1 s for speech commands, 10 s for speaker identification)
for _name, _kind in (("ssast_frame_base", "frame"), ("ssast_patch_base", "patch")):
    ENTRIES[_name] = _entry(_name, partial(SsastExpert, name=_name, kind=_kind), url_hint="pass a local checkpoint file")
globals().update(ENTRIES)


def fbank(*args, **kwargs):
    """Kaldi-compatible 80-bin fbank + deltas + CMVN baseline (s3prl/upstream/baseline/hubconf.py:43-48)."""
    from .upstream.baseline import FbankExpert

    return FbankExpert(**kwargs)


def fbank_no_cmvn(*args, **kwargs):
    """The fbank baseline's log-mel + deltas without CMVN (s3prl/upstream/baseline/hubconf.py:51-58, fbank_no_cmvn.yaml)."""
    from .upstream.baseline import FbankExpert

    kwargs["cmvn"] = False
    return FbankExpert(**kwargs)


ENTRIES["fbank"] = fbank
ENTRIES["fbank_no_cmvn"] = fbank_no_cmvn


def mel(*args, **kwargs):
    """80-bin log-mel spectrogram + CMVN (s3prl/upstream/baseline/hubconf.py mel entry, mel.yaml)."""
    from .upstream.baseline import SpectrogramExpert

    return SpectrogramExpert("mel")


def linear(*args, **kwargs):
    """201-bin log power spectrogram + CMVN (s3prl/upstream/baseline/hubconf.py linear entry, linear.yaml)."""
    from .upstream.baseline import SpectrogramExpert

    return SpectrogramExpert("linear")


ENTRIES["mel"] = mel
ENTRIES["linear"] = linear


def options() -> List[str]:
    """Names of the available entries (cf. s3prl.hub.options, s3prl/hub.py:40-54)."""
    return sorted(ENTRIES)


def install(hub_module) -> List[str]:
    """setattr every entry on the given module (``s3prl.hub``); returns the injected names."""
    for name, fn in ENTRIES.items():
        setattr(hub_module, name, fn)
    return sorted(ENTRIES)
