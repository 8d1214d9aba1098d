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

from typing import Callable, Dict, List

from .upstream.configs import ALIASES, ARCHS
from .upstream.expert import UpstreamExpert


def _make_entry(name: str) -> Callable:
    def entry(ckpt=None, model_config=None, refresh=False, *args, **kwargs):
        if isinstance(ckpt, str) and ckpt.startswith("http"):
            raise ValueError(f"{name}: remote checkpoints are not reachable here; pass a local converted ckpt")
        return UpstreamExpert(ckpt=ckpt, name=name, model_config=model_config, **kwargs)

    entry.__name__ = name
    entry.__doc__ = f"H100-native {name} upstream (s3prl_b200)."
    return entry


def _make_local_entry(family: str, suffix: str = "local") -> Callable:
    """``*_local`` / ``*_custom`` / ``*_url`` (hubert/hubconf.py:57-78 and its siblings): in the reference the latter two
    download ``ckpt`` when it is a URL and then behave like ``*_local``; there is no network here, so a URL is refused
    with a message and a path is read as the converted checkpoint it must be."""

    def entry(ckpt, *args, **kwargs):
        assert isinstance(ckpt, str), "a converted checkpoint path is required"
        if ckpt.startswith("http"):
            raise ValueError(f"{family}_{suffix}: remote checkpoints are not reachable here; download {ckpt} and pass the file")
        kwargs.pop("refresh", None)
        if kwargs.pop("legacy", False):  # hubert_custom(legacy=True): un-converted fairseq file, needs fairseq itself
            raise ValueError(f"{family}_{suffix}: legacy fairseq checkpoints are not supported; convert first "
                             "(s3prl_b200.upstream.convert.convert_fairseq_checkpoint)")
        return UpstreamExpert(ckpt=ckpt, name=f"{family}_local", **kwargs)

    entry.__name__ = f"{family}_{suffix}"
    return entry


ENTRIES: Dict[str, Callable] = {}
for _name in list(ARCHS) + list(ALIASES):
    ENTRIES[_name] = _make_entry(_name)
for _family in ("hubert", "wav2vec2", "wavlm", "unispeech_sat", "distiller", "data2vec"):
    ENTRIES[f"{_family}_local"] = _make_local_entry(_family)
    ENTRIES[f"{_family}_url"] = _make_local_entry(_family, "url")
for _family in ("hubert", "wav2vec2", "data2vec"):  # the families whose hubconf defines *_custom
    ENTRIES[f"{_family}_custom"] = _make_local_entry(_family, "custom")
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


def decoar2(ckpt=None, model_config=None, refresh=False, *args, **kwargs):
    """DeCoAR 2.0 (s3prl/upstream/decoar2/hubconf.py:34-42): the fabricated checkpoint without ``ckpt``, else the
    local ``{"model": state_dict}`` file."""
    from .upstream.decoar2 import Decoar2Expert

    if isinstance(ckpt, str) and ckpt.startswith("http"):
        raise ValueError("decoar2: remote checkpoints are not reachable here; pass a local checkpoint file")
    return Decoar2Expert(ckpt=ckpt, **kwargs)


def _make_decoar2_file_entry(suffix: str) -> Callable:
    """decoar2_local / decoar2_url / decoar2_custom (decoar2/hubconf.py:10-31): a local checkpoint file; a URL is refused."""

    def entry(ckpt, *args, **kwargs):
        from .upstream.decoar2 import Decoar2Expert

        assert isinstance(ckpt, str), "a checkpoint path is required"
        if ckpt.startswith("http"):
            raise ValueError(f"decoar2_{suffix}: remote checkpoints are not reachable here; download {ckpt} and pass the file")
        kwargs.pop("refresh", None)
        return Decoar2Expert(ckpt=ckpt, **kwargs)

    entry.__name__ = f"decoar2_{suffix}"
    return entry


ENTRIES["decoar2"] = decoar2
for _suffix in ("local", "url", "custom"):
    ENTRIES[f"decoar2_{_suffix}"] = _make_decoar2_file_entry(_suffix)


def _make_apc_entry(name: str, vq: bool, needs_ckpt: bool) -> Callable:
    """APC / VQ-APC (apc/hubconf.py, vq_apc/hubconf.py): the fabricated checkpoint without ``ckpt``, else the local
    ``{"config", "model"}`` file; a URL is refused (remote checkpoints cannot be reached offline)."""

    def entry(ckpt=None, *args, **kwargs):
        from .upstream.apc import ApcExpert

        if needs_ckpt:
            assert isinstance(ckpt, str), "a checkpoint path is required"
        if isinstance(ckpt, str) and ckpt.startswith("http"):
            raise ValueError(f"{name}: remote checkpoints are not reachable here; download {ckpt} and pass the file")
        kwargs.pop("refresh", None)
        kwargs.pop("model_config", None)
        return ApcExpert(ckpt=ckpt, name=name, vq=vq, **kwargs)

    entry.__name__ = name
    return entry


for _name in ("apc", "apc_360hr", "apc_960hr"):
    ENTRIES[_name] = _make_apc_entry(_name, False, False)
for _name in ("vq_apc", "vq_apc_360hr", "vq_apc_960hr"):
    ENTRIES[_name] = _make_apc_entry(_name, True, False)
ENTRIES["apc_local"] = _make_apc_entry("apc_local", False, True)
ENTRIES["apc_url"] = _make_apc_entry("apc_url", False, True)
ENTRIES["vq_apc_url"] = _make_apc_entry("vq_apc_url", True, True)


def _make_decoar_entry(name: str, all_layers: bool, needs_ckpt: bool) -> Callable:
    """DeCoAR (decoar/hubconf.py, decoar_layers/hubconf.py): the fabricated checkpoint without ``ckpt``, else the
    local ``{"model"}`` file; a URL is refused (remote checkpoints cannot be reached offline)."""

    def entry(ckpt=None, *args, **kwargs):
        from .upstream.decoar import DecoarExpert

        if needs_ckpt:
            assert isinstance(ckpt, str), "a checkpoint path is required"
        if isinstance(ckpt, str) and ckpt.startswith("http"):
            raise ValueError(f"{name}: remote checkpoints are not reachable here; download {ckpt} and pass the file")
        kwargs.pop("refresh", None)
        return DecoarExpert(ckpt=ckpt, all_layers=all_layers, name=name, **kwargs)

    entry.__name__ = name
    return entry


for _family, _all in (("decoar", False), ("decoar_layers", True)):
    ENTRIES[_family] = _make_decoar_entry(_family, _all, False)
    for _suffix in ("local", "url", "custom"):
        ENTRIES[f"{_family}_{_suffix}"] = _make_decoar_entry(f"{_family}_{_suffix}", _all, True)


def options() -> List[str]:
    """Names of the available entries (cf. s3prl.hub.options, s3prl/hub.py:40-54)."""
    return sorted(ENTRIES)


def install(hub_module) -> List[str]:
    """setattr every entry on the given module (``s3prl.hub``); returns the injected names."""
    for name, fn in ENTRIES.items():
        setattr(hub_module, name, fn)
    return sorted(ENTRIES)
