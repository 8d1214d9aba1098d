"""``fbank`` baseline upstream on the GPU (s3prl/upstream/baseline/expert.py:23-79 with fbank.yaml).

    expert = FbankExpert()
    out = expert([wav_0, wav_1, ...])      # list of 1-D fp32 CUDA tensors
    out["hidden_states"] == [X],  X: [B, max_frames, 240]  (80 log-mel + delta + delta-delta, CMVN)
    FbankExpert(cmvn=False) is the ``fbank_no_cmvn`` entry (fbank_no_cmvn.yaml): the same features without CMVN.
    expert.get_downsample_rates("hidden_states") == 160
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List

import torch
import torch.nn as nn

from .. import lib as _lib


class FbankExpert(nn.Module):
    output_dim = 240
    downsample_rate = 160

    def __init__(self, model_config=None, cmvn: bool = True, **kwargs):
        super().__init__()
        self.cmvn = bool(cmvn)
        self.register_buffer("_device_anchor", torch.zeros(1), persistent=False)

    def get_downsample_rates(self, key: str) -> int:
        return self.downsample_rate

    def forward(self, wavs: List[torch.Tensor]) -> Dict[str, object]:
        lib = _lib.load()
        _lib.require_gpu()
        device = wavs[0].device
        if device.type != "cuda":
            raise _lib.S3BError("s3prl_b200 fbank runs on CUDA devices only (no CPU fallback)")
        wavs = [w.detach().to(torch.float32).contiguous() for w in wavs]
        lens = [int(w.numel()) for w in wavs]
        B = len(wavs)
        m = lib.s3b_fbank_num_frames(max(lens))
        if m < 1:
            raise ValueError("waveforms shorter than one 25 ms frame")
        with torch.cuda.device(device):
            out = torch.empty((B, m, self.output_dim), dtype=torch.float32, device=device)
            ptrs = (C.c_void_p * B)(*[w.data_ptr() for w in wavs])
            lens_c = (C.c_int64 * B)(*lens)
            opts = _lib.S3BSpectralOpts(cmvn=int(self.cmvn))
            _lib.check(
                lib.s3b_fbank_ex(ptrs, lens_c, B, C.byref(opts), C.c_void_p(out.data_ptr()),
                                 C.c_void_p(torch.cuda.current_stream(device).cuda_stream))
            )
        return {"last_hidden_state": out, "hidden_states": [out]}


class SpectrogramExpert(nn.Module):
    """``mel`` / ``linear`` baselines (s3prl/upstream/baseline/expert.py:52-79 with mel.yaml / linear.yaml).

    The length bookkeeping is the reference's, quirks included: the lengths after dropping trailing exact zeros
    (preprocessor.py:166-175) set how many frames CMVN runs over, ``round(len / (Lmax / n_frames))`` (:203-204), but
    the STFT still sees the batch padded to the longest ORIGINAL length (the trim there slices the channel axis, so
    Lmax and n_frames come from the untrimmed padding), and the final cut uses the ratio of the FIRST utterance
    (expert.py:62-64)."""

    downsample_rate = 160

    def __init__(self, feat_type: str = "mel", **kwargs):
        super().__init__()
        assert feat_type in ("mel", "linear")
        self.feat_type = feat_type
        self.output_dim = 80 if feat_type == "mel" else 201
        self.register_buffer("_device_anchor", torch.zeros(1), persistent=False)

    def get_downsample_rates(self, key: str) -> int:
        return self.downsample_rate

    @staticmethod
    def plan_lengths(orig_lens: List[int], trimmed_lens: List[int]):
        """(padded_len, feats_len, final_len, t_out) exactly as the reference's Python arithmetic yields them."""
        lp = max(orig_lens)
        n_frames = 1 + lp // 160
        downsample_rate = lp / n_frames
        feats_len = [round(n / downsample_rate) for n in trimmed_lens]
        tm = max(feats_len)
        ratio = tm / orig_lens[0]
        final_len = [min(round(n * ratio), tm) for n in orig_lens]
        return lp, feats_len, final_len, max(final_len)

    def forward(self, wavs: List[torch.Tensor]) -> Dict[str, object]:
        lib = _lib.load()
        _lib.require_gpu()
        device = wavs[0].device
        if device.type != "cuda":
            raise _lib.S3BError("s3prl_b200 mel/linear run on CUDA devices only (no CPU fallback)")
        wavs = [w.detach().to(torch.float32).contiguous() for w in wavs]
        lens = [int(w.numel()) for w in wavs]
        B = len(wavs)
        ptrs = (C.c_void_p * B)(*[w.data_ptr() for w in wavs])
        with torch.cuda.device(device):
            torch.cuda.current_stream(device).synchronize()  # the trim scan runs on the default stream
            trimmed = (C.c_int64 * B)()
            _lib.check(lib.s3b_trimmed_lengths(ptrs, (C.c_int64 * B)(*lens), B, trimmed))
            lp, feats_len, final_len, t_out = self.plan_lengths(lens, list(trimmed))
            out = torch.empty((B, t_out, self.output_dim), dtype=torch.float32, device=device)
            _lib.check(
                lib.s3b_melspec(ptrs, trimmed, B, lp, int(self.feat_type == "mel"), (C.c_int32 * B)(*feats_len),
                                (C.c_int32 * B)(*final_len), t_out, C.c_void_p(out.data_ptr()),
                                C.c_void_p(torch.cuda.current_stream(device).cuda_stream))
            )
        return {"last_hidden_state": out, "hidden_states": [out]}
