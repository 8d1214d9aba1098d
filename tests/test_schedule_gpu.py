"""The kernels a forward enqueues, counted per model kind.

A forward is a fixed sequence of launches for its model and batch; the profile counts them per category and
``s3b_launch_count`` in total. This pins both at one ragged batch for every model kind, with the expected counts
written as formulas of the model's config: a change to what a forward enqueues (a launch added, dropped, merged, or
accounted to another category) shows here, where the numerical tests would only see it through its result. With two
lanes each lane enqueues its own copy of the sequence; a DeCoAR model runs one lane whatever is asked.
"""
import ctypes as C
from dataclasses import replace

import pytest
import torch

pytestmark = pytest.mark.gpu

GEMM, ATTN, CONV0, NORM, MISC, GRU = range(6)  # the profile's categories (s3b_profile_read_ex)
LENS = (32000, 24011, 17003)  # a ragged batch, up to 2 s


def _encoder(name, **changes):
    from s3prl_b200.upstream.configs import ARCHS, XLS_R
    from s3prl_b200.upstream.expert import UpstreamExpert

    if name == "xls_r_1b":
        return UpstreamExpert(name="wav2vec2_local", arch=replace(XLS_R[name], **changes))
    return UpstreamExpert(name=name, arch=replace(ARCHS[name], **changes))


def _build(kind):
    from s3prl_b200.upstream.apc import ApcExpert
    from s3prl_b200.upstream.decoar import DecoarExpert
    from s3prl_b200.upstream.decoar2 import Decoar2Expert

    return {
        "hubert_base": lambda: _encoder("hubert_base", encoder_layers=2),
        "wav2vec2_large_ll60k": lambda: _encoder("wav2vec2_large_ll60k", encoder_layers=2),
        "wavlm_base_plus": lambda: _encoder("wavlm_base_plus", encoder_layers=2),
        "data2vec_base_960": lambda: _encoder("data2vec_base_960", encoder_layers=2),
        "distilhubert_base": lambda: _encoder("distilhubert_base"),
        "conformer_pre_ln": lambda: _encoder("wav2vec2_conformer_rope", encoder_layers=2),
        "conformer_post_ln": lambda: _encoder("wav2vec2_conformer_rope", encoder_layers=2, layer_norm_first=False,
                                              extractor_mode="default", conv_bias=False, normalize=False),
        "xls_r_hd80": lambda: _encoder("xls_r_1b", encoder_layers=2),
        "decoar2": lambda: Decoar2Expert(),
        "apc": lambda: ApcExpert(),
        "decoar": lambda: DecoarExpert(all_layers=False),
        "decoar_layers": lambda: DecoarExpert(all_layers=True),
    }[kind]()


def _encoder_counts(a):
    """Launches per category of one lane of an encoder model (ArchConfig a)."""
    n = [0] * 6
    NL, D = a.encoder_layers, a.encoder_embed_dim
    if a.frontend == "fbank":
        n[CONV0] += 2                     # fbank frames, CMVN
    else:
        n[MISC] += 1                      # waveform packing
        layer_norm = a.extractor_mode == "layer_norm"
        n[CONV0] += 1 if layer_norm else 3  # conv 0 with its LayerNorm, or with the GroupNorm's three kernels
        n[GEMM] += 6                      # conv 1..6
        if layer_norm:
            n[NORM] += 6                  # their per-frame LayerNorms
        if a.feature_layer_norm:
            n[NORM] += 1                  # LayerNorm(512)
    n[GEMM] += 1                          # post_extract_proj
    if a.conformer:
        if not a.layer_norm_first:
            n[NORM] += 1                  # encoder.layer_norm -> hidden state 0
        n[GEMM] += 9 * NL                 # ffn1 w_1, w_2; [q | k], v; linear_out; pointwise_conv1, 2; ffn2 w_1, w_2
        n[NORM] += 5 * NL                 # ffn1 LN, self_attn LN + RoPE, conv_module LN, ffn2 LN, final_layer_norm
        n[ATTN] += NL
        n[MISC] += NL                     # GLU + depthwise conv + BatchNorm + SiLU
        if a.layer_norm_first:
            n[NORM] += 1                  # encoder.layer_norm after the last layer
        return n
    cpg = D // a.conv_pos_groups
    if a.pos_conv_depth > 1:
        n[GEMM] += a.pos_conv_depth       # data2vec: one four-taps GEMM per positional conv block
        n[NORM] += a.pos_conv_depth       # and its combine kernel
    elif a.conv_pos % 4 == 0 and 4 * cpg in (192, 256):
        n[GEMM] += 1                      # pos_conv, four taps per k-block
        n[NORM] += 1                      # the combine kernel (+ encoder LayerNorm)
    else:
        n[GEMM] += 1                      # pos_conv, one tap per k-block
        if not a.layer_norm_first:
            n[NORM] += 1                  # encoder LayerNorm
    n[GEMM] += 4 * NL                     # QKV, out_proj, fc1, fc2
    n[ATTN] += NL
    n[NORM] += 2 * NL                     # pre-LN: LN1, LN2; post-LN: after attention, after fc2
    if a.layer_norm_first:
        n[NORM] += 1                      # encoder.layer_norm after the last layer
    if a.relative_position_embedding:
        n[MISC] += NL                     # WavLM gate
    if a.pred_heads:
        n[GEMM] += 1 + a.pred_heads       # Linear + GELU, then one SplitLinear GEMM per head
    return n


def _counts(kind, ex, B):
    """(launches per category of one lane, lanes a two-lane request runs)."""
    n = [0] * 6
    if kind == "apc":
        n[CONV0] = 2                      # fbank frames, CMVN
        n[GEMM] = ex.num_layers           # input GEMM per GRU layer
        n[GRU] = ex.num_layers            # recurrence per GRU layer
        return n, 2
    if kind.startswith("decoar") and kind != "decoar2":
        nl = 4                            # the LSTM stack's layers
        n[CONV0] = 2                      # fbank frames, CMVN
        n[GEMM] = 1 + 2 * nl              # post_extract_proj, then the input GEMM per layer and direction
        n[GRU] = 2 * nl * -(-B // 512)    # recurrence per layer and direction, one launch per 512 utterances
        return n, 1                       # one lane: the recurrence occupies the whole device
    return _encoder_counts(ex.arch), 2


KINDS = ["hubert_base", "wav2vec2_large_ll60k", "wavlm_base_plus", "data2vec_base_960", "distilhubert_base",
         "conformer_pre_ln", "conformer_post_ln", "xls_r_hd80", "decoar2", "apc", "decoar", "decoar_layers"]


@pytest.mark.parametrize("kind", KINDS)
def test_launches_per_forward(s3b_lib, kind):
    from s3prl_b200 import lib

    g = torch.Generator().manual_seed(3)
    wavs = [torch.randn(n, generator=g).cuda() for n in LENS]
    ex = _build(kind).to("cuda").eval()
    ex.lanes = 1
    ex(wavs)  # plans and tables built before anything is counted
    native = ex._native
    want, lanes = _counts(kind, ex, len(LENS))

    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    ex(wavs)
    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
    lib.check(native.lib.s3b_profile_read_ex(native.handle, 6, ms, fl, n, 1))
    lib.check(native.lib.s3b_profile_enable(native.handle, 0))
    assert list(n) == want, f"{kind}: launches per category {list(n)}, expected {want}"

    totals = []
    for ex.lanes in (1, 2):
        c0 = native.lib.s3b_launch_count(native.handle)
        ex(wavs)
        totals.append(native.lib.s3b_launch_count(native.handle) - c0)
    ex.lanes = 0
    torch.cuda.synchronize()
    assert totals == [sum(want), lanes * sum(want)], f"{kind}: launches with one and two lanes {totals}"
