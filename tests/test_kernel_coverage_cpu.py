"""Every configuration of the non-GEMM kernels a served model runs has a block test, as test_port_coverage_cpu.py
requires of the GEMM shapes: whole-forward parity, 2e-4 relative per hidden state, can hide a misplaced column or a
dropped tap at a configuration no block test runs. Per kernel family:

- positional conv (D, groups, k, taps per k-block 1 | 4, mode 0 | 1 | 2, post-LN): test_gemm_layouts_gpu.POS_CONFIGS
  (test_posconv without the LayerNorm, test_posconv_post_ln with it for modes 0 and 2), the 80- / 120-channel groups
  of test_xls_r_gpu.WIDE_GROUP_DIMS and the 24- / 40-channel ones of test_lighthubert_gpu.NARROW_POS_DIMS (both with
  and without the LayerNorm);
- attention (H, head dim, bias "none" | "wavlm"): test_blocks_gpu.ATTENTION_CASES and BIAS_HEADS, test_xls_r_gpu.HEADS
  and SSAST's window attention (test_ssast_blocks_gpu.TOKENS);
- LayerNorm (D, eps, GELU): test_blocks_gpu.LAYERNORM_DIMS, test_xls_r_gpu / test_port_shapes_gpu.LAYERNORM_WIDE_D,
  test_lighthubert_gpu.NARROW_LN_DIMS (all eps 1e-5, with and without GELU) and SSAST's eps 1e-6
  (test_ssast_blocks_gpu.LN_GEOMETRIES);
- LayerNorm + RoPE (D): test_conformer_gpu.ROPE_CASES, test_port_shapes_gpu.ROPE_WIDTHS;
- the Conformer's depthwise conv (D, k): test_conformer_gpu.test_depthwise_block and
  test_kernel_coverage_gpu.DEPTHWISE_SERVED;
- the conv front end (extractor_mode, conv_bias): test_frontend_gpu.test_groupnorm / test_layernorm at CONV0_BIAS;
- the fbank front end (window, mel bins, step, CMVN, operand format) of APC, VQ-APC, DeCoAR, DeCoAR 2.0 and NPC:
  test_fbank_frontend_gpu.CONFIGS, formed from the hub entries whose expert is one of those kinds;
- the 128-bin fbank front end (window, mel bins, normalisation, operand layout, operand format) of SSAST and MAE-AST:
  test_fbank128_frontend_gpu.CONFIGS, formed from the hub entries whose expert module is ssast or mae_ast.

The configurations are formed from the served geometries (test_port_coverage_cpu._geometries: configs.ARCHS,
configs.XLS_R, decoar2.DECOAR2, the LightHuBERT subnets; plus SSAST), with the model.cu rules that pick a
formulation restated below, so a new geometry fails here, without a GPU, until its configurations have a block test."""
import inspect
import sys

from s3prl_b200 import hub
from s3prl_b200.upstream import apc, decoar, decoar2, lighthubert, mae_ast, npc, ssast
from test_blocks_gpu import ATTENTION_CASES, BIAS_HEADS, LAYERNORM_DIMS
from test_conformer_gpu import DEPTHWISE_D, DEPTHWISE_KS, ROPE_CASES
from test_fbank128_frontend_gpu import CONFIGS as FBANK128_CONFIGS
from test_fbank128_frontend_gpu import MAE_AST_NORM, SSAST_NORM
from test_fbank_frontend_gpu import CMVN_ALL_FRAMES
from test_fbank_frontend_gpu import CONFIGS as FBANK_CONFIGS
from test_frontend_gpu import CONV0_BIAS
from test_gemm_layouts_gpu import POS_CONFIGS
from test_kernel_coverage_gpu import DEPTHWISE_SERVED
from test_lighthubert_gpu import NARROW_LN_DIMS, NARROW_POS_DIMS
from test_port_coverage_cpu import CONV_DIM, _geometries
from test_port_shapes_gpu import LAYERNORM_WIDE_D as LN_1280
from test_port_shapes_gpu import ROPE_WIDTHS
from test_ssast_blocks_gpu import HD as SSAST_HD
from test_ssast_blocks_gpu import LN_EPS as SSAST_LN_EPS
from test_ssast_blocks_gpu import LN_GEOMETRIES, TOKENS
from test_xls_r_gpu import HEADS, WIDE_GROUP_DIMS
from test_xls_r_gpu import LAYERNORM_WIDE_D as LN_1920

LN_EPS = 1e-5  # s3b_model's ln_eps and launch_layernorm's default
# the model kinds add_fbank_frontend serves (model.cu kGruStack, kLstmStack, kFbankEncoder, kNpcStack), by the module
# of their expert
FBANK_MODULES = (apc, decoar, decoar2, npc)
HOP = 160  # kaldi fbank's frame shift in samples


# ------------------------------------------------------------------------------------------------
# model.cu's rules, restated
# ------------------------------------------------------------------------------------------------
def _posconv4_only(cpg):
    """model.cu posconv4_only: 24 and 40 channels per group run four taps per k-block only."""
    return cpg in (24, 40)


def _posconv_cpg_ok(cpg):
    """model.cu posconv_cpg_ok."""
    return (cpg % 16 == 0 and 16 <= cpg <= 64) or cpg in (80, 120) or _posconv4_only(cpg)


def _pos_taps(arch):
    """model.cu pos_taps: conv_pos, or max(3, conv_pos / depth) per data2vec block."""
    return max(3, arch.conv_pos // arch.pos_conv_depth) if arch.pos_conv_depth > 1 else arch.conv_pos


def _posconv4_ok(arch):
    """model.cu posconv4_ok: the four-taps formulation."""
    cpg = arch.encoder_embed_dim // arch.conv_pos_groups
    if arch.pos_conv_depth > 1:
        return True
    return arch.conv_pos % 4 == 0 and (_posconv4_only(cpg) or cpg in (48, 64))


# ------------------------------------------------------------------------------------------------
# served configurations
# ------------------------------------------------------------------------------------------------
def _served_posconv():
    """(D, groups, k, taps, mode, post-LN) -> models. add_pos_conv: data2vec runs pos_conv_depth blocks of mode 1 and
    a last one of mode 2, which alone carries the post-LN encoder LayerNorm; the others one conv of mode 0."""
    served = {}
    for name, a in _geometries().items():
        if a.conformer:  # no pos_conv
            continue
        D, G = a.encoder_embed_dim, a.conv_pos_groups
        assert _posconv_cpg_ok(D // G), (name, D // G)
        post_ln = not a.layer_norm_first
        taps = 4 if _posconv4_ok(a) else 1
        k = _pos_taps(a)
        if a.pos_conv_depth > 1:
            keys = [(D, G, k, taps, 1, False), (D, G, k, taps, 2, post_ln)]
        else:
            keys = [(D, G, k, taps, 0, post_ln)]
        for key in keys:
            served.setdefault(key, []).append(name)
    return served


def _covered_posconv():
    cov = set()
    for D, G, k, taps, mode in POS_CONFIGS:
        cov.add((D, G, k, taps, mode, False))  # test_posconv
        if mode != 1:
            cov.add((D, G, k, taps, mode, True))  # test_posconv_post_ln
    for D in WIDE_GROUP_DIMS:  # test_posconv_wide_groups: k = 128, one tap, with and without the LayerNorm
        cov |= {(D, 16, 128, 1, 0, False), (D, 16, 128, 1, 0, True)}
    for D in NARROW_POS_DIMS:  # test_posconv_four_taps_narrow_groups
        cov |= {(D, 16, 128, 4, 0, False), (D, 16, 128, 4, 0, True)}
    return cov


def _served_attention():
    """(H, head dim, bias) -> models; WavLM's gated relative-position bias where relative_position_embedding."""
    served = {}
    for name, a in _geometries().items():
        H = a.encoder_attention_heads
        key = (H, a.encoder_embed_dim // H, "wavlm" if a.relative_position_embedding else "none")
        served.setdefault(key, []).append(name)
    for kind in ssast.KINDS:
        key = (ssast.HEADS, ssast.EMBED // ssast.HEADS, "none")
        served.setdefault(key, []).append(f"ssast_{kind} window attention")
    return served


def _covered_attention():
    cov = {(H, 64, "none") for _, _, H, _ in ATTENTION_CASES}
    cov |= {(H, 64, "wavlm") for H in BIAS_HEADS}
    cov |= {(H, hd, "none") for H, hd in HEADS}
    if TOKENS:
        cov.add((ssast.HEADS, SSAST_HD, "none"))
    return cov


def _served_layernorm():
    """(D, eps, gelu) -> where the forward calls launch_layernorm."""
    served = {}
    for name, a in _geometries().items():
        served.setdefault((a.encoder_embed_dim, LN_EPS, 0), []).append(f"{name} encoder")
        if a.frontend == "conv":
            if a.extractor_mode == "layer_norm":  # add_conv_frontend: conv 1..6 per-frame LayerNorm + GELU
                served.setdefault((CONV_DIM, LN_EPS, 1), []).append(f"{name} conv stack")
            if a.feature_layer_norm:  # add_post_extract_proj: LayerNorm(512)
                served.setdefault((CONV_DIM, LN_EPS, 0), []).append(f"{name} post_extract_proj")
    for kind in ssast.KINDS:
        served.setdefault((ssast.EMBED, 1e-6, 0), []).append(f"ssast_{kind} encoder")
    return served


def _covered_layernorm():
    cov = {(D, LN_EPS, gelu) for D in list(LAYERNORM_DIMS) + list(NARROW_LN_DIMS) + [LN_1280, LN_1920]
           for gelu in (0, 1)}
    if LN_GEOMETRIES:
        cov.add((ssast.EMBED, SSAST_LN_EPS, 0))
    return cov


def _served_rope():
    served = {}
    for name, a in _geometries().items():
        if a.conformer:
            served.setdefault(a.encoder_embed_dim, []).append(name)
    return served


def _served_depthwise():
    served = {}
    for name, a in _geometries().items():
        if a.conformer:
            served.setdefault((a.encoder_embed_dim, a.depthwise_conv_kernel_size), []).append(name)
    return served


def _served_frontend():
    served = {}
    for name, a in _geometries().items():
        if a.frontend == "conv":
            served.setdefault((a.extractor_mode, a.conv_bias), []).append(name)
    return served


def _hub_expert(entry):
    """The expert class a hub entry makes (hub._entry's `make`, unwrapped from its partial); None for the others."""
    make = inspect.getclosurevars(entry).nonlocals.get("make")
    return getattr(make, "func", make)


def _fbank_step(mod):
    """model.cu add_fbank_frontend: every second frame for kFbankEncoder (DeCoAR 2.0), else every frame; the
    module's downsample rate over the hop."""
    return mod.DOWNSAMPLE_RATE // HOP


def _served_fbank_frontend():
    """(window, mel bins, step, CMVN, operand format) -> hub entries. add_fbank_frontend runs launch_decoar2_features
    for every fbank kind: fbank_frames_kernel<true> (the hamming window), the expert module's mel bins, CMVN over all
    frames, written in the model's operand scheme, which S3B_GEMM_SCHEME selects at run time: both formats."""
    served = {}
    for name, entry in hub.ENTRIES.items():
        mod = sys.modules.get(getattr(_hub_expert(entry), "__module__", ""))
        if mod not in FBANK_MODULES:
            continue
        for fmt in (0, 1):
            key = ("hamming", mod.NUM_MEL_BINS, _fbank_step(mod), CMVN_ALL_FRAMES, fmt)
            served.setdefault(key, []).append(name)
    return served


# the 128-bin front ends (fbank.cu ssast_fbank_kernel + ssast_patches_kernel, mae_ast_fbank_kernel) by the module of
# their expert: (window, normalisation)
FBANK128_MODULES = {ssast: ("hanning", SSAST_NORM), mae_ast: ("povey", MAE_AST_NORM)}


def _served_fbank128_frontend():
    """(window, mel bins, normalisation, operand layout, operand format) -> hub entries whose expert module is ssast or
    mae_ast: the layout is the module's KINDS entry of every kind the entry can serve (mae_ast_local / _url take the
    file's own), both operand formats (S3B_GEMM_SCHEME selects one at run time)."""
    served = {}
    for name, entry in hub.ENTRIES.items():
        mod = sys.modules.get(getattr(_hub_expert(entry), "__module__", ""))
        if mod not in FBANK128_MODULES:
            continue
        window, norm = FBANK128_MODULES[mod]
        for layout in mod.KINDS.values():
            for fmt in (0, 1):
                served.setdefault((window, mod.NUM_BINS, norm, layout, fmt), []).append(name)
    return served


FAMILIES = {  # name -> (served, covered)
    "positional conv (D, groups, k, taps per k-block, mode, post-LN)": (_served_posconv, _covered_posconv),
    "attention (H, head dim, bias)": (_served_attention, _covered_attention),
    "LayerNorm (D, eps, gelu)": (_served_layernorm, _covered_layernorm),
    "LayerNorm + RoPE (D)": (_served_rope, lambda: {D for _, _, D in ROPE_CASES} | set(ROPE_WIDTHS)),
    "depthwise conv (D, k)": (_served_depthwise,
                              lambda: {(DEPTHWISE_D, k) for k in DEPTHWISE_KS} | set(DEPTHWISE_SERVED)),
    "conv front end (extractor_mode, conv_bias)": (
        _served_frontend, lambda: {(m, b) for m in ("default", "layer_norm") for b in CONV0_BIAS}),
    "fbank front end (window, mel bins, step, CMVN, operand format)": (_served_fbank_frontend, lambda: set(FBANK_CONFIGS)),
    "128-bin fbank front end (window, mel bins, normalisation, operand layout, operand format)": (
        _served_fbank128_frontend, lambda: set(FBANK128_CONFIGS)),
}


def _assert_covered(family):
    served, covered = FAMILIES[family]
    cov = covered()
    missing = {key: models for key, models in served().items() if key not in cov}
    assert not missing, f"{family} without a block test: " + "; ".join(
        f"{key} run by {', '.join(models[:3])}" + (f" and {len(models) - 3} more" if len(models) > 3 else "")
        for key, models in sorted(missing.items(), key=lambda kv: str(kv[0])))


# ------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------
def test_served_set_is_formed():
    """Every family enumerates something, and the set holds the configurations that were once only seen by whole-model
    goldens: LightHuBERT student small's 32-channel one-tap tiles and data2vec large's k = 19 blocks."""
    for family, (served, _) in FAMILIES.items():
        assert served(), family
    pos = _served_posconv()
    student_small = f"lighthubert.SUBNETS[{('student_hubert', 'small')}]"
    assert student_small in pos[(512, 16, 128, 1, 0, True)]
    assert "configs.ARCHS['data2vec_large_ll60k']" in pos[(1024, 16, 19, 4, 1, False)]
    assert "configs.ARCHS['data2vec_large_ll60k']" in pos[(1024, 16, 19, 4, 2, True)]
    assert "configs.XLS_R['xls_r_2b']" in _served_attention()[(16, 120, "none")]
    assert (1024, 31) in _served_depthwise()
    assert (ssast.EMBED, 1e-6, 0) in _served_layernorm()
    assert len(lighthubert.SUBNETS) == sum(1 for n in _geometries() if n.startswith("lighthubert."))
    fb = _served_fbank_frontend()
    names = {n for models in fb.values() for n in models}
    assert {"apc", "vq_apc", "decoar", "decoar_layers", "decoar2", "npc", "npc_360hr", "npc_960hr"} <= names
    assert "decoar2" in fb[("hamming", 80, 2, CMVN_ALL_FRAMES, 1)] and "npc" in fb[("hamming", 80, 1, CMVN_ALL_FRAMES, 0)]
    fb128 = _served_fbank128_frontend()
    names = {n for models in fb128.values() for n in models}
    assert {"ssast_frame_base", "ssast_patch_base", "mae_ast_frame", "mae_ast_patch", "mae_ast_local",
            "mae_ast_url"} <= names
    assert "mae_ast_patch" in fb128[("povey", 128, MAE_AST_NORM, (16, 16), 1)]
    assert "ssast_frame_base" in fb128[("hanning", 128, SSAST_NORM, ((128, 2), (128, 1)), 0)]


def test_posconv_rules_match_the_model():
    """The restated rules on the configurations model.cu documents: 48 / 64 channels and k % 4 == 0 take four taps,
    32 / 80 / 120 one, data2vec's blocks four at k = max(3, conv_pos // depth)."""
    from dataclasses import replace

    from s3prl_b200.upstream.configs import ARCHS, XLS_R

    assert _posconv4_ok(ARCHS["hubert_base"]) and _posconv4_ok(ARCHS["hubert_large_ll60k"])
    assert not _posconv4_ok(XLS_R["xls_r_1b"]) and not _posconv4_ok(XLS_R["xls_r_2b"])
    assert not _posconv4_ok(replace(ARCHS["hubert_base"], encoder_embed_dim=512))
    assert _posconv4_ok(replace(ARCHS["hubert_base"], encoder_embed_dim=384))
    assert _pos_taps(ARCHS["data2vec_large_ll60k"]) == 19 == ARCHS["data2vec_large_ll60k"].pos_conv_kernel
    assert not _posconv_cpg_ok(128) and not _posconv_cpg_ok(8) and _posconv_cpg_ok(32)


def test_every_served_posconv_has_a_block_test():
    _assert_covered("positional conv (D, groups, k, taps per k-block, mode, post-LN)")


def test_every_served_attention_has_a_block_test():
    _assert_covered("attention (H, head dim, bias)")


def test_fbank_step_rule_matches_the_models():
    """The step restated from each kind's downsample rate is the decimation its expert's frame count implies:
    num_frames(n) = ceil(m / step) with m = 1 + (n - 400) // 160 kaldi frames, at lengths on frame edges."""
    for mod in FBANK_MODULES:
        step = _fbank_step(mod)
        for n in (560, 561, 719, 720, 879, 880, 16000, 16001, 328000):
            assert mod.num_frames(n) == -(-(1 + (n - 400) // HOP) // step), (mod.__name__, n)
    assert [_fbank_step(mod) for mod in FBANK_MODULES] == [1, 1, 2, 1]


def test_every_served_fbank_frontend_has_a_block_test():
    _assert_covered("fbank front end (window, mel bins, step, CMVN, operand format)")


def test_every_served_fbank128_frontend_has_a_block_test():
    _assert_covered("128-bin fbank front end (window, mel bins, normalisation, operand layout, operand format)")


def test_every_served_layernorm_has_a_block_test():
    _assert_covered("LayerNorm (D, eps, gelu)")


def test_every_served_layernorm_rope_has_a_block_test():
    _assert_covered("LayerNorm + RoPE (D)")


def test_every_served_depthwise_has_a_block_test():
    _assert_covered("depthwise conv (D, k)")


def test_every_served_frontend_has_a_block_test():
    _assert_covered("conv front end (extractor_mode, conv_bias)")
