"""Every GEMM shape (N, K) a served model runs has a block test: a row of test_port_shapes_gpu.PORT_LINEARS,
test_gemm_layouts_gpu.LINEAR_SHAPES or test_blocks_gpu.LINEAR_CASES, which check each output element against fp64 (the
first two also against the operand scheme's emulation). Whole-forward parity, 2e-4 relative per hidden state, can hide a
dropped k-step or a misplaced column at a shape no block test runs. test_gemm_cluster_gpu.LINEAR_SHAPES does not count:
it checks bit-identity across cluster sizes, not the values.

The shapes are formed from the served geometries themselves (configs.ARCHS, configs.XLS_R, decoar2.DECOAR2,
lighthubert.SUBNETS and SSAST's embed / FFN widths and patch shapes), so a new geometry fails here, without a GPU, until
its shapes have a block test; SSAST's patch GEMM counts as covered through test_ssast_blocks_gpu.PATCH_GEMMS, which
must keep, for each model, its smallest window and the windows on each side of a 128-row tile. The recurrent
models' GEMMs are fixed by those models and are stated with the model.cu function that builds each. Convolutions (the
conv stack, positional conv, NPC, modified CPC's conv 1..4) have block tests of their own and are not listed."""
from dataclasses import replace

from s3prl_b200.upstream import apc, cpc, decoar, lighthubert, ssast
from s3prl_b200.upstream.configs import ARCHS, XLS_R
from s3prl_b200.upstream.decoar2 import DECOAR2
from test_blocks_gpu import LINEAR_CASES
from test_gemm_layouts_gpu import LINEAR_SHAPES, SPLIT_SLICES
from test_port_shapes_gpu import PORT_LINEARS
from test_ssast_blocks_gpu import PATCH_GEMMS

CONV_DIM = 512  # model.cu kConvDim: the conv stack's channels, post_extract_proj's K
FBANK_K = 128  # model.cu kDecoar2K: the 80 fbank bins zero-padded to whole 64-wide k-blocks

# (N, K) of the recurrent models' GEMMs, by the model.cu function that builds them
FIXED = {
    # add_gru_stack: APC's GRU input GEMM, 3 gates of 512, over the fbank bins (layer 0) or the 512-wide layer below
    "apc.gru_input_l0": (3 * 512, FBANK_K),
    "apc.gru_input": (3 * 512, 512),
    # add_lstm_stack: DeCoAR's proj from the fbank bins to 1024, then per direction the LSTM input GEMM, 4 gates of
    # 1024, over the proj output (layer 0) or its direction's half of the 2048-wide layer below (lda 2048)
    "decoar.proj": (1024, FBANK_K),
    "decoar.lstm_input": (4 * 1024, 1024),
    # add_cpc_stack: modified CPC's LSTM input GEMM, 4 gates of 256, over conv 4's 256 channels
    "cpc.lstm_input": (4 * 256, 256),
}
# (N, K, lda) of the GEMMs that read a column slice of A: add_pred_heads (below, from the distiller's geometry) and
# add_lstm_stack's layers above 0
FIXED_SLICES = {"decoar.lstm_input": (4 * 1024, 1024, 2 * 1024)}


def _geometries():
    """name -> ArchConfig of every transformer or Conformer encoder served."""
    geo = {f"configs.ARCHS[{n!r}]": a for n, a in ARCHS.items()}
    geo.update({f"configs.XLS_R[{n!r}]": a for n, a in XLS_R.items()})
    geo["decoar2.DECOAR2"] = DECOAR2
    sup = lighthubert.supernet_arch({})
    for key, (E, H, F) in lighthubert.SUBNETS.items():  # as select_subnet cuts them
        geo[f"lighthubert.SUBNETS[{key}]"] = replace(sup, encoder_embed_dim=E, encoder_attention_heads=H,
                                                     encoder_ffn_embed_dim=F)
    return geo


def _linears(arch):
    """layer -> (N, K) of the GEMMs one encoder runs."""
    D, F = arch.encoder_embed_dim, arch.encoder_ffn_embed_dim
    if arch.conformer:  # add_conformer_layer: two FFNs, [q | k] and v, out, pointwise_conv1 and 2
        shapes = {"ffn.w_1": (F, D), "ffn.w_2": (D, F), "qk": (2 * D, D), "v": (D, D), "out": (D, D),
                  "pw1": (2 * D, D), "pw2": (D, D)}
    else:  # add_transformer_layer
        shapes = {"qkv": (3 * D, D), "out_proj": (D, D), "fc1": (F, D), "fc2": (D, F)}
    shapes["post_extract_proj"] = (D, CONV_DIM if arch.frontend == "conv" else FBANK_K)
    if arch.pred_heads:  # add_pred_heads: Linear(D, heads D) + GELU, then SplitLinear's [D][D] per head
        shapes["pred_heads"] = (arch.pred_heads * D, D)
        shapes["pred_split"] = (D, D)
    return shapes


def _ssast_linears():
    """layer -> (N, K) of SSAST's GEMMs: add_transformer_layer's four at the served width, and per model the patch
    GEMM that ssast_patch_params builds, [fshape x tshape] patch columns into the embedding width."""
    D, F = ssast.EMBED, ssast.FFN
    shapes = {"ssast.qkv": (3 * D, D), "ssast.out_proj": (D, D), "ssast.fc1": (F, D), "ssast.fc2": (D, F)}
    for kind, ((fs, ts), _) in ssast.KINDS.items():
        shapes[f"ssast_{kind}.patch_embed (model.cu ssast_patch_params)"] = (D, fs * ts)
    return shapes


def _covered():
    return ({(N, K) for _, N, K, _ in PORT_LINEARS} | {(N, K) for K, N in LINEAR_SHAPES}
            | {(N, K) for _, N, K, *_ in LINEAR_CASES} | {(N, K) for _, N, K, *_ in PATCH_GEMMS})


def _served():
    """(N, K) -> the layers that run it."""
    served = {}
    for gname, arch in _geometries().items():
        for layer, nk in _linears(arch).items():
            served.setdefault(nk, []).append(f"{gname}.{layer}")
    for layer, nk in list(FIXED.items()) + list(_ssast_linears().items()):
        served.setdefault(nk, []).append(layer)
    return served


def test_lighthubert_subnets_are_the_served_ones():
    """The subnets formed here are those select_subnet serves for the hub's checkpoints."""
    geo = list(_geometries().values())
    for kind in lighthubert.KINDS:
        _, sub = lighthubert.select_subnet(lighthubert.lighthubert_config(kind))
        assert sub in geo, kind


def test_fixed_shapes_match_the_models():
    """FIXED is stated by hand; a recurrent model whose width changes must change it too."""
    assert (apc.HIDDEN, apc.NUM_MEL_BINS) == (512, 80)
    assert (decoar.HIDDEN, decoar.NUM_MEL_BINS) == (1024, 80)
    assert cpc.HIDDEN == 256
    assert DECOAR2.frontend == "fbank"


def test_every_served_gemm_shape_has_a_block_test():
    covered = _covered()
    missing = {nk: layers for nk, layers in _served().items() if nk not in covered}
    assert not missing, "GEMM shapes (N, K) without a block test: " + "; ".join(
        f"{nk} run by {', '.join(layers[:3])}" + (f" and {len(layers) - 3} more" if len(layers) > 3 else "")
        for nk, layers in sorted(missing.items()))


def test_every_served_column_slice_has_a_block_test():
    """The GEMMs that read a strided column slice of A: test_gemm_layouts_gpu.test_linear_split_slice runs each
    (N, K, lda) at every a_off the model uses."""
    want = dict(FIXED_SLICES)
    for gname, arch in _geometries().items():
        if arch.pred_heads:
            D = arch.encoder_embed_dim
            want[f"{gname}.pred_split"] = (D, D, arch.pred_heads * D)
    have = {}
    for N, K, lda, a_off in SPLIT_SLICES:
        have.setdefault((N, K, lda), set()).add(a_off)
    for layer, (N, K, lda) in want.items():
        assert have.get((N, K, lda), set()) == set(range(0, lda, K)), (layer, (N, K, lda))


def test_ssast_patch_gemm_table_keeps_its_edges():
    """test_ssast_blocks_gpu.PATCH_GEMMS runs, for each SSAST model, its smallest window (one time patch) and the
    windows just below and just above a 128-row M tile (the patch GEMM's rows per window: t_dim for the frame model,
    P = 12 t_dim for the patch model, which steps by 12), so that a change to the window rules cannot drop them."""
    for kind in ssast.KINDS:
        (_, ts), _ = ssast.KINDS[kind]
        rows_of = {}
        for _, N, K, k, secs in PATCH_GEMMS:
            if k == kind:
                g = ssast.geometry(kind, secs)
                rows_of[secs] = g["P"]
                assert (N, K) == (ssast.EMBED, 256)
        step = ssast.geometry(kind, 10.0)["f_dim"]
        smallest = ssast.geometry(kind, max(400, ts * 160) / 16000)
        assert smallest["t_dim"] == 1 and smallest["P"] in rows_of.values(), kind
        assert any(128 - step <= r < 128 for r in rows_of.values()), (kind, sorted(rows_of.values()))
        assert any(128 < r <= 128 + step for r in rows_of.values()), (kind, sorted(rows_of.values()))
