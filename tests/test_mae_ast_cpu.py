"""MAE-AST without a GPU: the fp64 oracle against the executed reference's goldens, the frame, valid-token and
minimum-length rules against the reference expert, the fabricated file in the reference model, the loader's and the C
ABI's refusals, the hub entries, the coverage of MAE-AST's GEMM shapes and kernel configurations by its own block
tests, and ptxas's register report of the new kernels."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import mae_ast_oracle as MO  # noqa: E402
from test_mae_ast_gpu import ATTN_CASES, FRONT_LENS, GOLDENS, PROJ_ROWS  # noqa: E402
from test_ptxas_cpu import _assert_no_spills, _ptxas_report  # noqa: E402

CSRC = ROOT / "s3prl_b200" / "csrc"


def _reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()


def _wavs(lens, seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) * scale for n in lens]


@pytest.mark.parametrize("fixture", GOLDENS)
def test_oracle_matches_executed_reference(fixture):
    from s3prl_b200.upstream.mae_ast import fabricate_mae_ast_state_dict, prepare_mae_ast_tensors

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ck = fabricate_mae_ast_state_dict(g["weight_seed"], g["kind"], max_token_length=g["max_token_length"],
                                      **g["fabricate"])
    cfg, sd = prepare_mae_ast_tensors(ck, g["kind"])
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        with torch.no_grad():
            hs = MO.mae_ast_forward(_wavs(case["lens"], case["wav_seed"], case["wav_scale"]), sd, cfg)
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            s = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            ref = case["sub"][l].double()
            err = ((s - ref).norm() / ref.norm()).item()
            print(f"{fixture} lens={case['lens']} state {l}: oracle vs reference {err:.2e}")
            assert err < 2e-5, (fixture, l, err)
            assert abs(h.norm().item() / case["norms"][l].item() - 1) < 2e-5


def test_goldens_cover_the_mask_paths():
    """Ragged goldens have an utterance whose last patch is partly padded; the equal-length one takes the reference's
    fast exit (no utterance padded at its last frame)."""
    for fixture in GOLDENS:
        g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
        kt = MO.KINDS[g["kind"]][0]
        for case in g["cases"]:
            n = [1 + (L - 400) // 160 for L in case["lens"]]
            if fixture.endswith("_c2"):
                assert len(set(n)) == 1
    for fixture in ("mae_ast_frame", "mae_ast_patch", "mae_ast_variant"):
        g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
        kt = MO.KINDS[g["kind"]][0]
        n = [1 + (L - 400) // 160 for L in g["cases"][0]["lens"]]
        assert any(v % kt and v < max(n) for v in n), fixture


def _reference_expert(tmp_path, ck):
    _reference()
    from s3prl.upstream.mae_ast.expert import UpstreamExpert

    path = tmp_path / "mae_ast.pt"
    torch.save(ck, path)
    ex = UpstreamExpert(str(path))
    ex.eval()
    return ex


@pytest.mark.parametrize("kind", ["frame", "patch"])
def test_frame_and_valid_token_rules_match_the_reference(tmp_path, kind):
    """T', the output length and each utterance's valid tokens (the reference's padding mask, read back from its
    model) at small sizes, on both sides of a patch boundary; the C ABI gives the same numbers."""
    from s3prl_b200 import lib
    from s3prl_b200.upstream.mae_ast import fabricate_mae_ast_state_dict, num_frames, valid_frames

    ck = fabricate_mae_ast_state_dict(1, kind, layers=1, max_token_length=1024)
    ex = _reference_expert(tmp_path, ck)
    kt, kc = MO.KINDS[kind]
    nv = 128 // kc
    seen = {}
    orig = ex.model.forward_padding_mask

    def spy(features, padding_mask, feature_dim=128):
        m = orig(features, padding_mask, feature_dim)
        seen["valid"] = (~m).sum(-1).tolist()
        return m

    ex.model.forward_padding_mask = spy
    h = C.c_void_p()
    s3b = lib.load()
    cfg = lib.S3BMaeAstConfig(patch=int(kind == "patch"), embed_dim=768, num_heads=12, ffn_dim=3072, num_layers=1,
                              sine_pos=1, max_tokens=1024)
    lib.check(s3b.s3b_mae_ast_model_create(C.byref(cfg), C.byref(h)))
    try:
        edge = 400 + 160 * (kt - 1)
        for lens in ([edge, 400], [edge + 159, edge - 1], [edge + 160, 559, 400], [16000, 9000, 5360, 12345],
                     [5360, 5360], [2 * edge - 1, 1000]):
            with torch.no_grad():
                hs = ex(_wavs(lens, 3))["hidden_states"]
            L = max(lens)
            T = num_frames(kind, L)
            assert hs[0].shape[1] == T == s3b.s3b_num_frames(h, L), (lens, T)
            assert hs[0].shape[2] == nv * 768
            valid = (C.c_int32 * len(lens))()
            lib.check(s3b.s3b_valid_frames(h, (C.c_int64 * len(lens))(*lens), len(lens), L, valid))
            assert [v * nv for v in valid] == [v * nv for v in valid_frames(kind, lens, L)] == seen["valid"], lens
        # below one patch in the longest utterance there is no output frame
        assert num_frames(kind, edge - 1) == 0 and s3b.s3b_num_frames(h, edge - 1) == -1
        # under 400 samples an utterance has no fbank frame: the reference's fbank refuses it, and so does the library
        with torch.no_grad(), pytest.raises(AssertionError, match="window size"):
            ex(_wavs([edge, 399], 4))
        valid = (C.c_int32 * 2)()
        assert s3b.s3b_valid_frames(h, (C.c_int64 * 2)(edge, 399), 2, edge, valid) != 0
        assert "400 samples" in s3b.s3b_last_error().decode()
    finally:
        s3b.s3b_model_destroy(h)


def test_expert_refuses_short_utterances():
    from s3prl_b200.upstream.mae_ast import MaeAstExpert

    for kind, edge in (("frame", 560), ("patch", 2800)):
        ex = MaeAstExpert(kind=kind)
        with pytest.raises(ValueError, match="400"):
            ex._batch([torch.zeros(edge), torch.zeros(399)])
        with pytest.raises(ValueError, match=str(edge)):
            ex._batch([torch.zeros(edge - 1)])
        assert ex._batch([torch.zeros(edge), torch.zeros(400)])[2] == 1


@pytest.mark.parametrize("kw", [dict(kind="frame"), dict(kind="patch"),
                                dict(kind="patch", layers=3, layer_norm_first=True, enc_sine_pos=False)],
                         ids=["frame", "patch", "variant"])
def test_fabricated_file_loads_strictly_into_the_reference(tmp_path, kw):
    """The reference expert builds MAE_AST from the file's cfg and loads its state dict with strict=True."""
    from s3prl_b200.upstream.mae_ast import fabricate_mae_ast_state_dict

    ck = fabricate_mae_ast_state_dict(2, max_token_length=256, **kw)
    ex = _reference_expert(tmp_path, ck)
    ref = ex.model.state_dict()
    assert set(ref) == set(ck["model"])
    for k, t in ck["model"].items():
        assert torch.equal(ref[k], t), k
    assert ex.get_downsample_rates("hidden_states") == 160 * MO.KINDS[kw["kind"]][0]
    # the released configuration: post-LN, sinusoid pe from the formula, non-trivial batch-norm statistics
    if kw.get("layers") is None:
        assert ck["cfg"]["model"]["enc_sine_pos"] and ck["cfg"]["model"]["dec_sine_pos"]
        assert not ck["cfg"]["model"]["layer_norm_first"] and ck["cfg"]["model"]["decoder_layers"] == 2
        rm, rv = ck["model"]["batch_norm.running_mean"].item(), ck["model"]["batch_norm.running_var"].item()
        assert rm != 0 and rv != 1


def test_fabricated_pe_is_the_sinusoid_formula():
    _reference()
    from s3prl.upstream.mae_ast.mae_ast import SinusoidalPositionalEncoding

    from s3prl_b200.upstream.mae_ast import fabricate_mae_ast_state_dict

    ck = fabricate_mae_ast_state_dict(0, "frame", layers=1, max_token_length=300)
    assert torch.equal(ck["model"]["enc_sine_pos_embed.pe"], SinusoidalPositionalEncoding(768, 300).pe)


def test_loader_refusals_name_the_field(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.mae_ast import MaeAstExpert, fabricate_mae_ast_state_dict

    def save(ck, name="x.pt"):
        p = tmp_path / name
        torch.save(ck, p)
        return str(p)

    ck = fabricate_mae_ast_state_dict(1, "frame", max_token_length=64)

    def variant(model=None, task=None, drop=None):
        c = {"cfg": {"model": dict(ck["cfg"]["model"], **(model or {})), "task": dict(ck["cfg"]["task"], **(task or {}))},
             "model": {k: v for k, v in ck["model"].items() if k != drop}}
        return save(c)

    for drop in ("encoder.layers.7.fc2.bias", "post_extract_proj.weight", "batch_norm.running_var",
                 "enc_sine_pos_embed.pe", "encoder.layer_norm.weight"):
        with pytest.raises(KeyError, match=drop.replace(".", r"\.")):
            MaeAstExpert(ckpt=variant(drop=drop), kind="frame")
    # pre-LN without sine positions needs neither encoder.layer_norm nor pe
    c = fabricate_mae_ast_state_dict(1, "frame", layers=2, layer_norm_first=True, enc_sine_pos=False)
    c["model"] = {k: v for k, v in c["model"].items() if not k.startswith("encoder.layer_norm")}
    assert MaeAstExpert(ckpt=save(c, "pre.pt"), kind="frame").num_outputs == 2
    for model, task, field in (
        ({}, {"sample_rate": 8000}, "task.sample_rate"),
        ({}, {"feature_dim": 80}, "task.feature_dim"),
        ({"ast_kernel_size_time": 4}, {}, "ast_kernel_size_time"),
        ({"ast_kernel_stride_time": 1}, {}, "ast_kernel_stride_time"),
        ({"ast_kernel_stride_chan": 64}, {}, "ast_kernel_stride_chan"),
        ({"encoder_embed_dim": 1024}, {}, "encoder_embed_dim"),
        ({"encoder_attention_heads": 16}, {}, "encoder_attention_heads"),
        ({"encoder_ffn_embed_dim": 4096}, {}, "encoder_ffn_embed_dim"),
        ({"encoder_layers": 0}, {}, "encoder_layers"),
        ({"activation_fn": "relu"}, {}, "activation_fn"),
        ({"enc_conv_pos": True}, {}, "enc_conv_pos"),
    ):
        with pytest.raises(ValueError, match=field):
            MaeAstExpert(ckpt=variant(model, task), kind="frame")
    # a named entry given a file of the other geometry
    with pytest.raises(ValueError, match="ast_kernel_size_time"):
        hub.mae_ast_patch(variant())
    with pytest.raises(ValueError, match="not an MAE-AST checkpoint"):
        MaeAstExpert(ckpt=save({"model": {}}, "bad.pt"))
    bad = dict(ck["model"], **{"enc_sine_pos_embed.pe": torch.zeros(1, 8, 384)})
    with pytest.raises(ValueError, match="enc_sine_pos_embed.pe"):
        MaeAstExpert(ckpt=save({"cfg": ck["cfg"], "model": bad}, "pe.pt"))
    with pytest.raises(TypeError, match="hooks"):
        MaeAstExpert(hooks=[("x", None)])


def test_hub_entries(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.mae_ast import MaeAstExpert, fabricate_mae_ast_state_dict

    assert {"mae_ast_frame", "mae_ast_patch", "mae_ast_local", "mae_ast_url"} <= set(hub.options())
    for name, width, rate, T in (("mae_ast_frame", 768, 320, 49), ("mae_ast_patch", 8 * 768, 2560, 6)):
        e = hub.ENTRIES[name](refresh=True)
        assert isinstance(e, MaeAstExpert) and e.hidden_size == width and e.num_outputs == 12
        assert e.get_downsample_rates("hidden_states") == rate and e.num_frames(16000) == T
        assert e.pe_rows == 48000
    path = tmp_path / "patch.pt"
    torch.save(fabricate_mae_ast_state_dict(5, "patch", layers=2, max_token_length=128), path)
    for name in ("mae_ast_local", "mae_ast_url"):
        e = hub.ENTRIES[name](str(path))
        assert e.kind == "patch" and e.num_outputs == 2 and e.pe_rows == 128
        with pytest.raises(AssertionError):
            hub.ENTRIES[name]()
    assert hub.mae_ast_patch(str(path)).num_outputs == 2
    with pytest.raises(ValueError, match="remote checkpoints"):
        hub.mae_ast_url("https://www.cs.utexas.edu/~harwath/model_checkpoints/mae_ast/random_frame_75_12LayerEncoder.pt")
    with pytest.raises(ValueError, match="remote checkpoints"):
        hub.mae_ast_frame(ckpt="https://example.org/x.pt")


def test_run_downstream_injection():
    """The launcher installs every hub entry into the reference's s3prl.hub."""
    import types

    from s3prl_b200 import hub

    mod = types.ModuleType("s3prl_hub_stub")
    names = hub.install(mod)
    for name in ("mae_ast_frame", "mae_ast_patch", "mae_ast_local", "mae_ast_url"):
        assert name in names and getattr(mod, name) is hub.ENTRIES[name]


def _create(s3b, **over):
    from s3prl_b200 import lib

    c = lib.S3BMaeAstConfig(patch=0, embed_dim=768, num_heads=12, ffn_dim=3072, num_layers=12, sine_pos=1,
                            max_tokens=48000)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b.s3b_mae_ast_model_create(C.byref(c), C.byref(h))
    if rc == 0:
        s3b.s3b_model_destroy(h)
    return rc, s3b.s3b_last_error().decode()


def test_c_abi_refusals(s3b_lib):
    for over in (dict(), dict(patch=1), dict(num_layers=1), dict(num_layers=63), dict(layer_norm_first=1),
                 dict(sine_pos=0, max_tokens=0)):
        assert _create(s3b_lib, **over)[0] == 0, over
    for over, msg in ((dict(patch=2), "patch must be"), (dict(embed_dim=1024), "embed_dim"),
                      (dict(num_heads=16), "num_heads"), (dict(ffn_dim=4096), "ffn_dim"),
                      (dict(num_layers=0), "num_layers"), (dict(num_layers=64), "num_layers"),
                      (dict(layer_norm_first=2), "layer_norm_first"), (dict(sine_pos=2), "sine_pos"),
                      (dict(max_tokens=0), "max_tokens"), (dict(sine_pos=0), "max_tokens"),
                      (dict(struct_size=8), "struct_size")):
        rc, err = _create(s3b_lib, **over)
        assert rc != 0 and msg in err, (over, err)
    from s3prl_b200 import lib

    c = lib.S3BMaeAstConfig(patch=0, embed_dim=768, num_heads=12, ffn_dim=3072, num_layers=12, sine_pos=1, max_tokens=9)
    c.reserved[2] = 1
    h = C.c_void_p()
    assert s3b_lib.s3b_mae_ast_model_create(C.byref(c), C.byref(h)) != 0
    assert "reserved[2]" in s3b_lib.s3b_last_error().decode()


def test_block_tests_cover_the_models_shapes():
    """MAE-AST's GEMMs are post_extract_proj (768, 256) and the wav2vec 2.0 encoder linears at width 768, which the
    GEMM layout tests already run; its key masks are multiples of nv tokens. The new block tests hold rows on both sides
    of a 128-row tile for the projection and at the 32 x 10 s frame model's M, key counts that are multiples of 8 but
    not of 64, and front-end lengths with n_b a multiple of kt and not, for both patch sizes."""
    from test_gemm_layouts_gpu import LINEAR_SHAPES

    from s3prl_b200.upstream.mae_ast import num_frames

    for k, n in ((768, 2304), (768, 768), (768, 3072), (3072, 768)):
        assert (k, n) in LINEAR_SHAPES
    assert {127, 128, 129} <= set(PROJ_ROWS) and 32 * num_frames("frame", 160000) in PROJ_ROWS
    for N, valid in ATTN_CASES:
        assert any(v % 8 == 0 and v % 64 != 0 for v in valid) and N in valid
    assert {8 * num_frames("patch", 160000), 8 * num_frames("patch", 16000), num_frames("frame", 160000)} == {
        N for N, _ in ATTN_CASES}
    frames = [1 + (n - 400) // 160 for n in FRONT_LENS]
    for kt in (2, 16):
        assert any(f % kt == 0 for f in frames) and any(f % kt for f in frames)
    assert min(FRONT_LENS) == 400


def test_ptxas_no_spills(tmp_path):
    """The positions + LayerNorm kernel and the front-end kernel keep everything in registers."""
    _assert_no_spills(_ptxas_report(tmp_path, CSRC / "mae_ast.cu"))
    log = _ptxas_report(tmp_path, CSRC / "fbank.cu")
    assert "mae_ast_fbank_kernel" in log
    _assert_no_spills(log)
