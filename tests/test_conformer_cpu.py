"""CPU tests of the wav2vec 2.0 Conformer (rotary attention) support: configuration parsing and refusals, the fabricated
checkpoint against the reference's own model skeleton, the C ABI's configuration checks, the new kernels' register
use, and the Conformer oracle (tests/conformer_oracle.py) against the executed-reference goldens. None of them needs a
GPU."""
import ctypes as C
import subprocess
import sys
from dataclasses import replace
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]

CONFORMER_CFG = dict(
    layer_type="conformer", pos_enc_type="rope", attn_type="espnet", depthwise_conv_kernel_size=31,
    extractor_mode="layer_norm", conv_bias=True, layer_norm_first=True, encoder_layers=24, encoder_embed_dim=1024,
    encoder_ffn_embed_dim=4096, encoder_attention_heads=16,
)


def test_arch_entry_and_config_parsing():
    from s3prl_b200.upstream.configs import ARCHS, arch_from_reference_cfg
    from s3prl_b200.upstream.convert import reference_model_cfg

    a = ARCHS["wav2vec2_conformer_rope"]
    assert a.conformer and a.family == "wav2vec2" and a.family_id == 1
    assert (a.encoder_layers, a.encoder_embed_dim, a.encoder_ffn_embed_dim, a.encoder_attention_heads) == (24, 1024, 4096, 16)
    assert a.extractor_mode == "layer_norm" and a.conv_bias and a.layer_norm_first and a.normalize
    assert (a.pos_enc_type, a.attn_type, a.depthwise_conv_kernel_size) == ("rope", "espnet", 31)
    assert a.num_outputs == 25
    got = arch_from_reference_cfg("wav2vec2", CONFORMER_CFG, {"normalize": True})
    assert got == a
    assert arch_from_reference_cfg("wav2vec2", reference_model_cfg(a), {"normalize": True}) == a
    k15 = arch_from_reference_cfg("wav2vec2", dict(CONFORMER_CFG, depthwise_conv_kernel_size=15))
    assert k15.depthwise_conv_kernel_size == 15
    # a transformer checkpoint keeps today's fields
    t = arch_from_reference_cfg("wav2vec2", {"encoder_layers": 12})
    assert not t.conformer and t.layer_type == "transformer"


@pytest.mark.parametrize(
    "change,message",
    [
        (dict(pos_enc_type="rel_pos"), "rel_pos"),
        (dict(pos_enc_type="abs"), "'abs'"),
        (dict(attn_type=""), "attn_type"),
        (dict(attn_type="fairseq"), "attn_type"),
        (dict(depthwise_conv_kernel_size=30), "odd"),
        (dict(depthwise_conv_kernel_size=65), "odd"),
        (dict(layer_type="mamba"), "layer_type"),
    ],
)
def test_unsupported_conformers_are_refused(change, message):
    from s3prl_b200.upstream.configs import arch_from_reference_cfg

    with pytest.raises(ValueError, match=message):
        arch_from_reference_cfg("wav2vec2", dict(CONFORMER_CFG, **change))


def test_conformer_only_for_wav2vec2():
    from s3prl_b200.upstream.configs import arch_from_reference_cfg

    with pytest.raises(ValueError, match="wav2vec2"):
        arch_from_reference_cfg("hubert", CONFORMER_CFG)


def test_hub_entry_and_absent_variants():
    from s3prl_b200 import hub

    names = set(hub.options())
    assert "wav2vec2_conformer_rope" in names
    for n in ("wav2vec2_conformer_relpos", "xls_r_1b", "xls_r_2b"):
        assert n not in names
    assert not any("s2st" in n for n in names)


def test_fabricated_keys_load_into_the_reference_skeleton():
    """Every fabricated key exists in the reference's Wav2Vec2Model built from reference_model_cfg, with the same
    shape; the skeleton's only extra encoder keys are the unused pos_conv and two buffers: the rotary inv_freq and
    BatchNorm's num_batches_tracked (an eval forward reads neither's learned value)."""
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available on this machine")
    ref_runtime.activate()
    from s3prl.upstream.utils import merge_with_parent
    from s3prl.upstream.wav2vec2.wav2vec2_model import Wav2Vec2Config, Wav2Vec2Model

    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.convert import reference_model_cfg
    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = replace(ARCHS["wav2vec2_conformer_rope"], encoder_layers=2, depthwise_conv_kernel_size=15)
    sd = fabricate_state_dict(cfg, seed=0)
    skeleton = Wav2Vec2Model(merge_with_parent(Wav2Vec2Config, reference_model_cfg(cfg))).state_dict()
    unknown = sorted(set(sd) - set(skeleton))
    assert not unknown, unknown[:5]
    for k, v in sd.items():
        assert tuple(skeleton[k].shape) == tuple(v.shape), k
    extra = {k for k in set(skeleton) - set(sd) if k.startswith("encoder.")}
    allowed = ("rotary_emb.inv_freq", "batch_norm.num_batches_tracked")
    assert extra and all(k.startswith("encoder.pos_conv.") or k.endswith(allowed) for k in extra), extra
    assert any(k.endswith("batch_norm.running_var") for k in sd)
    var = sd["encoder.layers.0.conv_module.batch_norm.running_var"]
    assert 0.5 <= var.min() and var.max() <= 1.5
    assert sd["encoder.layers.0.conv_module.batch_norm.running_mean"].abs().max() > 0


def test_expert_refuses_layer_results_options():
    from s3prl_b200.upstream.expert import UpstreamExpert

    for kw in (dict(feature_selection="fairseq_layers"), dict(feature_selection="fairseq_layers_before_residual"),
               dict(hooks=[("self.model.encoder", lambda i, o: o[0])])):
        with pytest.raises(TypeError, match="Conformer"):
            UpstreamExpert(name="wav2vec2_conformer_rope", state_dict={}, **kw)


def _create(lib, s3b_lib, **fields):
    base = dict(family=1, extractor_layer_norm=1, conv_bias=1, layer_norm_first=1, num_layers=2, embed_dim=1024,
                ffn_dim=4096, num_heads=16, pos_conv_kernel=128, pos_conv_groups=16)
    cfg = lib.S3BConfig(**dict(base, **fields))
    h = C.c_void_p()
    r = s3b_lib.s3b_model_create(C.byref(cfg), C.byref(h))
    if r == 0:
        s3b_lib.s3b_model_destroy(h)
    return r, s3b_lib.s3b_last_error().decode()


def test_c_abi_config_checks(s3b_lib):
    from s3prl_b200 import lib

    assert C.sizeof(lib.S3BConfig) == 23 * 4  # the new fields come out of `reserved`
    assert _create(lib, s3b_lib)[0] == 0
    for k in (1, 3, 31, 63):
        assert _create(lib, s3b_lib, conformer=1, depthwise_kernel=k)[0] == 0, k
    for fields, msg in ((dict(conformer=1, depthwise_kernel=30), "odd"), (dict(conformer=1, depthwise_kernel=65), "odd"),
                        (dict(conformer=1, depthwise_kernel=0), "odd"), (dict(conformer=2, depthwise_kernel=31), "0 or 1"),
                        (dict(depthwise_kernel=31), "Conformer"), (dict(conformer=1, depthwise_kernel=31, family=0), "wav2vec2")):
        r, err = _create(lib, s3b_lib, **fields)
        assert r != 0 and msg in err, (fields, err)


def test_conformer_kernels_do_not_spill(tmp_path):
    """ptxas -v on the depthwise kernel's source and on norm.cu (LayerNorm + RoPE): no spill stores or loads."""
    sys.path.insert(0, str(ROOT))
    from s3prl_b200 import build

    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    for name in ("conformer.cu", "norm.cu"):
        src = ROOT / "s3prl_b200" / "csrc" / name
        cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas=-v", "-c", str(src), "-o", str(tmp_path / (src.stem + ".o"))]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, f"nvcc failed:\n{r.stderr}"
        kernels = [l for l in r.stderr.splitlines() if "Compiling entry function" in l]
        assert any("depthwise_glu_kernel" in l or "layernorm_rope_kernel" in l for l in kernels), name
        spills = [l for l in r.stderr.splitlines() if "spill" in l and not l.strip().startswith("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads")]
        assert not spills, spills


GOLDEN = ROOT / "tests" / "golden"


def _check_oracle_against_golden(fixture):
    """The Conformer oracle (tests/conformer_oracle.py) against the executed reference
    (tools/make_conformer_golden.py): same bars as tests/test_oracle_cpu.py's model fixtures."""
    import torch

    sys.path.insert(0, str(ROOT / "tests"))
    import conformer_oracle

    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.weights import fabricate_state_dict

    fx = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    cfg = ARCHS[fx["arch"]]
    sd = fabricate_state_dict(cfg, seed=fx["weight_seed"])
    cs, ts = fx["channel_stride"], fx.get("time_stride", 1)
    for case in fx["cases"]:
        g = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(n, generator=g) for n in case["lens"]]
        with torch.no_grad():
            hs, _pad = conformer_oracle.conformer_forward(wavs, sd, cfg)
        assert len(hs) == case["num_hidden"] == cfg.encoder_layers + 1
        assert tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            ref = case["sub"][l]
            got = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            rel = ((got.double() - ref.double()).norm() / ref.double().norm()).item()
            assert rel < 2e-5, (fixture, l, rel)
            assert abs(h.double().norm().item() - case["norms"][l].item()) < 2e-5 * case["norms"][l].item()


def test_oracle_matches_reference():
    _check_oracle_against_golden("conformer_rope")


@pytest.mark.slow
def test_oracle_matches_reference_at_baseline_size():
    _check_oracle_against_golden("conformer_rope_c3")
