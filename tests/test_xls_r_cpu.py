"""CPU tests of the XLS-R 1B / 2B support (80- and 120-wide attention heads, 1920-channel encoders): the C ABI's
configuration checks, configuration parsing, converted-checkpoint round trips through wav2vec2_local, the attention
kernels' register use, and the CPU oracle against the executed-reference goldens (tools/make_xls_r_golden.py). None of
them needs a GPU."""
import ctypes as C
import re
import subprocess
import sys
from dataclasses import replace
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"


def _create(s3b_lib, cfg, **over):
    from s3prl_b200.upstream.expert import _c_config

    c = _c_config(cfg)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_model_create(C.byref(c), C.byref(h))
    if rc == 0:
        s3b_lib.s3b_model_destroy(h)
    return rc, s3b_lib.s3b_last_error().decode()


def test_table_values_and_not_hub_entries():
    from s3prl_b200 import hub
    from s3prl_b200.upstream.configs import ARCHS, XLS_R

    one, two = XLS_R["xls_r_1b"], XLS_R["xls_r_2b"]
    assert (one.encoder_layers, one.encoder_embed_dim, one.encoder_ffn_embed_dim, one.encoder_attention_heads) == (
        48, 1280, 5120, 16)
    assert (two.encoder_layers, two.encoder_embed_dim, two.encoder_ffn_embed_dim, two.encoder_attention_heads) == (
        48, 1920, 7680, 16)
    for a in (one, two):
        assert a.family == "wav2vec2" and a.extractor_mode == "layer_norm" and a.conv_bias and a.layer_norm_first
        assert a.normalize and (a.conv_pos, a.conv_pos_groups) == (128, 16) and not a.conformer
    assert not set(XLS_R) & set(ARCHS) and not set(XLS_R) & set(hub.options())


def test_model_create_accepts_and_refuses(s3b_lib):
    from s3prl_b200 import lib
    from s3prl_b200.upstream.configs import ARCHS, XLS_R

    for name, a in XLS_R.items():
        assert _create(s3b_lib, a) == (0, s3b_lib.s3b_last_error().decode()), name
    one = XLS_R["xls_r_1b"]
    for over in (dict(embed_dim=768, num_heads=16, ffn_dim=3072),  # 48-wide heads
                 dict(embed_dim=1536, num_heads=16, ffn_dim=6144),  # 96
                 dict(num_heads=10)):  # 128
        rc, msg = _create(s3b_lib, one, **over)
        assert rc != 0 and "head dim" in msg and "64, 80 or 120" in msg, (over, msg)
    rc, msg = _create(s3b_lib, one, embed_dim=2048, num_heads=16, ffn_dim=8192)
    assert rc != 0 and "embed_dim" in msg and "1920" in msg
    rc, msg = _create(s3b_lib, ARCHS["wavlm_large"], embed_dim=1280, num_heads=16, ffn_dim=5120)
    assert rc != 0 and "wavlm" in msg and "num_heads" in msg, msg
    rc, msg = _create(s3b_lib, ARCHS["wav2vec2_conformer_rope"], embed_dim=1280, num_heads=16, ffn_dim=5120)
    assert rc != 0 and "conformer" in msg and "num_heads" in msg, msg
    rc, msg = _create(s3b_lib, one, pos_conv_groups=10)  # 128 channels per group
    assert rc != 0 and "16, 32, 48, 64, 80 or 120" in msg
    assert lib.FAMILY_WAV2VEC2 == 1


def test_arch_from_reference_cfg():
    """XLS-R-style fairseq model_cfg / task_cfg dicts (as converted from the released files) map onto the table."""
    from s3prl_b200.upstream.configs import XLS_R, arch_from_reference_cfg
    from s3prl_b200.upstream.convert import reference_model_cfg

    for name, a in XLS_R.items():
        model_cfg = dict(
            _name="wav2vec2", extractor_mode="layer_norm", encoder_layers=48, encoder_embed_dim=a.encoder_embed_dim,
            encoder_ffn_embed_dim=a.encoder_ffn_embed_dim, encoder_attention_heads=16, activation_fn="gelu",
            layer_norm_first=True, conv_feature_layers="[(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512,2,2)] + [(512,2,2)]",
            conv_bias=True, conv_pos=128, conv_pos_groups=16, latent_temp=[2.0, 0.1, 0.999995], quantize_targets=True,
            feature_grad_mult=1.0,
        )
        assert arch_from_reference_cfg("wav2vec2", model_cfg, {"_name": "audio_pretraining", "normalize": True}) == a
        assert arch_from_reference_cfg("wav2vec2", reference_model_cfg(a), {"normalize": True}) == a, name


def test_converted_checkpoint_round_trip(tmp_path):
    """2-layer variants of both shapes: save_converted_checkpoint -> load_reference_checkpoint and wav2vec2_local
    give back the configuration and every tensor (no GPU needed until the first forward)."""
    from s3prl_b200 import hub
    from s3prl_b200.upstream.configs import XLS_R
    from s3prl_b200.upstream.convert import save_converted_checkpoint
    from s3prl_b200.upstream.weights import fabricate_state_dict, load_reference_checkpoint

    for name, a in XLS_R.items():
        cfg = replace(a, encoder_layers=2)
        sd = fabricate_state_dict(cfg, 0)
        assert sd["encoder.pos_conv.0.weight_v"].shape == (cfg.encoder_embed_dim, cfg.encoder_embed_dim // 16, 128)
        path = tmp_path / f"{name}.pt"
        save_converted_checkpoint(path, cfg, sd)
        got_cfg, got_sd = load_reference_checkpoint(str(path), "wav2vec2")
        assert got_cfg == cfg, name
        assert got_sd.keys() == sd.keys() and all(torch.equal(got_sd[k], sd[k]) for k in sd)
        e = hub.ENTRIES["wav2vec2_local"](str(path))
        assert e.arch == cfg and e.num_layers == 2
        assert hub.ENTRIES["wav2vec2_custom"](str(path)).arch == cfg


def test_attention_kernels_no_spill_no_serialisation(tmp_path):
    """ptxas -v on attention.cu with the library's flags: no C7520 (serialised wgmma) in any instantiation and no spill
    in the 80- and 120-wide ones (one CTA per SM, up to 168 registers). The 64-wide kernels are the unchanged ones
    (two CTAs per SM hold them to 96 registers, where ptxas keeps a few bytes of stack outside the key loop)."""
    sys.path.insert(0, str(ROOT))
    from s3prl_b200 import build

    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    src = ROOT / "s3prl_b200" / "csrc" / "attention.cu"
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas=-v", "-c", str(src), "-o", str(tmp_path / "attention.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, f"nvcc failed:\n{r.stderr}"
    log = r.stderr
    assert "C7520" not in log, log
    widths, current = {}, None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '_ZN3s3b16attention_kernelILi(\d+)ELb(\d)E", ln)
        if m:
            current = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and current is not None:
            widths[current] = int(m.group(1)) + int(m.group(2))
    assert set(widths) == {(64, 0), (64, 1), (80, 0), (120, 0)}, widths
    assert widths[(80, 0)] == 0 and widths[(120, 0)] == 0, widths


def _check_oracle_against_golden(fixture):
    """The shared CPU oracle (oracle/upstream_oracle.py) against the executed reference, with the bars
    tests/test_oracle_cpu.py applies to the other model fixtures (2e-5 relative per layer and on the norm)."""
    sys.path.insert(0, str(ROOT / "oracle"))
    import upstream_oracle as O

    from s3prl_b200.upstream.configs import XLS_R
    from s3prl_b200.upstream.weights import fabricate_state_dict

    fx = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    cfg = XLS_R[fx["arch"]]
    sd = fabricate_state_dict(cfg, seed=fx["weight_seed"])
    cs, ts = fx["channel_stride"], fx.get("time_stride", 1)
    worst = 0.0
    for case in fx["cases"]:
        g = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(n, generator=g) for n in case["lens"]]
        with torch.no_grad():
            hs, _pad = O.upstream_forward(wavs, sd, cfg)
        assert len(hs) == case["num_hidden"] == cfg.encoder_layers + 1
        assert tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            ref = case["sub"][l]
            got = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            rel = ((got.double() - ref.double()).norm() / ref.double().norm()).item()
            worst = max(worst, rel)
            assert rel < 2e-5, (fixture, l, rel)
            assert abs(h.double().norm().item() - case["norms"][l].item()) < 2e-5 * case["norms"][l].item()
    print(f"{fixture}: oracle vs reference, worst per-layer relative error {worst:.3e} (bound 2e-5)")


@pytest.mark.slow
@pytest.mark.parametrize("fixture", ["xls_r_1b", "xls_r_2b"])
def test_oracle_matches_reference(fixture):
    _check_oracle_against_golden(fixture)
