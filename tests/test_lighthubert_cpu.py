"""LightHuBERT without a GPU: subnet choice, the cut against the reference's own set_sample_config, the config and
checkpoint refusals, the fp64 oracle against the executed reference's goldens, the C ABI's acceptance of the new
widths, and the hub entries."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import lighthubert_oracle as LO  # noqa: E402

GOLDENS = ("lighthubert_small", "lighthubert_base", "lighthubert_stage1", "lighthubert_student_small",
           "lighthubert_small_c2", "lighthubert_variant_default", "lighthubert_variant_bias")


def _reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()


@pytest.mark.parametrize(
    "over,width",
    [
        (dict(_name="hubert_pruner", pruner_supernet="x/lighthubert_small.yaml"), 384),
        (dict(_name="hubert_pruner", pruner_supernet="X/Base.YAML"), 640),
        (dict(_name="hubert_pruner", pruner_supernet="custom.yaml"), 640),  # supernet_type's default "base"
        (dict(_name="hubert_pruner", pruner_supernet="custom.yaml", supernet_type="small"), 384),
        (dict(_name="hubert_pruner", pruner_supernet="small.yaml", supernet_type="base"), 384),
        (dict(_name="student_hubert"), 768),
        (dict(_name="student_hubert", supernet_type="small"), 512),
        (dict(_name="student_hubert", pruner_supernet="small.yaml"), 768),  # students ignore pruner_supernet
    ],
)
def test_subnet_choice(over, width):
    from s3prl_b200.upstream.lighthubert import select_subnet

    _, sub = select_subnet(over)
    assert (sub.encoder_embed_dim, sub.encoder_attention_heads, sub.encoder_ffn_embed_dim) == (width, width // 64, 4 * width)
    assert sub.encoder_layers == 12 and sub.normalize and sub.family == "hubert"


@pytest.mark.parametrize("kind,over", [("small", {}), ("base", {}), ("stage1", {}), ("stage1", dict(supernet_type="small"))])
def test_cut_equals_reference_set_sample_config(kind, over):
    """Every tensor the forward reads equals the reference module's own sampled parameter after the expert's
    set_sample_config; pos_conv is compared as the folded weight the reference convolves with."""
    _reference()
    from s3prl.upstream.lighthubert.lighthubert import LightHuBERT, LightHuBERTConfig

    from s3prl_b200.upstream.lighthubert import (cut_subnet, fabricate_lighthubert_state_dict, lighthubert_config,
                                                 select_subnet, supernet_arch)

    cfg = lighthubert_config(kind, **over)
    stype, sub = select_subnet(cfg)
    sd = fabricate_lighthubert_state_dict(3, cfg)
    rc = LightHuBERTConfig(cfg)
    rc.supernet_type = stype
    model = LightHuBERT(rc)
    model.load_state_dict(sd, strict=True)
    model.set_sample_config(model.supernet.subnet if cfg["_name"] == "hubert_pruner" else model.supernet.max_subnet)
    cut = cut_subnet(sd, supernet_arch(cfg), sub)
    E = sub.encoder_embed_dim
    assert model.sample_embed_dim == E
    checked = 0
    for l, layer in enumerate(model.encoder.layers):
        p = f"encoder.layers.{l}"
        mods = {"self_attn.q_proj": layer.self_attn.q_proj, "self_attn.k_proj": layer.self_attn.k_proj,
                "self_attn.v_proj": layer.self_attn.v_proj, "self_attn.out_proj": layer.self_attn.out_proj,
                "fc1": layer.fc1, "fc2": layer.fc2}
        for n, m in mods.items():
            for w in ("weight", "bias"):
                assert torch.equal(cut[f"{p}.{n}.{w}"], m.samples[w]), (p, n, w)
                checked += 1
        for n in ("self_attn_layer_norm", "final_layer_norm"):
            m = getattr(layer, n)
            for w in ("weight", "bias"):
                assert torch.equal(cut[f"{p}.{n}.{w}"], m.samples[w]), (p, n, w)
    pe = model.post_extract_proj
    assert torch.equal(cut["post_extract_proj.weight"], pe.samples["weight"])
    assert torch.equal(cut["post_extract_proj.bias"], pe.samples["bias"])
    ln = model.encoder.layer_norm
    assert torch.equal(cut["encoder.layer_norm.weight"], ln.samples["weight"])
    conv = model.encoder.pos_conv[0]
    with torch.no_grad():
        # weight_norm's pre-forward hook forms the weight at supernet size, then SConv1d.forward cuts it
        w_ref, b_ref = conv._sample_parameters(torch._weight_norm(conv.weight_v, conv.weight_g, 2), conv.bias)
    v, g = cut["encoder.pos_conv.0.weight_v"].double(), cut["encoder.pos_conv.0.weight_g"].double()
    w = v * (g / v.norm(dim=(0, 1), keepdim=True))  # what s3b_model_finalize folds
    assert w.shape == w_ref.shape == (E, E // 16, 128)
    assert torch.allclose(w, w_ref.double(), rtol=1e-6, atol=1e-9)
    assert torch.equal(cut["encoder.pos_conv.0.bias"], b_ref)
    # a prefix slice of fc1 / fc2 or a norm over the cut v alone would not match
    if E < 768:
        assert not torch.equal(cut["encoder.layers.0.fc1.weight"], sd["encoder.layers.0.fc1.weight"][: 4 * E, :E])
        vc = sd["encoder.pos_conv.0.weight_v"][:E, : E // 16]
        w_local = vc * (sd["encoder.pos_conv.0.weight_g"] / vc.norm(dim=(0, 1), keepdim=True))
        assert not torch.allclose(w_local.double(), w_ref.double(), rtol=1e-3)
    assert checked == 12 * 12


def test_config_refusals_name_the_field():
    from s3prl_b200.upstream.lighthubert import lighthubert_config, select_subnet

    for over, field in ((dict(_name="hubert"), "_name"), (dict(encoder_layers=6), "encoder_layers"),
                        (dict(layer_type="conformer"), "layer_type"),
                        (dict(conv_feature_layers="[(512,10,5)] + [(512,3,2)] * 4"), "conv_feature_layers"),
                        (dict(pos_conv_depth=5), "pos_conv_depth"), (dict(layer_norm_first=True), "layer_norm_first"),
                        (dict(activation_fn="relu"), "activation_fn"),
                        (dict(encoder_embed_dim=512, encoder_attention_heads=8, encoder_ffn_embed_dim=2048),
                         "encoder_embed_dim")):
        with pytest.raises(ValueError, match=field):
            select_subnet(lighthubert_config("base", **over))
    cfg = lighthubert_config("small")
    del cfg["pruner_supernet"]
    with pytest.raises(ValueError, match="pruner_supernet"):
        select_subnet(cfg)
    # spacing of conv_feature_layers and unrelated keys are not refused
    _, sub = select_subnet(lighthubert_config("small", conv_feature_layers="[(512, 10, 5)] + [(512, 3, 2)] * 4 + "
                                              "[(512, 2, 2)] * 2", label_rate=50, teacher_embed_dim=768))
    assert sub.encoder_embed_dim == 384


def test_checkpoint_reader_and_missing_tensor(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.lighthubert import (LighthubertExpert, cut_subnet, fabricate_lighthubert_state_dict,
                                                 lighthubert_config, select_subnet, supernet_arch)

    cfg = lighthubert_config("base", conv_bias=True)
    sd = fabricate_lighthubert_state_dict(5, cfg)
    path = tmp_path / "lighthubert.pt"
    torch.save({"cfg": {"model": cfg}, "model": sd}, path)
    for n in ("lighthubert_local", "lighthubert_url", "lighthubert_small"):
        e = hub.ENTRIES[n](str(path), refresh=True)
        assert isinstance(e, LighthubertExpert) and e.hidden_size == 640 and e.supernet_type == "base"
        assert torch.equal(e._state_dict_host["feature_extractor.conv_layers.3.0.bias"],
                           sd["feature_extractor.conv_layers.3.0.bias"])
        assert torch.equal(e._state_dict_host["encoder.layers.4.fc2.bias"], sd["encoder.layers.4.fc2.bias"][:640])
    bad = dict(sd)
    del bad["encoder.layers.7.fc1.weight"]
    with pytest.raises(KeyError, match="encoder.layers.7.fc1.weight"):
        cut_subnet(bad, supernet_arch(cfg), select_subnet(cfg)[1])
    torch.save({"cfg": {"model": cfg}, "model": bad}, path)
    with pytest.raises(KeyError, match="encoder.layers.7.fc1.weight"):
        LighthubertExpert(str(path))
    torch.save({"cfg": {"model": dict(cfg, activation_fn="relu")}, "model": sd}, path)
    with pytest.raises(ValueError, match="activation_fn"):
        LighthubertExpert(str(path))
    torch.save({"model": sd}, path)
    with pytest.raises(ValueError, match="not a LightHuBERT checkpoint"):
        LighthubertExpert(str(path))


def test_hub_entries_and_wrapper_counts():
    from s3prl_b200 import hub
    from s3prl_b200.nn.upstream import S3PRLUpstream
    from s3prl_b200.upstream.lighthubert import LighthubertExpert, fabricate_lighthubert_state_dict

    names = ("lighthubert", "lighthubert_small", "lighthubert_base", "lighthubert_stage1")
    assert set(names) | {"lighthubert_local", "lighthubert_url"} <= set(hub.options())
    for n, width in zip(names, (384, 384, 640, 768)):
        e = hub.ENTRIES[n](refresh=True)
        assert isinstance(e, LighthubertExpert) and e.hidden_size == width and e.num_outputs == 13
        assert e.get_downsample_rates("hidden_states") == 320 and e.num_frames(16000) == 49
        up = S3PRLUpstream(n)
        assert up.num_layers == 13 and up.hidden_sizes == [width] * 13 and up.downsample_rates == [320] * 13
    for n in ("lighthubert_local", "lighthubert_url"):
        with pytest.raises(AssertionError):
            hub.ENTRIES[n]()
    for n in names + ("lighthubert_local", "lighthubert_url"):
        with pytest.raises(ValueError, match="remote"):
            hub.ENTRIES[n](ckpt="https://huggingface.co/mechanicalsea/lighthubert/resolve/main/lighthubert_small.pt")
    for kw in (dict(hooks=[("self.model", lambda i, o: o)]), dict(feature_selection="fairseq_layers")):
        with pytest.raises(TypeError):
            hub.ENTRIES["lighthubert"](**kw)
    r = LighthubertExpert(kind="base", randomize_seed=7)
    fresh = LighthubertExpert(kind="base")
    assert not torch.equal(r._state_dict_host["encoder.layers.0.fc1.weight"], fresh._state_dict_host["encoder.layers.0.fc1.weight"])
    assert set(fabricate_lighthubert_state_dict(0)) >= set(fresh._state_dict_host)


def _create(s3b_lib, **over):
    from s3prl_b200 import lib

    c = lib.S3BConfig(family=0, extractor_layer_norm=1, normalize_wav=1, num_layers=12, embed_dim=384, ffn_dim=1536,
                      num_heads=6, pos_conv_kernel=128, pos_conv_groups=16, proj_hidden0=1)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_model_create(C.byref(c), C.byref(h))
    if rc == 0:
        s3b_lib.s3b_model_destroy(h)
    return rc, s3b_lib.s3b_last_error().decode()


def test_c_abi_accepts_the_subnet_widths_and_refuses_the_rest(s3b_lib):
    for E, H, F in ((384, 6, 1536), (640, 10, 2560), (768, 12, 3072), (512, 8, 2048)):
        assert _create(s3b_lib, embed_dim=E, num_heads=H, ffn_dim=F)[0] == 0, E
    assert _create(s3b_lib, proj_hidden0=0)[0] == 0
    for over, msg in ((dict(pos_conv_kernel=126), "multiple of 4"), (dict(pos_conv_depth=5, family=1, proj_hidden0=0), "pos_conv_depth"),
                      (dict(proj_hidden0=2), "proj_hidden0"), (dict(family=1), "proj_hidden0"),
                      (dict(layer_norm_first=1), "proj_hidden0"), (dict(embed_dim=640, num_heads=10, pos_conv_groups=32), "= 20)")):
        rc, err = _create(s3b_lib, **over)
        assert rc != 0 and msg in err, (over, err)


@pytest.mark.parametrize("fixture", GOLDENS)
def test_oracle_matches_executed_reference(fixture):
    from s3prl_b200.upstream.lighthubert import cut_subnet, fabricate_lighthubert_state_dict, select_subnet, supernet_arch

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    cfg = g["config"]
    _, sub = select_subnet(cfg)
    sd = cut_subnet(fabricate_lighthubert_state_dict(g["weight_seed"], cfg), supernet_arch(cfg), sub)
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        gen = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(m, generator=gen) * case["wav_scale"] for m in case["lens"]]
        with torch.no_grad():
            hs = LO.lighthubert_forward(wavs, sd, sub)
        assert len(hs) == case["num_hidden"] == 13 and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            s = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            ref = case["sub"][l].double()
            err = ((s - ref).norm() / ref.norm()).item()
            print(f"{fixture} lens={case['lens']} state {l}: abs max {h.abs().max().item():.3f}, oracle vs reference {err:.2e}")
            assert err < 2e-5, (fixture, l, err)
            assert abs(h.norm().item() / case["norms"][l].item() - 1) < 2e-5
        # hidden state 0's padded frames come out as zeros in the reference too (its in-place index_put)
        chunk = max(case["lens"]) // hs[0].shape[1]
        for b, n in enumerate(case["lens"]):
            v = -(-n // chunk)
            if ts == 1 and v < hs[0].shape[1]:
                assert torch.all(case["sub"][0][b, v:] == 0) and torch.all(hs[0][b, v:] == 0)
