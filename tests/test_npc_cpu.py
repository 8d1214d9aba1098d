"""CPU tests of NPC (``npc``): the C ABI's configuration checks and frame rules, the fabricated checkpoint against the
reference's ``NPC(...).state_dict()``, the checkpoint reader's refusals, the hub entries, ``S3PRLUpstream``'s counts,
the fp64 CPU oracle against the executed-reference goldens (tools/make_npc_golden.py) and the masking property of the
oracle. None of them needs a GPU."""
import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import apc_oracle as AO  # noqa: E402
import npc_oracle as NO  # noqa: E402

GOLDENS = ("npc_ref", "npc_ref_c2", "npc_ref_variant")


def _reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()


def _create(s3b_lib, **over):
    from s3prl_b200 import lib

    c = lib.S3BNpcConfig(n_blocks=4, hidden=512, kernel_size=15, mask_size=5, residual=1, batch_norm=1, act=0)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_npc_model_create(C.byref(c), C.byref(h))
    return rc, s3b_lib.s3b_last_error().decode(), h


def test_config_accepts_and_refuses(s3b_lib):
    from s3prl_b200 import lib

    assert C.sizeof(lib.S3BNpcConfig) == 12 * 4
    for over, outputs in ((dict(), 9), (dict(n_blocks=1, kernel_size=9, mask_size=1), 3),
                          (dict(n_blocks=2, kernel_size=9, mask_size=3, act=1, residual=0, batch_norm=0), 5)):
        rc, msg, h = _create(s3b_lib, **over)
        assert rc == 0, msg
        assert s3b_lib.s3b_num_outputs(h) == outputs
        s3b_lib.s3b_model_destroy(h)
    for over, want in ((dict(n_blocks=0), "n_blocks"), (dict(hidden=256), "hidden"), (dict(kernel_size=14), "kernel_size"),
                       (dict(mask_size=4), "mask_size"), (dict(kernel_size=13), "kernel_size"),
                       (dict(residual=2), "residual"), (dict(batch_norm=2), "batch_norm"), (dict(act=2), "act"),
                       (dict(struct_size=12), "struct_size")):
        rc, msg, _ = _create(s3b_lib, **over)
        assert rc != 0 and want in msg, (over, msg)
    c = lib.S3BNpcConfig(n_blocks=4, hidden=512, kernel_size=15, mask_size=5)
    c.reserved[1] = 1
    h = C.c_void_p()
    assert s3b_lib.s3b_npc_model_create(C.byref(c), C.byref(h)) != 0
    assert "reserved" in s3b_lib.s3b_last_error().decode()


def test_frame_rules(s3b_lib):
    from s3prl_b200.upstream.npc import num_frames

    rc, msg, h = _create(s3b_lib)
    assert rc == 0, msg
    try:
        for n in (400, 560, 16000, 160000):
            assert s3b_lib.s3b_num_frames(h, n) == num_frames(n) == 1 + (n - 400) // 160
        lens = [16000, 12345, 560]
        out = (C.c_int32 * 3)()
        assert s3b_lib.s3b_valid_frames(h, (C.c_int64 * 3)(*lens), 3, 16000, out) == 0
        assert list(out) == [98, 75, 2]
        assert s3b_lib.s3b_valid_frames(h, (C.c_int64 * 2)(16000, 559), 2, 16000, out) != 0
        assert "NPC" in s3b_lib.s3b_last_error().decode()
    finally:
        s3b_lib.s3b_model_destroy(h)


@pytest.mark.parametrize("over", [{}, {"n_blocks": 2, "kernel_size": 9, "mask_size": 3, "batch_norm": False,
                                       "residual": False, "vq": None}])
def test_fabricated_keys_match_the_reference_model(over):
    _reference()
    from s3prl.upstream.npc.npc import NPC

    from s3prl_b200.upstream.npc import fabricate_npc_state_dict, npc_config

    paras = npc_config(**over)["model"]["paras"]
    ref = NPC(80, **paras).state_dict()
    sd = fabricate_npc_state_dict(0, paras)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.items()}
    # the fabricated masks are the reference's own
    assert all(torch.equal(sd[k], ref[k]) for k in ref if k.endswith("conv_mask"))


def test_config_validation_and_refusals():
    from s3prl_b200.upstream.npc import npc_config, validate_config

    p = validate_config(npc_config())
    assert p == {"hidden_size": 512, "n_blocks": 4, "kernel_size": 15, "mask_size": 5, "residual": True,
                 "batch_norm": True, "activate": "relu"}
    assert validate_config(npc_config(activate="tanh", n_blocks=1, kernel_size=5, mask_size=1))["n_blocks"] == 1
    for over, want in ((dict(hidden_size=256), "hidden_size"), (dict(n_blocks=0), "n_blocks"),
                       (dict(kernel_size=14), "kernel_size"), (dict(mask_size=2), "mask_size"),
                       (dict(kernel_size=13), "kernel_size"), (dict(activate="gelu"), "activate"),
                       (dict(disable_cross_layer=True), "disable_cross_layer"),
                       (dict(dim_bottleneck=64, vq=None), "dim_bottleneck"), (dict(foo=1), "foo")):
        with pytest.raises(ValueError, match=want):
            validate_config(npc_config(**over))
    c = npc_config()
    del c["model"]["paras"]["mask_size"]
    with pytest.raises(ValueError, match="mask_size"):
        validate_config(c)
    for key, value in (("feat_type", "mfcc"), ("feat_dim", 40), ("cmvn", False), ("frame_shift", 12.5)):
        c = npc_config()
        c["data"]["audio"][key] = value
        with pytest.raises(ValueError, match=key):
            validate_config(c)
    # disable_cross_layer False and a null dim_bottleneck are the defaults and are accepted
    assert validate_config(npc_config(disable_cross_layer=False, dim_bottleneck=None))["n_blocks"] == 4


def test_checkpoint_reader_and_refusals(tmp_path):
    from s3prl_b200.upstream.npc import fabricate_npc_state_dict, load_npc_checkpoint, npc_config, required_keys

    sd = fabricate_npc_state_dict(3)
    path = tmp_path / "npc.ckpt"
    torch.save({"config": npc_config(), "model": sd}, path)
    paras, got = load_npc_checkpoint(str(path))
    assert paras["n_blocks"] == 4 and sorted(got) == sorted(required_keys(paras))
    assert all(torch.equal(got[k], sd[k]) for k in got)
    missing = {k: v for k, v in sd.items() if k != "blocks.2.bn1.running_var"}
    torch.save({"config": npc_config(), "model": missing}, path)
    with pytest.raises(KeyError, match="blocks.2.bn1.running_var"):
        load_npc_checkpoint(str(path))
    torch.save({"model": sd}, path)
    with pytest.raises(ValueError, match="not an NPC checkpoint"):
        load_npc_checkpoint(str(path))


def test_disagreeing_conv_mask_is_refused(tmp_path):
    """A file whose conv_mask leaves weight on a tap its config masks (the masks of mask_size 3 under a config that
    says 5) is refused, naming the block; the library refuses it again at finalize (tests/test_npc_gpu.py)."""
    from s3prl_b200.upstream.npc import fabricate_npc_state_dict, load_npc_checkpoint, npc_config

    sd = fabricate_npc_state_dict(0, npc_config(mask_size=3)["model"]["paras"])
    path = tmp_path / "npc.ckpt"
    torch.save({"config": npc_config(), "model": sd}, path)
    with pytest.raises(ValueError, match="masked_convs.0.conv_mask"):
        load_npc_checkpoint(str(path))
    # a mask wider than the config's only zeroes more weight: the reference computes with it, and so does the model
    sd = fabricate_npc_state_dict(0)
    sd["masked_convs.2.conv_mask"][:, :, 1] = 0
    torch.save({"config": npc_config(), "model": sd}, path)
    assert load_npc_checkpoint(str(path))[0]["n_blocks"] == 4


def test_hub_entries_and_wrapper_counts(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.nn.upstream import S3PRLUpstream
    from s3prl_b200.upstream.npc import NpcExpert, fabricate_npc_state_dict, npc_config

    names = set(hub.options())
    assert {"npc", "npc_360hr", "npc_960hr", "npc_local", "npc_url"} <= names
    for n in ("npc", "npc_360hr", "npc_960hr"):
        e = hub.ENTRIES[n](refresh=True)
        assert isinstance(e, NpcExpert) and e.get_downsample_rates("hidden_states") == 160 and e.num_outputs == 9
    for n in ("npc", "npc_url", "npc_local"):
        with pytest.raises(ValueError, match="remote"):
            hub.ENTRIES[n](ckpt="https://example.org/npc_360hr.ckpt")
    for n in ("npc_local", "npc_url"):
        with pytest.raises(AssertionError):
            hub.ENTRIES[n]()
    variant = npc_config(n_blocks=2, kernel_size=9, mask_size=3)
    sd = fabricate_npc_state_dict(5, variant["model"]["paras"])
    path = tmp_path / "npc.ckpt"
    torch.save({"config": variant, "model": sd}, path)
    for n in ("npc_local", "npc_url", "npc"):
        e = hub.ENTRIES[n](str(path), refresh=True)
        assert e.num_outputs == 5 and torch.equal(e._state_dict_host["masked_convs.1.conv.weight"],
                                                  sd["masked_convs.1.conv.weight"])
    for kw in (dict(hooks=[("self.model", lambda i, o: o)]), dict(feature_selection="hidden_states")):
        with pytest.raises(TypeError):
            hub.ENTRIES["npc"](**kw)
    up = S3PRLUpstream("npc")
    assert up.num_layers == 9 and up.hidden_sizes == [512] * 9 and up.downsample_rates == [160] * 9


@pytest.mark.parametrize("fixture", GOLDENS)
def test_oracle_matches_executed_reference(fixture):
    from s3prl_b200.upstream.npc import fabricate_npc_state_dict, hidden_states_info, npc_config, validate_config

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    config = npc_config(**g["paras"])
    paras = validate_config(config)
    sd = fabricate_npc_state_dict(g["weight_seed"], config["model"]["paras"])
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        gen = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(n, generator=gen) for n in case["lens"]]
        assert tuple(case["names"]) == hidden_states_info(paras["n_blocks"])
        with torch.no_grad():
            hs, _ = NO.npc_forward(wavs, sd, paras)
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            ref = case["sub"][l]
            err = ((sub.double() - ref.double()).norm() / ref.double().norm()).item()
            print(f"{fixture} lens={case['lens']} state {l}: abs max {h.abs().max().item():.3f}, "
                  f"oracle vs reference {err:.2e}")
            assert err < 2e-5, (fixture, l, err)
            assert abs(h.norm().item() / case["norms"][l].item() - 1) < 2e-5


def test_masked_outputs_ignore_the_centre():
    """Masked conv i and feat at frame t do not change when the CMVN'd features within (mask_size - 1) / 2 frames of t
    change: every block's receptive field grows by one frame a side, and masked conv i masks mask_size + 2 (i + 1)
    centred taps, so the band it ignores covers what the blocks before it spread from those frames."""
    from s3prl_b200.upstream.npc import fabricate_npc_state_dict, npc_config, validate_config

    config = npc_config()
    paras = validate_config(config)
    sd = fabricate_npc_state_dict(1)
    gen = torch.Generator().manual_seed(9)
    x, lens = AO.batch_features([torch.randn(16000, generator=gen)])
    t, r = 50, (paras["mask_size"] - 1) // 2
    y = x.clone()
    y[:, t - r : t + r + 1] += torch.randn(1, 2 * r + 1, 80, generator=gen)
    with torch.no_grad():
        a, _ = NO.npc_forward(None, sd, paras, feats=(x, lens))
        b, _ = NO.npc_forward(None, sd, paras, feats=(y, lens))
    n = paras["n_blocks"]
    for i in range(n):
        assert (a[2 * i][:, t] - b[2 * i][:, t]).abs().max() > 1e-3  # the blocks do see the change
        assert torch.allclose(a[2 * i + 1][:, t], b[2 * i + 1][:, t], rtol=0, atol=1e-12), i
        assert (a[2 * i + 1][:, t + r + i + 2] - b[2 * i + 1][:, t + r + i + 2]).abs().max() > 1e-6
    assert torch.allclose(a[2 * n][:, t], b[2 * n][:, t], rtol=0, atol=1e-12)
