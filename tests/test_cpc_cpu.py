"""CPU tests of modified CPC (``modified_cpc``): the C ABI's configuration checks and frame rule, the fabricated
checkpoint against the reference's ``CPCModel(...).state_dict()``, the config and checkpoint refusals, the hub entries,
``S3PRLUpstream``'s counts, the fp64 CPU oracle against the executed-reference goldens (tools/make_cpc_golden.py) and
the padding property of the oracle. None of them needs a GPU."""
import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import cpc_oracle as CO  # noqa: E402

GOLDENS = ("cpc_ref", "cpc_ref_c2", "cpc_ref_variant")


def _reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()


def _create(s3b_lib, **over):
    from s3prl_b200 import lib

    c = lib.S3BCpcConfig(hidden=256, num_layers=1)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_cpc_model_create(C.byref(c), C.byref(h))
    return rc, s3b_lib.s3b_last_error().decode(), h


def test_config_accepts_and_refuses(s3b_lib):
    from s3prl_b200 import lib

    assert C.sizeof(lib.S3BCpcConfig) == 7 * 4
    for n in (1, 2, 8):
        rc, msg, h = _create(s3b_lib, num_layers=n)
        assert rc == 0, msg
        assert s3b_lib.s3b_num_outputs(h) == 2
        s3b_lib.s3b_model_destroy(h)
    for over, want in ((dict(num_layers=0), "num_layers"), (dict(num_layers=9), "num_layers"),
                       (dict(hidden=512), "hidden"), (dict(struct_size=12), "struct_size")):
        rc, msg, _ = _create(s3b_lib, **over)
        assert rc != 0 and want in msg, (over, msg)
    c = lib.S3BCpcConfig(hidden=256, num_layers=1)
    c.reserved[2] = 1
    h = C.c_void_p()
    assert s3b_lib.s3b_cpc_model_create(C.byref(c), C.byref(h)) != 0
    assert "reserved" in s3b_lib.s3b_last_error().decode()


def _conv_chain(n: int) -> int:
    """The output length of torch's Conv1d chain, from torch itself (shape inference on the meta device)."""
    x = torch.empty(1, 1, n, device="meta")
    for s, p in zip(CO.STRIDES, CO.PADDINGS):
        if x.shape[-1] + 2 * p < 2 * s:
            return 0
        w = torch.empty(1, x.shape[1], 2 * s, device="meta")
        x = torch.nn.functional.conv1d(x, w, stride=s, padding=p)
    return x.shape[-1]


def test_frame_rule(s3b_lib):
    from s3prl_b200.upstream.cpc import num_frames

    rc, msg, h = _create(s3b_lib)
    assert rc == 0, msg
    try:
        # the table checked against the reference on CPU: 158 samples raise there, 159 give one frame
        for n, want in ((158, 0), (159, 1), (318, 1), (319, 2), (16000, 100), (160000, 1000), (160159, 1001)):
            assert num_frames(n) == want == _conv_chain(n), n
            assert s3b_lib.s3b_num_frames(h, n) == (want if want > 0 else -1), n
        # every residue of L mod 160, at two magnitudes
        for base in (16000, 160000):
            for n in range(base, base + 160):
                assert s3b_lib.s3b_num_frames(h, n) == num_frames(n) == _conv_chain(n), n
        # individual utterances may be shorter than one frame: the reference pads them to the longest
        lens = [16000, 12345, 100]
        out = (C.c_int32 * 3)()
        assert s3b_lib.s3b_valid_frames(h, (C.c_int64 * 3)(*lens), 3, 16000, out) == 0
        assert list(out) == [100, num_frames(12345), 0]
        assert s3b_lib.s3b_valid_frames(h, (C.c_int64 * 1)(158), 1, 158, out) != 0
        assert "conv stack" in s3b_lib.s3b_last_error().decode()
    finally:
        s3b_lib.s3b_model_destroy(h)


@pytest.mark.parametrize("levels", [1, 2])
def test_fabricated_keys_match_the_reference_model(levels):
    _reference()
    from s3prl.upstream.cpc.model import CPCAR, CPCEncoder, CPCModel

    from s3prl_b200.upstream.cpc import fabricate_cpc_state_dict, required_keys

    ref = CPCModel(CPCEncoder(256, "layerNorm"), CPCAR(256, 256, False, levels, "LSTM")).state_dict()
    sd = fabricate_cpc_state_dict(0, levels)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.items()}
    assert sorted(required_keys(levels)) == sorted(ref)
    if levels == 1:
        assert sum(v.numel() for v in ref.values()) == 1843456


def test_config_validation_and_refusals():
    from s3prl_b200.upstream.cpc import cpc_config, validate_config

    assert validate_config(cpc_config()) == {"num_layers": 1}
    assert validate_config(cpc_config(nLevelsGRU=8, cpc_mode="none"))["num_layers"] == 8
    # training-only fields are ignored, whatever their value
    assert validate_config(cpc_config(nPredicts=3, rnnMode="linear", negativeSamplingExt=16, samplingType="uniform"))
    # a partial config is overlaid on the defaults, as loadArgs does
    assert validate_config({"nLevelsGRU": 2}) == {"num_layers": 2}
    for over, want in ((dict(encoder_type="mfcc"), "encoder_type"), (dict(encoder_type="lfb"), "encoder_type"),
                       (dict(normMode="batchNorm"), "normMode"), (dict(normMode="instanceNorm"), "normMode"),
                       (dict(normMode="ID"), "normMode"), (dict(hiddenEncoder=512), "hiddenEncoder"),
                       (dict(hiddenGar=512), "hiddenGar"), (dict(arMode="GRU"), "arMode"),
                       (dict(arMode="transformer"), "arMode"), (dict(arMode="no_ar"), "arMode"),
                       (dict(arMode="RNN"), "arMode"), (dict(nLevelsGRU=0), "nLevelsGRU"),
                       (dict(nLevelsGRU=9), "nLevelsGRU"), (dict(nLevelsGRU=True), "nLevelsGRU"),
                       (dict(cpc_mode="reverse"), "cpc_mode"), (dict(samplingType="sequential"), "samplingType")):
        with pytest.raises(ValueError, match=want):
            validate_config(cpc_config(**over))
    with pytest.raises(ValueError, match="config"):
        validate_config(["not", "a", "dict"])


def test_checkpoint_reader_and_refusals(tmp_path):
    from s3prl_b200.upstream.cpc import cpc_config, fabricate_cpc_state_dict, load_cpc_checkpoint, required_keys

    sd = fabricate_cpc_state_dict(3, 2)
    path = tmp_path / "cpc.pt"
    torch.save({"config": cpc_config(nLevelsGRU=2), "weights": sd, "best": None}, path)
    cfg, got = load_cpc_checkpoint(str(path))
    assert cfg == {"num_layers": 2} and sorted(got) == sorted(required_keys(2))
    assert all(torch.equal(got[k], sd[k]) for k in got)
    for key in ("gEncoder.batchNorm3.bias", "gAR.baseNet.weight_hh_l1"):
        torch.save({"config": cpc_config(nLevelsGRU=2), "weights": {k: v for k, v in sd.items() if k != key}}, path)
        with pytest.raises(KeyError, match=key.replace(".", r"\.")):
            load_cpc_checkpoint(str(path))
    torch.save({"weights": sd}, path)
    with pytest.raises(ValueError, match="not a CPC checkpoint"):
        load_cpc_checkpoint(str(path))
    torch.save({"config": cpc_config(arMode="GRU"), "weights": sd}, path)
    with pytest.raises(ValueError, match="arMode"):
        load_cpc_checkpoint(str(path))


def test_hub_entries_and_wrapper_counts(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.nn.upstream import S3PRLUpstream
    from s3prl_b200.upstream.cpc import CpcExpert, cpc_config, fabricate_cpc_state_dict

    assert {"modified_cpc", "cpc_local", "cpc_url"} <= set(hub.options())
    e = hub.ENTRIES["modified_cpc"](refresh=True)
    assert isinstance(e, CpcExpert) and e.get_downsample_rates("hidden_states") == 160 and e.num_outputs == 2
    assert e.num_frames(16000) == 100
    for n in ("modified_cpc", "cpc_url", "cpc_local"):
        with pytest.raises(ValueError, match="remote"):
            hub.ENTRIES[n](ckpt="https://dl.fbaipublicfiles.com/librilight/CPC_checkpoints/60k_epoch4-d0f474de.pt")
    for n in ("cpc_local", "cpc_url"):
        with pytest.raises(AssertionError):
            hub.ENTRIES[n]()
    sd = fabricate_cpc_state_dict(5, 2)
    path = tmp_path / "cpc.pt"
    torch.save({"config": cpc_config(nLevelsGRU=2), "weights": sd}, path)
    for n in ("cpc_local", "cpc_url", "modified_cpc"):
        e = hub.ENTRIES[n](str(path), refresh=True)
        assert e.cfg["num_layers"] == 2 and torch.equal(e._state_dict_host["gAR.baseNet.weight_ih_l1"],
                                                        sd["gAR.baseNet.weight_ih_l1"])
    for kw in (dict(hooks=[("self.model", lambda i, o: o)]), dict(feature_selection="hidden_states")):
        with pytest.raises(TypeError):
            hub.ENTRIES["modified_cpc"](**kw)
    # randomize: fresh weights of the same shape
    r = CpcExpert(randomize_seed=7)
    assert not torch.equal(r._state_dict_host["gEncoder.conv1.weight"], fabricate_cpc_state_dict(0)["gEncoder.conv1.weight"])
    up = S3PRLUpstream("modified_cpc")
    assert up.num_layers == 2 and up.hidden_sizes == [256] * 2 and up.downsample_rates == [160] * 2


def test_expert_refuses_a_batch_without_a_frame():
    from s3prl_b200.upstream.cpc import CpcExpert

    e = CpcExpert()
    with pytest.raises(ValueError, match="159 samples"):
        e._batch([torch.zeros(158), torch.zeros(40)])
    assert e._batch([torch.zeros(159), torch.zeros(40)]) == ([159, 40], 159, 1)


@pytest.mark.parametrize("fixture", GOLDENS)
def test_oracle_matches_executed_reference(fixture):
    from s3prl_b200.upstream.cpc import HIDDEN_STATES_INFO, cpc_config, fabricate_cpc_state_dict, validate_config

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    n = validate_config(cpc_config(**g["config"]))["num_layers"]
    sd = fabricate_cpc_state_dict(g["weight_seed"], n)
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        gen = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(m, generator=gen) * case["wav_scale"] for m in case["lens"]]
        assert tuple(case["names"]) == HIDDEN_STATES_INFO
        with torch.no_grad():
            hs = CO.forward(wavs, sd, n)
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            ref = case["sub"][l]
            err = ((sub - ref.double()).norm() / ref.double().norm()).item()
            print(f"{fixture} lens={case['lens']} state {l}: abs max {h.abs().max().item():.3f}, "
                  f"oracle vs reference {err:.2e}")
            assert err < 2e-5, (fixture, l, err)
            assert abs(h.norm().item() / case["norms"][l].item() - 1) < 2e-5


def test_only_the_last_frame_depends_on_the_padded_length():
    """Padding an utterance further changes only its frame T(L_b) - 1 (and adds frames after it), in both hidden
    states: frames t < T(L_b) - 1 read no padding sample beyond the utterance's own, and no state that did."""
    from s3prl_b200.upstream.cpc import fabricate_cpc_state_dict, num_frames

    sd = fabricate_cpc_state_dict(2)
    gen = torch.Generator().manual_seed(11)
    changed = 0
    for L in range(4000, 4160, 23):
        w = torch.randn(L, generator=gen) * 0.1
        T = num_frames(L)
        with torch.no_grad():
            a = CO.forward([w], sd, 1)
            b = CO.forward([w], sd, 1, max_len=L + 800)
        for l in range(2):
            # equal up to fp64 rounding (a longer input can take a differently blocked convolution)
            assert (a[l][:, : T - 1] - b[l][:, : T - 1]).abs().max() < 1e-10, (L, l)
        changed += int((a[0][:, T - 1] - b[0][:, T - 1]).abs().max() > 1e-6)
    assert changed > 0  # the last frame usually does see the padding
