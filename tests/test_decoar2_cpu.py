"""CPU tests of DeCoAR 2.0 (``decoar2``): the C ABI's configuration checks for ``frontend = 1``, the frame rules against
the reference's own FeatureExtractor, the fabricated checkpoint against ``Decoar2().state_dict()``, the hub entries and
checkpoint reading, the CPU oracle against the executed-reference goldens (tools/make_decoar2_golden.py), and the fbank
kernels' register use. None of them needs a GPU."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))


def _reference():
    """The reference package, or a skip when it is not installed here."""
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()


def _create(s3b_lib, **over):
    from s3prl_b200.upstream.decoar2 import DECOAR2
    from s3prl_b200.upstream.expert import _c_config

    c = _c_config(DECOAR2)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_model_create(C.byref(c), C.byref(h))
    msg = s3b_lib.s3b_last_error().decode()
    return rc, msg, h


def test_config_accepts_and_refuses(s3b_lib):
    from s3prl_b200 import lib
    from s3prl_b200.upstream.decoar2 import DECOAR2
    from s3prl_b200.upstream.expert import _c_config

    assert C.sizeof(lib.S3BConfig) == 23 * 4  # `frontend` comes out of `reserved`
    assert _c_config(DECOAR2).frontend == 1 and list(_c_config(DECOAR2).reserved) == [0, 0]
    rc, msg, h = _create(s3b_lib)
    assert rc == 0, msg
    s3b_lib.s3b_model_destroy(h)
    for over, want in ((dict(frontend=2), "frontend must be 0"),
                       (dict(family=0), "wav2vec2 family"), (dict(family=2), "wav2vec2 family"),
                       (dict(family=3, no_feature_layer_norm=1), "wav2vec2 family"),
                       (dict(conformer=1, depthwise_kernel=31), "Conformer"),
                       (dict(pos_conv_depth=5, pos_conv_kernel=95), "pos_conv_depth"),
                       (dict(extractor_layer_norm=1), "no conv stack"), (dict(conv_bias=1), "no conv stack"),
                       (dict(normalize_wav=1), "no conv stack")):
        rc, msg, _ = _create(s3b_lib, **over)
        assert rc != 0 and want in msg, (over, msg)
    # no_feature_layer_norm alone is refused by the distiller pairing rule first, with the frontend rule behind it
    rc, msg, _ = _create(s3b_lib, no_feature_layer_norm=1)
    assert rc != 0


def _native_frames(s3b_lib, lens, max_len=None):
    rc, msg, h = _create(s3b_lib)
    assert rc == 0, msg
    try:
        T = s3b_lib.s3b_num_frames(h, max_len or max(lens))
        out = (C.c_int32 * len(lens))()
        rc = s3b_lib.s3b_valid_frames(h, (C.c_int64 * len(lens))(*lens), len(lens), max_len or max(lens), out)
        return T, (list(out) if rc == 0 else s3b_lib.s3b_last_error().decode())
    finally:
        s3b_lib.s3b_model_destroy(h)


def test_frame_rules_closed_form(s3b_lib):
    from s3prl_b200.upstream.decoar2 import num_frames

    rc, msg, h = _create(s3b_lib)
    assert rc == 0, msg
    try:
        for n in list(range(300, 4001)) + [16000, 100003, 160000, 320000, 4_800_001]:
            m = 0 if n < 400 else 1 + (n - 400) // 160
            assert num_frames(n) == (m + 1) // 2, n
            assert s3b_lib.s3b_num_frames(h, n) == (num_frames(n) if n >= 400 else -1), n
    finally:
        s3b_lib.s3b_model_destroy(h)
    assert s3b_lib.s3b_num_frames(None, 16000) == 49  # NULL model: the conv stack's rule, unchanged
    assert _native_frames(s3b_lib, [16000, 12345, 800, 560]) == (49, [49, 38, 2, 1])
    _, msg = _native_frames(s3b_lib, [16000, 559])
    assert "560" in msg


def test_frame_rules_match_reference(s3b_lib):
    """len(FeatureExtractor()(wav)) of the reference over every length 400..4000 and a few long ones."""
    _reference()
    from s3prl.upstream.decoar2.audio import FeatureExtractor

    from s3prl_b200.upstream.decoar2 import num_frames

    fe = FeatureExtractor()
    g = torch.Generator().manual_seed(0)
    base = torch.randn(400_000, generator=g)
    for n in list(range(400, 4001)) + [16000, 100003, 160000, 399_999]:
        with torch.no_grad():
            got = len(fe(base[:n].unsqueeze(0)))
        assert num_frames(n) == got, n
        if n >= 560:
            T, valid = _native_frames(s3b_lib, [n, 560], max_len=n)
            assert T == got and valid[0] == got, n


def test_fabricated_checkpoint_matches_reference_model():
    _reference()
    from s3prl.upstream.decoar2.decoar2 import Decoar2

    from s3prl_b200.upstream.decoar2 import fabricate_decoar2_state_dict

    ref = Decoar2().state_dict()
    sd = fabricate_decoar2_state_dict(0)
    assert sd.keys() == ref.keys()
    assert all(tuple(sd[k].shape) == tuple(ref[k].shape) for k in sd)
    assert torch.equal(fabricate_decoar2_state_dict(0)["post_extract_proj.weight"], sd["post_extract_proj.weight"])
    assert not torch.equal(fabricate_decoar2_state_dict(1)["post_extract_proj.weight"], sd["post_extract_proj.weight"])


def test_hub_entries_and_checkpoints(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.nn.upstream import S3PRLUpstream
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.decoar2 import DECOAR2, Decoar2Expert, fabricate_decoar2_state_dict

    names = set(hub.options())
    for n in ("decoar2", "decoar2_local", "decoar2_url", "decoar2_custom"):
        assert n in names
    assert "decoar2" not in ARCHS and DECOAR2.frontend == "fbank" and ARCHS["wav2vec2_base_960"].frontend == "conv"
    url = "https://huggingface.co/s3prl/converted_ckpts/resolve/main/checkpoint_decoar2.pt"
    for n in ("decoar2", "decoar2_local", "decoar2_url", "decoar2_custom"):
        with pytest.raises(ValueError, match="not reachable"):
            hub.ENTRIES[n](ckpt=url)
    e = hub.ENTRIES["decoar2"](feature_selection="c", upstream_feature_normalize=True)  # swallowed, as the reference
    assert isinstance(e, Decoar2Expert) and (e.num_layers, e.hidden_size) == (12, 768)
    assert e.get_downsample_rates("hidden_states") == 320
    sd = fabricate_decoar2_state_dict(0)
    path = tmp_path / "decoar2.pt"
    torch.save({"model": dict(sd, **{"extra.unused": torch.zeros(3)})}, path)
    for n in ("decoar2_local", "decoar2_url", "decoar2_custom"):
        loaded = hub.ENTRIES[n](str(path), refresh=True)._state_dict_host
        assert loaded.keys() == sd.keys() and all(torch.equal(loaded[k], sd[k]) for k in sd)
    assert hub.ENTRIES["decoar2"](ckpt=str(path))._state_dict_host.keys() == sd.keys()
    del sd["encoder.layers.3.fc1.bias"]
    torch.save({"model": sd}, path)
    with pytest.raises(KeyError, match="encoder.layers.3.fc1.bias"):
        hub.ENTRIES["decoar2_local"](str(path))
    torch.save(sd, path)
    with pytest.raises(ValueError, match="'model'"):
        hub.ENTRIES["decoar2_local"](str(path))
    up = S3PRLUpstream("decoar2", randomize=True)
    assert (up.num_layers, up.hidden_sizes, up.downsample_rates) == (13, [768] * 13, [320] * 13)
    torch.manual_seed(0)
    a = S3PRLUpstream("decoar2", randomize=True).upstream._state_dict_host
    assert not torch.equal(a["post_extract_proj.weight"], fabricate_decoar2_state_dict(0)["post_extract_proj.weight"])


def test_short_utterances_are_refused():
    from s3prl_b200.upstream.decoar2 import Decoar2Expert

    e = Decoar2Expert()
    with pytest.raises(ValueError, match="560"):
        e([torch.zeros(16000), torch.zeros(559)])
    with pytest.raises(ValueError, match="560"):
        e.forward_host([torch.zeros(400)])


@pytest.mark.parametrize("fixture", ["decoar2_ref", "decoar2_ref_c2"])
def test_oracle_matches_reference_golden(fixture):
    """tests/decoar2_oracle.py against the executed reference: 2e-5 relative per layer and on the norm."""
    import decoar2_oracle as D

    from s3prl_b200.upstream.decoar2 import fabricate_decoar2_state_dict

    fx = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    sd = fabricate_decoar2_state_dict(fx["weight_seed"])
    cs, ts = fx["channel_stride"], fx["time_stride"]
    worst = 0.0
    for case in fx["cases"]:
        g = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(n, generator=g) for n in case["lens"]]
        with torch.no_grad():
            hs, _pad = D.decoar2_forward(wavs, sd)
        assert len(hs) == case["num_hidden"] == 13 and tuple(hs[0].shape) == tuple(case["shape"])
        assert case["names"] == [f"self.model.encoder.layers[{i}]" for i in range(12)] + ["self.model.encoder"]
        for l, h in enumerate(hs):
            ref = case["sub"][l]
            got = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            rel = ((got.double() - ref.double()).norm() / ref.double().norm()).item()
            worst = max(worst, rel)
            assert rel < 2e-5, (fixture, l, rel)
            assert abs(h.double().norm().item() - case["norms"][l].item()) < 2e-5 * case["norms"][l].item()
    print(f"{fixture}: oracle vs reference, worst per-layer relative error {worst:.3e} (bound 2e-5)")


def test_fbank_kernels_no_spills(tmp_path):
    """ptxas -v on fbank.cu with the library's flags: no kernel spills (the hamming frame kernel and the CMVN /
    decimation kernel among them)."""
    from test_ptxas_cpu import _assert_no_spills, _ptxas_report

    log = _ptxas_report(tmp_path, ROOT / "s3prl_b200" / "csrc" / "fbank.cu")
    assert "decoar2_cmvn_kernel" in log and "fbank_frames_kernelILb1E" in log
    _assert_no_spills(log)
