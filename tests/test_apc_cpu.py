"""CPU tests of APC / VQ-APC (``apc``, ``vq_apc``): the C ABI's configuration checks and frame rules, the fabricated
checkpoint against the reference's ``APC(...).state_dict()``, the checkpoint reader's refusals, the hub entries, the
CPU oracle against the executed-reference goldens (tools/make_apc_golden.py), the long memory of the fabricated
weights, and the recurrence kernel's compile-time budget. None of them needs a GPU."""
import ctypes as C
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import apc_oracle as AO  # noqa: E402

GOLDENS = ("apc_ref", "apc_ref_c2", "vq_apc_ref")


def _reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()


def _create(s3b_lib, **over):
    from s3prl_b200 import lib

    c = lib.S3BApcConfig(num_layers=3, hidden=512, residual=1)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_apc_model_create(C.byref(c), C.byref(h))
    return rc, s3b_lib.s3b_last_error().decode(), h


def test_config_accepts_and_refuses(s3b_lib):
    from s3prl_b200 import lib

    assert C.sizeof(lib.S3BApcConfig) == 8 * 4
    for residual in (0, 1):
        rc, msg, h = _create(s3b_lib, residual=residual)
        assert rc == 0, msg
        assert s3b_lib.s3b_num_outputs(h) == 3
        s3b_lib.s3b_model_destroy(h)
    for over, want in ((dict(num_layers=2), "num_layers"), (dict(num_layers=4), "num_layers"),
                       (dict(hidden=256), "hidden"), (dict(residual=2), "residual"),
                       (dict(struct_size=12), "struct_size")):
        rc, msg, _ = _create(s3b_lib, **over)
        assert rc != 0 and want in msg, (over, msg)
    c = lib.S3BApcConfig(num_layers=3, hidden=512, residual=1)
    c.reserved[2] = 1
    h = C.c_void_p()
    assert s3b_lib.s3b_apc_model_create(C.byref(c), C.byref(h)) != 0
    assert "reserved" in s3b_lib.s3b_last_error().decode()


def test_frame_rules(s3b_lib):
    from s3prl_b200.upstream.apc import num_frames

    rc, msg, h = _create(s3b_lib)
    assert rc == 0, msg
    try:
        for n in (400, 559, 560, 16000, 160000, 100003):
            assert s3b_lib.s3b_num_frames(h, n) == num_frames(n) == 1 + (n - 400) // 160
        assert s3b_lib.s3b_num_frames(h, 399) == -1
        lens = [16000, 12345, 560]
        out = (C.c_int32 * 3)()
        assert s3b_lib.s3b_valid_frames(h, (C.c_int64 * 3)(*lens), 3, 16000, out) == 0
        assert list(out) == [num_frames(n) for n in lens] == [98, 75, 2]
        assert s3b_lib.s3b_valid_frames(h, (C.c_int64 * 2)(16000, 559), 2, 16000, out) != 0
        assert "560" in s3b_lib.s3b_last_error().decode()
    finally:
        s3b_lib.s3b_model_destroy(h)


@pytest.mark.parametrize("vq", [False, True])
def test_fabricated_keys_match_the_reference_model(vq):
    _reference()
    from s3prl.upstream.apc.apc import APC

    from s3prl_b200.upstream.apc import apc_config, fabricate_apc_state_dict

    ref = APC(80, **apc_config(vq=vq)["model"]["paras"]).state_dict()
    sd = fabricate_apc_state_dict(0, vq)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.items()}
    # apc and vq_apc of one seed share the GRU weights
    plain = fabricate_apc_state_dict(0, False)
    assert all(torch.equal(plain[k], sd[k]) for k in plain if k.startswith("rnn_layers."))


def test_checkpoint_reader_and_refusals(tmp_path):
    from s3prl_b200.upstream.apc import apc_config, fabricate_apc_state_dict, load_apc_checkpoint, required_keys

    sd = fabricate_apc_state_dict(3, vq=True)
    path = tmp_path / "vq.ckpt"
    torch.save({"config": apc_config(residual=False, vq=True), "model": sd}, path)
    residual, got = load_apc_checkpoint(str(path))
    assert residual is False and sorted(got) == sorted(required_keys())
    assert all(torch.equal(got[k], sd[k]) for k in got)

    def refused(config, want, model=sd):
        p = tmp_path / "bad.ckpt"
        torch.save({"config": config, "model": model}, p)
        with pytest.raises(ValueError, match=want):
            load_apc_checkpoint(str(p))

    def edit(section, key, value):
        c = apc_config()
        c[section]["audio" if section == "data" else "paras"][key] = value
        return c

    refused(edit("data", "feat_type", "mfcc"), "feat_type")
    refused(edit("data", "feat_dim", 40), "feat_dim")
    refused(edit("data", "cmvn", False), "cmvn")
    refused(edit("data", "frame_shift", 12.5), "frame_shift")
    refused(edit("data", "frame_length", 20), "frame_length")
    refused(edit("data", "dither", 1.0), "dither")
    refused(edit("model", "hidden_size", 256), "hidden_size")
    refused(edit("model", "num_layers", 4), "num_layers")
    refused(edit("model", "bidirectional", True), "bidirectional")
    c = apc_config()
    del c["model"]["paras"]["residual"]
    refused(c, "residual")
    ok = apc_config()
    ok["data"]["audio"].update(frame_length=25.0, frame_shift=10.0, decode_wav=True)
    p = tmp_path / "ok.ckpt"
    torch.save({"config": ok, "model": sd}, p)
    assert load_apc_checkpoint(str(p))[0] is True
    missing = {k: v for k, v in sd.items() if k != "rnn_layers.2.bias_hh_l0"}
    torch.save({"config": apc_config(), "model": missing}, p)
    with pytest.raises(KeyError, match="rnn_layers.2.bias_hh_l0"):
        load_apc_checkpoint(str(p))
    torch.save({"model": sd}, p)
    with pytest.raises(ValueError, match="not an APC checkpoint"):
        load_apc_checkpoint(str(p))


def test_hub_entries(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.apc import ApcExpert, apc_config, fabricate_apc_state_dict

    names = set(hub.options())
    apc = {"apc", "apc_360hr", "apc_960hr", "apc_local", "apc_url", "vq_apc", "vq_apc_360hr", "vq_apc_960hr",
           "vq_apc_url"}
    assert apc <= names and "wav2vec2_conformer_relpos" not in names
    for n in ("apc", "vq_apc_960hr"):
        e = hub.ENTRIES[n](refresh=True)
        assert isinstance(e, ApcExpert) and e.get_downsample_rates("hidden_states") == 160
    for n in ("apc", "apc_url", "vq_apc_url", "apc_local"):
        with pytest.raises(ValueError, match="remote"):
            hub.ENTRIES[n](ckpt="https://example.org/apc_360hr.ckpt")
    sd = fabricate_apc_state_dict(5)
    path = tmp_path / "apc.ckpt"
    torch.save({"config": apc_config(residual=False), "model": sd}, path)
    for n in ("apc_local", "apc_url", "vq_apc_url", "apc"):
        e = hub.ENTRIES[n](str(path), refresh=True)
        assert e.residual is False and torch.equal(e._state_dict_host["rnn_layers.1.weight_hh_l0"],
                                                   sd["rnn_layers.1.weight_hh_l0"])
    for kw in (dict(hooks=[("self.model", lambda i, o: o)]), dict(feature_selection="hidden_states")):
        with pytest.raises(TypeError):
            hub.ENTRIES["apc"](**kw)


@pytest.mark.parametrize("fixture", GOLDENS)
def test_oracle_matches_executed_reference(fixture):
    from s3prl_b200.upstream.apc import HIDDEN_STATES_INFO, fabricate_apc_state_dict

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    sd = fabricate_apc_state_dict(g["weight_seed"], g["vq"])
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        gen = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(n, generator=gen) for n in case["lens"]]
        assert tuple(case["names"]) == HIDDEN_STATES_INFO
        with torch.no_grad():
            hs, _ = AO.apc_forward(wavs, sd, residual=True)
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            ref = case["sub"][l]
            err = ((sub.double() - ref.double()).norm() / ref.double().norm()).item()
            assert err < 2e-5, (fixture, l, err)
            assert abs(h.double().norm().item() / case["norms"][l].item() - 1) < 2e-5


def test_fabricated_weights_have_long_memory():
    """Perturbing the first 10 frames of the features still moves the outputs at frames >= 300 measurably: the
    recurrence carries state over hundreds of steps, so a test of it can see a wrong carry."""
    from s3prl_b200.upstream.apc import fabricate_apc_state_dict

    sd = fabricate_apc_state_dict(0)
    gen = torch.Generator().manual_seed(7)
    wav = torch.randn(16000 * 4, generator=gen)
    x, lens = AO.batch_features([wav])
    y = x.clone()
    y[:, :10] += torch.randn(1, 10, 80, generator=gen)
    with torch.no_grad():
        a, _ = AO.apc_forward(None, sd, feats=(x, lens))
        b, _ = AO.apc_forward(None, sd, feats=(y, lens))
    for l in range(3):
        late = (a[l][:, 300:] - b[l][:, 300:]).abs().max().item()
        assert late > 1e-3, (l, late)
    assert a[2].std().item() > 0.2  # the hidden states are not near zero either


def test_gru_kernel_compile_budget(tmp_path):
    """gru.cu: no register spills, no local-memory stack, and its shared memory within the 227 KB a CTA can opt in to
    (a static_assert in the source, so a compile that passes has checked it)."""
    from s3prl_b200 import build

    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    src = ROOT / "s3prl_b200" / "csrc" / "gru.cu"
    assert "static_assert(sizeof(GruSmem) <= 227 * 1024" in src.read_text()
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas=-v", "-c", str(src), "-o", str(tmp_path / "gru.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    assert any("gru_cluster_kernel" in e for e in entries), r.stderr[-2000:]
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(entries)
    assert all(int(a) == 0 and int(b) == 0 and int(c) == 0 for a, b, c in frames), r.stderr
