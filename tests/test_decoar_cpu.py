"""CPU tests of DeCoAR (``decoar``, ``decoar_layers``): the C ABI's configuration checks and frame rules, the
fabricated checkpoint against the reference's ``Decoar().state_dict()``, the checkpoint reader's refusals, the hub
entries, the CPU oracle against the executed-reference goldens (tools/make_decoar_golden.py), the long memory of the
fabricated weights, and the recurrence kernel's compile-time budget. None of them needs a GPU."""
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
import decoar_oracle as DO  # noqa: E402

GOLDENS = ("decoar_ref", "decoar_layers_ref", "decoar_layers_ref_c2")


def _reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()


def _create(s3b_lib, **over):
    from s3prl_b200 import lib

    c = lib.S3BDecoarConfig(num_layers=4, hidden=1024, all_layers=1)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_decoar_model_create(C.byref(c), C.byref(h))
    return rc, s3b_lib.s3b_last_error().decode(), h


def test_config_accepts_and_refuses(s3b_lib):
    from s3prl_b200 import lib

    assert C.sizeof(lib.S3BDecoarConfig) == 8 * 4
    for all_layers, outputs in ((0, 1), (1, 4)):
        rc, msg, h = _create(s3b_lib, all_layers=all_layers)
        assert rc == 0, msg
        assert s3b_lib.s3b_num_outputs(h) == outputs
        assert s3b_lib.s3b_default_lanes(h, 32, 160000) == 1  # one lane at any batch size
        s3b_lib.s3b_model_destroy(h)
    for over, want in ((dict(num_layers=3), "num_layers"), (dict(hidden=512), "hidden"),
                       (dict(all_layers=2), "all_layers"), (dict(struct_size=12), "struct_size")):
        rc, msg, _ = _create(s3b_lib, **over)
        assert rc != 0 and want in msg, (over, msg)
    c = lib.S3BDecoarConfig(num_layers=4, hidden=1024, all_layers=0)
    c.reserved[1] = 1
    h = C.c_void_p()
    assert s3b_lib.s3b_decoar_model_create(C.byref(c), C.byref(h)) != 0
    assert "reserved" in s3b_lib.s3b_last_error().decode()


def test_frame_rules(s3b_lib):
    from s3prl_b200.upstream.decoar import num_frames

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


def test_fabricated_keys_match_the_reference_model():
    _reference()
    from s3prl.upstream.decoar.decoar import Decoar

    from s3prl_b200.upstream.decoar import fabricate_decoar_state_dict, required_keys

    ref = Decoar().state_dict()
    sd = fabricate_decoar_state_dict(0)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.items()}
    assert sorted(required_keys()) == sorted(ref)


def test_checkpoint_reader_and_refusals(tmp_path):
    from s3prl_b200.upstream.decoar import fabricate_decoar_state_dict, load_decoar_checkpoint, required_keys

    sd = fabricate_decoar_state_dict(3)
    path = tmp_path / "decoar.ckpt"
    torch.save({"model": dict(sd, **{"unused.weight": torch.zeros(3)})}, path)  # unknown keys are ignored
    got = load_decoar_checkpoint(str(path))
    assert sorted(got) == sorted(required_keys())
    assert all(torch.equal(got[k], sd[k]) for k in got)
    for gone in ("backward_lstm.weight_hh_l2", "forward_lstm.bias_hh_l3", "post_extract_proj.bias"):
        torch.save({"model": {k: v for k, v in sd.items() if k != gone}}, path)
        with pytest.raises(KeyError, match=re.escape(gone)):
            load_decoar_checkpoint(str(path))
    torch.save(sd, path)
    with pytest.raises(ValueError, match="not a DeCoAR checkpoint"):
        load_decoar_checkpoint(str(path))


def test_hub_entries(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.decoar import DecoarExpert, fabricate_decoar_state_dict

    names = {f"{f}{s}" for f in ("decoar", "decoar_layers") for s in ("", "_local", "_url", "_custom")}
    assert names <= set(hub.options())
    for n in ("decoar", "decoar_layers"):
        e = hub.ENTRIES[n](refresh=True)
        assert isinstance(e, DecoarExpert) and e.get_downsample_rates("hidden_states") == 160
        assert e.all_layers == (n == "decoar_layers") and e.num_outputs == (4 if e.all_layers else 1)
    for n in sorted(names):
        with pytest.raises(ValueError, match="remote"):
            hub.ENTRIES[n](ckpt="https://example.org/checkpoint_decoar.pt")
    sd = fabricate_decoar_state_dict(5)
    path = tmp_path / "decoar.ckpt"
    torch.save({"model": sd}, path)
    for n in sorted(names):
        e = hub.ENTRIES[n](str(path), refresh=True)
        assert e.all_layers == n.startswith("decoar_layers")
        assert torch.equal(e._state_dict_host["backward_lstm.weight_hh_l1"], sd["backward_lstm.weight_hh_l1"])
    for kw in (dict(hooks=[("self.model", lambda i, o: o)]), dict(feature_selection="hidden_states")):
        with pytest.raises(TypeError):
            hub.ENTRIES["decoar"](**kw)


def test_short_utterance_is_refused():
    from s3prl_b200.upstream.decoar import DecoarExpert

    with pytest.raises(ValueError, match="560"):
        DecoarExpert()([torch.zeros(16000), torch.zeros(559)])


@pytest.mark.parametrize("fixture", GOLDENS)
def test_oracle_matches_executed_reference(fixture):
    from s3prl_b200.upstream.decoar import fabricate_decoar_state_dict

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    sd = fabricate_decoar_state_dict(g["weight_seed"])
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        gen = torch.Generator().manual_seed(case["wav_seed"])
        wavs = [torch.randn(n, generator=gen) for n in case["lens"]]
        with torch.no_grad():
            layers, m = DO.decoar_forward(wavs, sd)
        hs = layers if g["all_layers"] else layers[-1:]  # decoar: the concat of the last layer only
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for h in hs:
            for b, mb in enumerate(m):
                assert torch.equal(h[b, mb:], torch.zeros_like(h[b, mb:]))  # padding frames exactly 0
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            ref = case["sub"][l]
            err = ((sub.double() - ref.double()).norm() / ref.double().norm()).item()
            assert err < 2e-5, (fixture, l, err)
            assert abs(h.double().norm().item() / case["norms"][l].item() - 1) < 2e-5


def test_fabricated_weights_have_long_memory():
    """Perturbing the first 50 frames of the features still moves the forward direction's outputs at frames >= 350
    measurably, and perturbing the last 50 moves the backward direction's outputs 300 frames before them."""
    from s3prl_b200.upstream.decoar import fabricate_decoar_state_dict

    sd = fabricate_decoar_state_dict(0)
    gen = torch.Generator().manual_seed(7)
    wav = torch.randn(16000 * 6, generator=gen)
    x, lens = AO.batch_features([wav])
    T = lens[0]
    head, tail = x.clone(), x.clone()
    head[:, :50] += torch.randn(1, 50, 80, generator=gen)
    tail[:, T - 50:] += torch.randn(1, 50, 80, generator=gen)
    with torch.no_grad():
        a, _ = DO.decoar_forward(None, sd, feats=(x, lens))
        b, _ = DO.decoar_forward(None, sd, feats=(head, lens))
        c, _ = DO.decoar_forward(None, sd, feats=(tail, lens))
    for l in range(4):
        fwd = (a[l][:, 350:, :1024] - b[l][:, 350:, :1024]).abs().max().item()
        bwd = (a[l][:, : T - 350, 1024:] - c[l][:, : T - 350, 1024:]).abs().max().item()
        assert fwd > 1e-3 and bwd > 1e-3, (l, fwd, bwd)
    assert a[3].std().item() > 0.2  # the hidden states are not near zero either


def test_lstm_kernel_compile_budget(tmp_path):
    """lstm.cu: no register spills, no local-memory stack, and its shared memory within the 227 KB a CTA can opt in to
    (a static_assert in the source, so a compile that passes has checked it; ptxas reports no static shared memory)."""
    from s3prl_b200 import build

    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    src = ROOT / "s3prl_b200" / "csrc" / "lstm.cu"
    assert "static_assert(sizeof(LstmSmem) <= 227 * 1024" in src.read_text()
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas=-v", "-c", str(src), "-o", str(tmp_path / "lstm.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    entries = re.findall(r"Compiling entry function '([^']+)'", r.stderr)
    assert any("lstm_grid_kernel" in e for e in entries), r.stderr[-2000:]
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) == len(entries)
    assert all(int(a) == 0 and int(b) == 0 and int(c) == 0 for a, b, c in frames), r.stderr
    smem = [int(v) for v in re.findall(r"(\d+) bytes smem", r.stderr)]
    assert all(v <= 227 * 1024 for v in smem), smem
