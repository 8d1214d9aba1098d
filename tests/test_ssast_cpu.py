"""SSAST without a GPU: the fp64 oracle against the executed reference's goldens, the frame-count and window rules,
the re-gridded positional table against the reference's own ASTModel, the loader's refusals, the fabricated file in
the reference, the C ABI's bookkeeping and refusals, and the hub entries."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import ssast_oracle as SO  # noqa: E402

GOLDENS = ("ssast_frame", "ssast_patch", "ssast_frame_w10", "ssast_patch_w10")


def _reference():
    sys.path.insert(0, str(ROOT / "oracle"))
    import ref_runtime
    import timm_shim

    if ref_runtime.reference_root() is None:
        pytest.skip("the reference (s3prl) is not available")
    ref_runtime.activate()
    timm_shim.install()


def _wavs(lens, seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) * scale for n in lens]


@pytest.mark.parametrize("fixture", GOLDENS)
def test_oracle_matches_executed_reference(fixture):
    from s3prl_b200.upstream.ssast import fabricate_ssast_state_dict, prepare_ssast_tensors

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    kind, win = g["kind"], g["window_secs"]
    sd = prepare_ssast_tensors(fabricate_ssast_state_dict(g["weight_seed"], kind), kind, win)
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        with torch.no_grad():
            hs = SO.ssast_forward(_wavs(case["lens"], case["wav_seed"], case["wav_scale"]), sd, kind, win)
        assert len(hs) == case["num_hidden"] == 12 and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            s = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            ref = case["sub"][l].double()
            err = ((s - ref).norm() / ref.norm()).item()
            print(f"{fixture} lens={case['lens']} state {l}: abs max {h.abs().max().item():.3f}, oracle vs reference "
                  f"{err:.2e} (timm shim: {g['timm_shim']})")
            assert err < 2e-5, (fixture, l, err)
            assert abs(h.norm().item() / case["norms"][l].item() - 1) < 2e-5


def _reference_frames(kind, window_secs, max_len):
    """The reference expert's output length: its windows' time patches, then h[:, :len(range(0, max_len, rate))]."""
    S = int(window_secs * 16000)
    tl = int(window_secs * 16000 / 160)
    nseg = len(list(range(0, max_len, S)))
    t_dim = tl - 1 if kind == "frame" else (tl - 16) // 10 + 1
    return min(nseg * t_dim, len(range(0, max_len, 160 if kind == "frame" else 1600)))


@pytest.mark.parametrize("kind", ["frame", "patch"])
@pytest.mark.parametrize("window_secs", [1.0, 10.0])
def test_frame_and_segment_rules(s3b_lib, kind, window_secs):
    from s3prl_b200 import lib
    from s3prl_b200.upstream.ssast import geometry, num_frames, num_segments

    g = geometry(kind, window_secs)
    h = C.c_void_p()
    cfg = lib.S3BSsastConfig(patch=int(kind == "patch"), window_samples=g["S"], embed_dim=768, num_heads=12, num_layers=12)
    lib.check(s3b_lib.s3b_ssast_model_create(C.byref(cfg), C.byref(h)))
    try:
        assert s3b_lib.s3b_num_outputs(h) == 12
        for L in (1, 2, 159, 160, 161, 1599, 1600, 1601, 15999, 16000, 16001, 40000, 159999, 160000, 160001, 480000):
            T = _reference_frames(kind, window_secs, L)
            assert num_frames(kind, window_secs, L) == T == s3b_lib.s3b_num_frames(h, L), (L, T)
            assert num_segments(g["S"], L) == -(-L // g["S"])
        lens = [1, 15999, 16000, 16001, 9000]
        valid = (C.c_int32 * len(lens))()
        lib.check(s3b_lib.s3b_valid_frames(h, (C.c_int64 * len(lens))(*lens), len(lens), 16001, valid))
        T = _reference_frames(kind, window_secs, 16001)
        assert list(valid) == [min(T, -(-n // g["rate"])) for n in lens]
    finally:
        s3b_lib.s3b_model_destroy(h)
    # the goldens' shapes follow the same rule
    for fixture in GOLDENS:
        gd = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
        for case in gd["cases"]:
            f_dim = 12 if gd["kind"] == "patch" else 1
            assert tuple(case["shape"]) == (len(case["lens"]), _reference_frames(gd["kind"], gd["window_secs"],
                                                                                  max(case["lens"])), 768 * f_dim)


@pytest.mark.parametrize("kind", ["frame", "patch"])
@pytest.mark.parametrize("window_secs", [1.0, 10.0])
def test_pos_embed_regrid_equals_reference(tmp_path, kind, window_secs):
    """1 s: the time crop (t_dim < p_t_dim) for both models; 10 s: the (8, t_dim) interpolation (t_dim > p_t_dim).
    The fabricated file loads into the reference's ASTModel, whose fine-tuning constructor re-grids its table."""
    _reference()
    from s3prl.upstream.ssast.ast_models import ASTModel

    from s3prl_b200.upstream.ssast import KINDS, fabricate_ssast_state_dict, geometry, prepare_ssast_tensors

    sd = fabricate_ssast_state_dict(4, kind)
    path = tmp_path / "ssast.pth"
    torch.save(sd, path)
    (fs, ts), (fst, tst) = KINDS[kind]
    g = geometry(kind, window_secs)
    crop = g["t_dim"] < (1024 - ts) // ts + 1
    assert crop == (window_secs == 1.0)
    model = ASTModel(fshape=fs, tshape=ts, fstride=fst, tstride=tst, input_fdim=128, input_tdim=g["TL"],
                     model_size="base", pretrain_stage=False, load_pretrained_mdl_path=str(path))
    ours = prepare_ssast_tensors(sd, kind, window_secs)
    assert ours["pos_embed"].shape == model.v.pos_embed.shape == (1, 2 + g["P"], 768)
    assert torch.equal(ours["pos_embed"], model.v.pos_embed.detach())
    ref = model.v.state_dict()
    for k, t in ours.items():
        if k != "pos_embed":
            assert torch.equal(t, ref[k]), k


@pytest.mark.parametrize("kind", ["frame", "patch"])
def test_fabricated_file_matches_the_reference_pretraining_model(kind):
    """Every fabricated key exists in the reference's pretraining ASTModel (DataParallel) with the same shape, and the
    model has no key the file lacks: the file is a complete pretraining checkpoint of the believed format."""
    _reference()
    from s3prl.upstream.ssast.ast_models import ASTModel

    from s3prl_b200.upstream.ssast import KINDS, fabricate_ssast_state_dict

    (fs, ts), _ = KINDS[kind]
    ref = torch.nn.DataParallel(ASTModel(fshape=fs, tshape=ts, fstride=fs, tstride=ts, input_fdim=128, input_tdim=1024,
                                         model_size="base", pretrain_stage=True)).state_dict()
    sd = fabricate_ssast_state_dict(0, kind)
    assert set(sd) == set(ref)
    for k, t in sd.items():
        assert tuple(t.shape) == tuple(ref[k].shape), k


def test_loader_refusals_name_the_field(tmp_path):
    from s3prl_b200 import hub
    from s3prl_b200.upstream.ssast import SsastExpert, fabricate_ssast_state_dict

    def save(sd, name="x.pth"):
        p = tmp_path / name
        torch.save(sd, p)
        return str(p)

    sd = fabricate_ssast_state_dict(1, "frame")
    bad = dict(sd)
    del bad["module.v.blocks.7.mlp.fc2.bias"]
    with pytest.raises(KeyError, match="module.v.blocks.7.mlp.fc2.bias"):
        SsastExpert(ckpt=save(bad), kind="frame")
    with pytest.raises(ValueError, match="patch_embed.proj.weight"):
        SsastExpert(ckpt=save(sd), kind="patch")  # a frame checkpoint for the patch model
    bad = dict(sd, **{"module.v.patch_embed.proj.weight": torch.zeros(768, 1, 8, 8)})
    with pytest.raises(ValueError, match="patch_embed.proj.weight"):
        SsastExpert(ckpt=save(bad), kind="frame")
    bad = dict(sd, **{"module.v.cls_token": torch.zeros(1, 1, 384)})
    with pytest.raises(ValueError, match="cls_token"):
        SsastExpert(ckpt=save(bad), kind="frame")
    bad = dict(sd, **{"module.p_input_tdim": torch.tensor(512)})
    with pytest.raises(ValueError, match="p_input_tdim"):
        SsastExpert(ckpt=save(bad), kind="frame")
    with pytest.raises(ValueError, match="window_secs"):
        SsastExpert(kind="patch", window_secs=0.15)  # 15 frames: no 16-frame patch
    with pytest.raises(ValueError, match="window_secs"):
        SsastExpert(kind="frame", window_secs=0.02)  # shorter than one 25 ms frame
    with pytest.raises(ValueError, match="window_secs"):
        SsastExpert(kind="frame", window_secs=12.0)
    with pytest.raises(ValueError, match="not an SSAST checkpoint"):
        SsastExpert(ckpt=save({"model": {}}), kind="frame")
    with pytest.raises(ValueError, match="remote checkpoints"):
        hub.ssast_frame_base(ckpt="https://www.dropbox.com/s/nx6nl4d4bl71sm8/SSAST-Base-Frame-400.pth?dl=1")
    # a local file is read; the ignored heads may be absent
    keep = {k: v for k, v in sd.items() if "predlayer" not in k and "head" not in k and k != "module.mask_embed"}
    e = hub.ssast_frame_base(save(keep, "local.pth"), window_secs=10.0, refresh=True)
    assert e.num_frames(160000) == 999 and e.hidden_size == 768


def test_hub_entries():
    from s3prl_b200 import hub
    from s3prl_b200.upstream.ssast import SsastExpert

    assert {"ssast_frame_base", "ssast_patch_base"} <= set(hub.options())
    for name, width, rate, T in (("ssast_frame_base", 768, 160, 99), ("ssast_patch_base", 12 * 768, 1600, 9)):
        e = hub.ENTRIES[name](refresh=True)
        assert isinstance(e, SsastExpert) and e.hidden_size == width and e.num_outputs == 12
        assert e.get_downsample_rates("hidden_states") == rate and e.num_frames(16000) == T
        e10 = hub.ENTRIES[name](window_secs=10)
        assert e10.num_frames(160000) == (999 if width == 768 else 99)


def _create(s3b_lib, **over):
    from s3prl_b200 import lib

    c = lib.S3BSsastConfig(patch=0, window_samples=16000, embed_dim=768, num_heads=12, num_layers=12)
    for k, v in over.items():
        setattr(c, k, v)
    h = C.c_void_p()
    rc = s3b_lib.s3b_ssast_model_create(C.byref(c), C.byref(h))
    if rc == 0:
        s3b_lib.s3b_model_destroy(h)
    return rc, s3b_lib.s3b_last_error().decode()


def test_c_abi_refusals(s3b_lib):
    for over in (dict(), dict(patch=1), dict(window_samples=400), dict(patch=1, window_samples=2560),
                 dict(window_samples=160000)):
        assert _create(s3b_lib, **over)[0] == 0, over
    for over, msg in ((dict(patch=2), "patch must be"), (dict(embed_dim=384), "base is served"),
                      (dict(num_layers=6), "base is served"), (dict(window_samples=399), "window_samples"),
                      (dict(patch=1, window_samples=2559), "window_samples"), (dict(window_samples=160001), "window_samples"),
                      (dict(struct_size=8), "struct_size")):
        rc, err = _create(s3b_lib, **over)
        assert rc != 0 and msg in err, (over, err)
