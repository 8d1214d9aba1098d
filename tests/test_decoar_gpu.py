"""GPU tests of DeCoAR (``decoar``, ``decoar_layers``): the grid-resident LSTM recurrence kernel at block level
(``s3b_lstm_f32``) against an fp64 torch loop in both directions; the whole model against the executed-reference
goldens (tests/golden/decoar*_ref*.pt) in both GEMM operand schemes; ``decoar`` against ``decoar_layers``; the long
memory in both directions; bit-identical results across lanes, ``forward_host`` chunks and shards;
and the refusals. Bounds: recurrence block 1e-4 relative Frobenius and 2e-4 of the output scale elementwise; model
2e-4 relative per hidden state. Every check prints measured / bound."""
import ctypes as C
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import decoar_oracle as DO  # noqa: E402

pytestmark = pytest.mark.gpu

H = 1024
BLOCK_REL = 1e-4
BLOCK_ELEM = 2e-4
REL_TOL = 2e-4


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------
# recurrence block
# ------------------------------------------------------------------------------------------------
def _layer(seed=1, k=1):
    from s3prl_b200.upstream.decoar import fabricate_decoar_state_dict

    sd = fabricate_decoar_state_dict(seed)
    return [(sd[f"{d}_lstm.weight_ih_l{k}"], sd[f"{d}_lstm.weight_hh_l{k}"],
             sd[f"{d}_lstm.bias_ih_l{k}"], sd[f"{d}_lstm.bias_hh_l{k}"]) for d in ("forward", "backward")]


def _lstm_block(s3b_lib, xgs, whhs, bhhs, lens, out_fmt=-1):
    """Both directions into one [B, T, 2H] output (and planes); xgs / whhs / bhhs per direction."""
    from s3prl_b200 import lib

    B, T, _ = xgs[0].shape
    out = torch.full((B, T, 2 * H), float("nan"), device="cuda")
    planes = torch.full((B, T, 2 * H), float("nan"), device="cuda") if out_fmt >= 0 else None
    pl_dir = []
    for d in (0, 1):
        lib.check(s3b_lib.s3b_lstm_f32(
            C.c_void_p(xgs[d].data_ptr()), C.c_void_p(whhs[d].data_ptr()),
            C.c_void_p(bhhs[d].data_ptr()) if bhhs[d] is not None else None, (C.c_int32 * B)(*lens), B, T, d,
            out_fmt, C.c_void_p(out.data_ptr()), C.c_void_p(planes.data_ptr()) if planes is not None else None,
            _stream()))
        if planes is not None:
            pl_dir.append(planes[..., d * H:(d + 1) * H].clone())
    torch.cuda.synchronize()
    return out, (torch.cat(pl_dir, -1) if planes is not None else None)


def _lens(B, T, g):
    base = [T, 1, 2][:B]
    return base + [int(v) for v in torch.randint(1, T + 1, (B - len(base),), generator=g)]


@pytest.mark.parametrize("out_fmt", [-1, 1])
@pytest.mark.parametrize("B,T", [(1, 1), (1, 300), (16, 200), (17, 250), (33, 300)])
def test_lstm_block_matches_fp64(s3b_lib, B, T, out_fmt):
    g = torch.Generator().manual_seed(B * 7919 + T)
    layer = _layer()
    lens = _lens(B, T, g)
    x = torch.randn(B, T, H, generator=g) * 0.5
    # the forward direction gets b_hh folded into xg (as the model does), the backward one through the bhh argument
    xgs = [x @ layer[0][0].T + layer[0][2] + layer[0][3], x @ layer[1][0].T + layer[1][2]]
    out, planes = _lstm_block(s3b_lib, [xg.cuda().contiguous() for xg in xgs], [l[1].cuda() for l in layer],
                              [None, layer[1][3].cuda()], lens, out_fmt)
    ref = torch.cat([DO.lstm(xgs[0].double(), layer[0][1].double(), lens),
                     DO.lstm((xgs[1] + layer[1][3]).double(), layer[1][1].double(), lens, backward=True)], -1)
    out = out.cpu()
    for b, m in enumerate(lens):
        assert torch.equal(out[b, m:], torch.zeros_like(out[b, m:])), b  # padding frames exactly zero, both halves
        if planes is not None:
            assert torch.equal(planes[b, m:].cpu(), torch.zeros_like(out[b, m:])), b
    rel = _rel(out, ref)
    elem = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"lstm B={B} T={T} fmt={out_fmt}: rel {rel:.3e} (measured/bound {rel / BLOCK_REL:.3f}), "
          f"elementwise {elem:.3e} ({elem / BLOCK_ELEM:.3f})")
    assert rel < BLOCK_REL and elem < BLOCK_ELEM
    if planes is not None:
        prel = _rel(planes.cpu(), out)
        print(f"  planes vs fp32 {prel:.3e}")
        assert prel < 1e-5  # the operand planes carry the fp32 output at operand precision


def test_lstm_block_bit_identical_in_any_batch(s3b_lib):
    """An utterance's outputs do not depend on the batch around it: alone, in a batch of 17 and in a batch of 520
    (two launches of at most 512 utterances) they are bit-identical."""
    T = 40
    g = torch.Generator().manual_seed(9)
    layer = _layer(2, 0)
    whhs = [l[1].cuda() for l in layer]
    x = torch.randn(520, T, H, generator=g) * 0.5
    xgs = [(x @ l[0].T + l[2] + l[3]).cuda().contiguous() for l in layer]
    lens = [int(v) for v in torch.randint(1, T + 1, (520,), generator=g)]
    lens[3] = T
    big, _ = _lstm_block(s3b_lib, xgs, whhs, [None, None], lens)
    mid, _ = _lstm_block(s3b_lib, [xg[100:117].contiguous() for xg in xgs], whhs, [None, None], lens[100:117])
    assert torch.equal(mid, big[100:117])
    for i in (3, 108, 519):
        alone, _ = _lstm_block(s3b_lib, [xg[i:i + 1].contiguous() for xg in xgs], whhs, [None, None], lens[i:i + 1])
        assert torch.equal(alone[0], big[i]), i


def test_lstm_block_refusals_and_fits(s3b_lib):
    ok = C.c_int32(-1)
    assert s3b_lib.s3b_lstm_fits(C.byref(ok)) == 0, s3b_lib.s3b_last_error()
    print(f"s3b_lstm_fits: {ok.value}")
    assert ok.value == 1
    xg = torch.zeros(1, 4, 4 * H, device="cuda")
    w = torch.zeros(4 * H, H, device="cuda")
    out = torch.zeros(1, 4, 2 * H, device="cuda")
    for lens, direction, want in (([5], 0, b"lens"), ([4], 2, b"direction")):
        r = s3b_lib.s3b_lstm_f32(C.c_void_p(xg.data_ptr()), C.c_void_p(w.data_ptr()), None, (C.c_int32 * 1)(*lens),
                                 1, 4, direction, -1, C.c_void_p(out.data_ptr()), None, None)
        assert r != 0 and want in s3b_lib.s3b_last_error()


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _expert(scheme, all_layers=True, **kw):
    from s3prl_b200.upstream.decoar import DecoarExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        ex = DecoarExpert(all_layers=all_layers, **kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


@pytest.mark.parametrize("scheme", ["f16q8", "bf16x3"])
@pytest.mark.parametrize("fixture", ["decoar_ref", "decoar_layers_ref", "decoar_layers_ref_c2"])
def test_matches_reference_golden(s3b_lib, fixture, scheme):
    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ex = _expert(scheme, all_layers=g["all_layers"], seed=g["weight_seed"])
    cs, ts = g["channel_stride"], g["time_stride"]
    worst = 0.0
    for case in g["cases"]:
        wavs = [w.cuda() for w in _wavs(case["lens"], case["wav_seed"])]
        res = ex(wavs)
        hs = res["hidden_states"]
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        assert res["last_hidden_state"] is hs[-1] or torch.equal(res["last_hidden_state"], hs[-1])
        for l, h in enumerate(hs):
            for b, n in enumerate(case["lens"]):
                m = 1 + (n - 400) // 160
                assert torch.equal(h[b, m:], torch.zeros_like(h[b, m:]))
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu()
            worst = max(worst, _rel(sub, case["sub"][l]))
    print(f"decoar {fixture} scheme={scheme}: worst per-hidden-state relative error {worst:.3e} "
          f"(measured/bound {worst / REL_TOL:.3f})")
    assert worst < REL_TOL


def test_decoar_is_decoar_layers_last(s3b_lib):
    wavs = [w.cuda() for w in _wavs([32000, 17000, 9000], seed=4)]
    last = _expert(None, all_layers=False)(wavs)["hidden_states"]
    layers = _expert(None, all_layers=True)(wavs)["hidden_states"]
    assert len(last) == 1 and len(layers) == 4
    assert torch.equal(last[0], layers[3])


def test_long_memory_on_gpu(s3b_lib):
    """Changing only the first 0.5 s of a 6 s utterance moves the forward half of every layer's output more than 300
    frames later; changing only the last 0.5 s moves the backward half more than 300 frames before it."""
    ex = _expert(None)
    g = torch.Generator().manual_seed(7)
    wav = torch.randn(96000, generator=g)
    head, tail = wav.clone(), wav.clone()
    head[:8000] += torch.randn(8000, generator=g)
    tail[-8000:] += torch.randn(8000, generator=g)
    a, b, c = (torch.stack(ex([w.cuda()])["hidden_states"]) for w in (wav, head, tail))
    T = a.shape[2]
    for l in range(4):
        fwd = (a[l, :, 50 + 300:, :H] - b[l, :, 50 + 300:, :H]).abs().max().item()
        bwd = (a[l, :, : T - 50 - 300, H:] - c[l, :, : T - 50 - 300, H:]).abs().max().item()
        print(f"layer {l}: forward change 300 frames after {fwd:.3e}, backward change 300 frames before {bwd:.3e}")
        assert fwd > 1e-3 and bwd > 1e-3


def test_bit_identical_lanes_shards_host(s3b_lib):
    ex = _expert(None)
    lens = [int(v) for v in torch.randint(560, 96000, (16,), generator=torch.Generator().manual_seed(3))]
    lens[5] = 96000
    wavs = [w.cuda() for w in _wavs(lens, seed=21)]
    full = torch.stack(ex(wavs)["hidden_states"])
    for lanes in (1, 2):  # lanes = 2 runs as one lane
        ex.lanes = lanes
        assert torch.equal(torch.stack(ex(wavs)["hidden_states"]), full), lanes
    ex.lanes = 0
    # sharded: two halves with global_max_len, and an utterance alone
    ex.global_max_len = max(lens)
    halves = [torch.stack(ex(wavs[s])["hidden_states"]) for s in (slice(0, 8), slice(8, 16))]
    assert torch.equal(torch.cat(halves, dim=1), full)
    alone = torch.stack(ex([wavs[11]])["hidden_states"])
    assert torch.equal(alone[:, 0], full[:, 11])
    ex.global_max_len = None
    # forward_host: 16 utterances run as two host chunks, 8 as one
    host16 = ex.forward_host([w.cpu() for w in wavs])
    assert torch.equal(host16, full.cpu())
    host8 = ex.forward_host([w.cpu() for w in wavs[:8]])
    assert torch.equal(host8, torch.stack(ex(wavs[:8])["hidden_states"]).cpu())


def test_forward_ex_refusals_and_profile(s3b_lib):
    from s3prl_b200 import lib

    ex = _expert(None)
    native = ex._native
    wavs = [w.cuda() for w in _wavs([16000, 8000], seed=1)]
    T = ex.num_frames(16000)
    out = torch.empty(4, 2, T, 2 * H, device="cuda")
    extra = torch.empty(4, 2, T, 2 * H, device="cuda")
    ptrs = (C.c_void_p * 2)(*[w.data_ptr() for w in wavs])
    for field in ("ffn_out", "last_residual"):
        opts = lib.S3BForwardOpts(**{field: extra.data_ptr()})
        r = native.lib.s3b_forward_ex(native.handle, ptrs, (C.c_int64 * 2)(16000, 8000), 2, 16000,
                                      C.c_void_p(out.data_ptr()), _stream(), C.byref(opts))
        assert r != 0 and b"ffn_out / last_residual" in native.lib.s3b_last_error()
    with pytest.raises(ValueError, match="560"):
        ex([torch.zeros(559, device="cuda")])
    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    ex(wavs)
    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
    lib.check(native.lib.s3b_profile_read_ex(native.handle, 6, ms, fl, n, 1))
    lib.check(native.lib.s3b_profile_enable(native.handle, 0))
    # post_extract_proj + 8 input GEMMs, fbank + CMVN, 8 recurrences (4 layers x 2 directions)
    assert list(n) == [9, 0, 2, 0, 0, 8], list(n)
    assert abs(fl[5] - 8 * 8.0 * H * H * 2 * T) < 1.0
    print(f"decoar profile ms: gemm {ms[0]:.3f} front end {ms[2]:.3f} recurrence {ms[5]:.3f}")


def test_repeated_calls_are_bit_identical(s3b_lib):
    """6 identical calls after a first one give its result bit for bit and each adds the same launch count."""
    from s3prl_b200.upstream.decoar import DecoarExpert

    g = torch.Generator().manual_seed(5)
    wavs = [torch.randn(n, generator=g).cuda() for n in (24000, 16000, 9000, 20000, 7000)]
    e = DecoarExpert(all_layers=True).to("cuda")
    ref = torch.stack(e(wavs)["hidden_states"]).clone()
    native = e._native
    counts = []
    for i in range(6):
        c0 = native.lib.s3b_launch_count(native.handle)
        res = e(wavs)
        counts.append(native.lib.s3b_launch_count(native.handle) - c0)
        assert torch.equal(torch.stack(res["hidden_states"]), ref), f"call {i + 1} changed the result"
    assert len(set(counts)) == 1, counts
