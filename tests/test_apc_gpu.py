"""GPU tests of APC / VQ-APC (``apc``, ``vq_apc``): the front end (kaldi fbank with the hamming window and CMVN, every
frame kept, written as operand planes) against torchaudio's own ``kaldi.fbank``; the GRU recurrence kernel at block
level (``s3b_gru_f32``) against the oracle's GRU in fp64; the whole model against the executed-reference goldens
(tests/golden/apc_ref*.pt, vq_apc_ref.pt) and the CPU oracle (tests/apc_oracle.py) in both GEMM operand schemes; and
bit-identical results across batch composition, lanes, shards, ``forward_host`` and apc / vq_apc.
Bounds: front end 1e-4 relative per utterance; recurrence block 1e-4 relative Frobenius and 2e-4 of the output scale
elementwise; model 2e-4 relative per layer. Every check prints measured / bound."""
import ctypes as C
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import apc_oracle as AO  # noqa: E402

pytestmark = pytest.mark.gpu

FEAT_REL = 1e-4
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
# front end
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_fmt", [0, 1])
def test_features_match_torchaudio(s3b_lib, out_fmt):
    from torchaudio.compliance import kaldi

    from s3prl_b200 import lib
    from s3prl_b200.upstream.apc import num_frames

    lens = [16000, 12345, 800, 560, 160000]
    wavs = _wavs(lens, seed=3)
    T = num_frames(max(lens))
    dev = [w.cuda() for w in wavs]
    out = torch.full((len(wavs), T, 80), float("nan"), device="cuda")
    ptrs = (C.c_void_p * len(wavs))(*[w.data_ptr() for w in dev])
    lib.check(s3b_lib.s3b_apc_features_f32(ptrs, (C.c_int64 * len(lens))(*lens), len(lens), out_fmt,
                                           C.c_void_p(out.data_ptr()), _stream()))
    torch.cuda.synchronize()
    out = out.cpu()
    worst = 0.0
    for b, w in enumerate(wavs):
        y = kaldi.fbank(w[None], num_mel_bins=80, sample_frequency=16000, window_type="hamming")
        ref = (y - y.mean(0, keepdim=True)) / (1e-10 + y.std(0, keepdim=True))
        m = len(ref)
        assert m == num_frames(len(w))
        assert torch.isfinite(out[b, :m]).all()
        assert torch.equal(out[b, m:], torch.zeros_like(out[b, m:])), b
        worst = max(worst, _rel(out[b, :m], ref))
    print(f"apc features out_fmt={out_fmt}: worst relative error {worst:.3e} (measured/bound {worst / FEAT_REL:.3f})")
    assert worst < FEAT_REL


# ------------------------------------------------------------------------------------------------
# recurrence block
# ------------------------------------------------------------------------------------------------
def _gru_block(s3b_lib, xg, whh, bhh, res, lens, out_fmt):
    from s3prl_b200 import lib

    B, T, _ = xg.shape
    out = torch.full((B, T, 512), float("nan"), device="cuda")
    planes = torch.full((B, T, 512), float("nan"), device="cuda") if out_fmt >= 0 else None
    lib.check(s3b_lib.s3b_gru_f32(
        C.c_void_p(xg.data_ptr()), C.c_void_p(whh.data_ptr()), C.c_void_p(bhh.data_ptr()),
        C.c_void_p(res.data_ptr()) if res is not None else None, (C.c_int32 * B)(*lens), B, T, 512, out_fmt,
        C.c_void_p(out.data_ptr()), C.c_void_p(planes.data_ptr()) if planes is not None else None, _stream()))
    torch.cuda.synchronize()
    return out, planes


_BT = [(1, 1), (1, 1998), (3, 2), (3, 17), (32, 998), (70, 17), (70, 1998)]


@pytest.mark.parametrize("out_fmt", [0, 1])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("B,T", _BT)
def test_gru_block_matches_oracle(s3b_lib, B, T, residual, out_fmt):
    from s3prl_b200.upstream.apc import fabricate_apc_state_dict

    sd = fabricate_apc_state_dict(1)
    g = torch.Generator().manual_seed(B * 7919 + T)
    whh = sd["rnn_layers.1.weight_hh_l0"].cuda()
    bhh = sd["rnn_layers.1.bias_hh_l0"].cuda()
    x = torch.randn(B, T, 512, generator=g)
    xg = (x @ sd["rnn_layers.1.weight_ih_l0"].T + sd["rnn_layers.1.bias_ih_l0"]).cuda()
    lens = [T] + [int(v) for v in torch.randint(1, T + 1, (B - 1,), generator=g)]
    res = (0.5 * torch.randn(B, T, 512, generator=g)).cuda() if residual else None
    out, planes = _gru_block(s3b_lib, xg.contiguous(), whh, bhh, res, lens, out_fmt)
    ref = AO.gru(xg.double(), whh.double(), bhh.double(), lens)
    if residual:
        valid = (torch.arange(T, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]).unsqueeze(-1)
        ref = ref + torch.where(valid, res.double(), torch.zeros_like(res.double()))
    for b, m in enumerate(lens):
        assert torch.equal(out[b, m:], torch.zeros_like(out[b, m:])), b  # padded frames exactly zero
        assert torch.equal(planes[b, m:], torch.zeros_like(planes[b, m:])), b
    rel = _rel(out, ref)
    elem = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    prel = _rel(planes, out)
    print(f"gru B={B} T={T} residual={residual} fmt={out_fmt}: rel {rel:.3e} (measured/bound {rel / BLOCK_REL:.3f}), "
          f"elementwise {elem:.3e} ({elem / BLOCK_ELEM:.3f}); planes vs fp32 {prel:.3e}")
    assert rel < BLOCK_REL and elem < BLOCK_ELEM
    assert prel < 1e-5  # the operand planes carry the fp32 output at operand precision


def test_gru_block_refusals(s3b_lib):
    x = torch.zeros(1, 4, 1536, device="cuda")
    w = torch.zeros(1536, 512, device="cuda")
    b = torch.zeros(1536, device="cuda")
    out = torch.zeros(1, 4, 512, device="cuda")
    for lens, hidden, want in (([5], 512, b"lens"), ([4], 256, b"hidden")):
        r = s3b_lib.s3b_gru_f32(C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(b.data_ptr()), None,
                                (C.c_int32 * 1)(*lens), 1, 4, hidden, -1, C.c_void_p(out.data_ptr()), None, None)
        assert r != 0 and want in s3b_lib.s3b_last_error()


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _expert(scheme, vq=False, **kw):
    from s3prl_b200.upstream.apc import ApcExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        ex = ApcExpert(vq=vq, **kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("fixture", ["apc_ref", "apc_ref_c2", "vq_apc_ref"])
def test_matches_reference_golden(s3b_lib, fixture, scheme):
    from s3prl_b200.upstream.apc import HIDDEN_STATES_INFO

    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    ex = _expert(scheme, vq=g["vq"], seed=g["weight_seed"])
    cs, ts = g["channel_stride"], g["time_stride"]
    worst = 0.0
    for case in g["cases"]:
        wavs = [w.cuda() for w in _wavs(case["lens"], case["wav_seed"])]
        res = ex(wavs)
        assert tuple(res["_hidden_states_info"]) == HIDDEN_STATES_INFO == tuple(case["names"])
        hs = res["hidden_states"]
        assert len(hs) == 3 and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu()
            worst = max(worst, _rel(sub, case["sub"][l]))
    print(f"apc {fixture} scheme={scheme or 'default'}: worst per-layer relative error {worst:.3e} "
          f"(measured/bound {worst / REL_TOL:.3f})")
    assert worst < REL_TOL


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("residual", [True, False])
def test_matches_oracle_ragged(s3b_lib, tmp_path, scheme, residual):
    from s3prl_b200.upstream.apc import apc_config, fabricate_apc_state_dict

    sd = fabricate_apc_state_dict(2)
    path = tmp_path / "apc.ckpt"
    torch.save({"config": apc_config(residual=residual), "model": sd}, path)
    ex = _expert(scheme, ckpt=str(path))
    lens = [48000, 560, 31234, 16001, 47999, 9000]
    wavs = _wavs(lens, seed=11)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    ref, m = AO.apc_forward(wavs, sd, residual=residual)
    worst = max(_rel(h.cpu(), r) for h, r in zip(hs, ref))
    for h in hs:
        for b, mb in enumerate(m):
            assert torch.equal(h[b, mb:], torch.zeros_like(h[b, mb:]))
    print(f"apc ragged residual={residual} scheme={scheme or 'default'}: worst {worst:.3e} "
          f"(measured/bound {worst / REL_TOL:.3f})")
    assert worst < REL_TOL


def test_long_memory_on_gpu(s3b_lib):
    """The fabricated weights' long memory holds on the native path: perturbing the first 100 ms of a 4 s utterance
    moves every layer's output at frames >= 300."""
    ex = _expert(None)
    g = torch.Generator().manual_seed(7)
    wav = torch.randn(64000, generator=g)
    alt = wav.clone()
    alt[:1600] += torch.randn(1600, generator=g)
    a = torch.stack(ex([wav.cuda()])["hidden_states"])
    b = torch.stack(ex([alt.cuda()])["hidden_states"])
    for l in range(3):
        late = (a[l, :, 300:] - b[l, :, 300:]).abs().max().item()
        print(f"layer {l}: max change at frames >= 300: {late:.3e}")
        assert late > 1e-3


def test_bit_identical_batch_lanes_shards_host_vq(s3b_lib):
    ex = _expert(None)
    lens = [int(v) for v in torch.randint(560, 160000, (32,), generator=torch.Generator().manual_seed(3))]
    lens[5] = 160000
    wavs = [w.cuda() for w in _wavs(lens, seed=21)]
    full = torch.stack(ex(wavs)["hidden_states"])
    # an utterance alone, padded to the batch's max_len, vs inside the batch of 32
    ex.global_max_len = max(lens)
    for i in (0, 5, 17):
        alone = torch.stack(ex([wavs[i]])["hidden_states"])
        assert torch.equal(alone[:, 0], full[:, i]), i
    # sharded: two halves with global_max_len
    halves = [torch.stack(ex(wavs[s])["hidden_states"]) for s in (slice(0, 16), slice(16, 32))]
    assert torch.equal(torch.cat(halves, dim=1), full)
    ex.global_max_len = None
    for lanes in (1, 2):
        ex.lanes = lanes
        assert torch.equal(torch.stack(ex(wavs)["hidden_states"]), full), lanes
    ex.lanes = 0
    host = ex.forward_host([w.cpu() for w in wavs[:8]])
    dev8 = torch.stack(ex(wavs[:8])["hidden_states"]).cpu()
    assert torch.equal(host, dev8)
    vq = _expert(None, vq=True)
    assert torch.equal(torch.stack(vq(wavs[:8])["hidden_states"]).cpu(), dev8)


def test_forward_ex_refusals_and_profile(s3b_lib):
    from s3prl_b200 import lib

    ex = _expert(None)
    native = ex._native
    wavs = [w.cuda() for w in _wavs([16000, 8000], seed=1)]
    T = ex.num_frames(16000)
    out = torch.empty(3, 2, T, 512, device="cuda")
    ffn = torch.empty(3, 2, T, 512, device="cuda")
    opts = lib.S3BForwardOpts(ffn_out=ffn.data_ptr())
    ptrs = (C.c_void_p * 2)(*[w.data_ptr() for w in wavs])
    r = native.lib.s3b_forward_ex(native.handle, ptrs, (C.c_int64 * 2)(16000, 8000), 2, 16000,
                                  C.c_void_p(out.data_ptr()), _stream(), C.byref(opts))
    assert r != 0 and b"ffn_out" in native.lib.s3b_last_error()
    with pytest.raises(ValueError, match="560"):
        ex([torch.zeros(559, device="cuda")])
    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    ex(wavs)
    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
    lib.check(native.lib.s3b_profile_read_ex(native.handle, 6, ms, fl, n, 1))
    lib.check(native.lib.s3b_profile_enable(native.handle, 0))
    assert list(n) == [3, 0, 2, 0, 0, 3], list(n)  # 3 input GEMMs, fbank + CMVN, 3 recurrences
    print(f"apc profile ms: gemm {ms[0]:.3f} front end {ms[2]:.3f} recurrence {ms[5]:.3f}")


def test_repeated_calls_are_bit_identical(s3b_lib):
    """10 identical calls after a first one give its result bit for bit and each adds the same launch count."""
    from s3prl_b200.upstream.apc import ApcExpert

    g = torch.Generator().manual_seed(5)
    wavs = [torch.randn(n, generator=g).cuda() for n in (24000, 16000, 9000, 20000, 7000)]
    e = ApcExpert().to("cuda")
    ref = torch.stack(e(wavs)["hidden_states"]).clone()
    native = e._native
    counts = []
    for i in range(10):
        c0 = native.lib.s3b_launch_count(native.handle)
        res = e(wavs)
        counts.append(native.lib.s3b_launch_count(native.handle) - c0)
        assert torch.equal(torch.stack(res["hidden_states"]), ref), f"call {i + 1} changed the result"
    assert len(set(counts)) == 1, counts


def test_occupancy(s3b_lib):
    """At least one cluster of the recurrence kernel fits on the device (finalize fails otherwise)."""
    n = C.c_int32(-1)
    assert s3b_lib.s3b_gru_max_active_clusters(C.byref(n)) == 0, s3b_lib.s3b_last_error()
    print(f"recurrence kernel: {n.value} co-resident clusters of 16 CTAs")
    assert n.value >= 1
