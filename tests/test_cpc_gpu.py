"""GPU tests of modified CPC (``modified_cpc``): one conv + ChannelNorm + ReLU at block level (``s3b_cpc_conv_f32``)
against fp64 ``conv1d`` in both GEMM operand schemes at every residue of the input length mod the stride, the LSTM
recurrence at block level (``s3b_cpc_lstm_f32``) against fp64, the whole model against the executed-reference goldens
(tests/golden/cpc_ref*.pt) and the fp64 CPU oracle (tests/cpc_oracle.py), bit-identical results across batch order
and composition, padded length (frames before an utterance's last), shards, lanes, ``forward_host``, repeated calls and
a long-lived model after a poisoned call, and the launch counts.
Bounds: block 1e-4 relative Frobenius; model 2e-4 relative per hidden state. Every check prints measured / bound."""
import ctypes as C
import os
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
sys.path.insert(0, str(ROOT / "tests"))

import cpc_oracle as CO  # noqa: E402

pytestmark = pytest.mark.gpu

BLOCK_REL = 1e-4
REL_TOL = 2e-4


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _wavs(lens, seed, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) * scale for n in lens]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------------
# block level
# ------------------------------------------------------------------------------------------------
def _cpc_conv(s3b_lib, x, layer, w, bias, gamma, beta, scheme):
    from s3prl_b200 import lib

    B, L = x.shape[0], x.shape[1]
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    T = (L + 2 * p - 2 * s) // s + 1
    out = torch.full((B, T, 256), float("nan"), device="cuda")
    lib.check(s3b_lib.s3b_cpc_conv_f32(_ptr(x), B, L, layer, _ptr(w), _ptr(bias), _ptr(gamma), _ptr(beta), scheme,
                                       _ptr(out), _stream()))
    torch.cuda.synchronize()
    return out


def _conv_ref(x, layer, w, bias, gamma, beta):
    xin = x.double().unsqueeze(1) if layer == 0 else x.double().transpose(1, 2)
    y = F.conv1d(xin, w.double(), bias.double(), stride=CO.STRIDES[layer], padding=CO.PADDINGS[layer])
    return CO.channel_norm_relu(y, gamma.double(), beta.double()).transpose(1, 2)


_T = [1, 2, 127, 128, 129, 1000]


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("layer", [0, 1, 2, 3, 4])
def test_cpc_conv_block_matches_fp64(s3b_lib, scheme, layer):
    s, p = CO.STRIDES[layer], CO.PADDINGS[layer]
    cin = 1 if layer == 0 else 256
    worst, n = 0.0, 0
    for T in _T:
        for r in range(s):  # every residue of the input length mod the stride
            L = s * (T - 1) + 2 * s - 2 * p + r
            g = torch.Generator().manual_seed(1000 * layer + 10 * T + r)
            B = 3 if T < 1000 else 2
            x = (torch.randn(B, L, generator=g) * 0.1 if layer == 0 else torch.relu(torch.randn(B, L, 256, generator=g)))
            w = torch.randn(256, cin, 2 * s, generator=g) / (cin * 2 * s) ** 0.5
            bias, gamma, beta = 0.1 * torch.randn(256, generator=g), 0.5 + torch.rand(256, generator=g), \
                0.2 * torch.randn(256, generator=g)
            out = _cpc_conv(s3b_lib, x.cuda(), layer, w.cuda(), bias.cuda(), gamma.cuda(), beta.cuda(), scheme)
            ref = _conv_ref(x, layer, w, bias, gamma, beta)
            assert out.shape == ref.shape and out.shape[1] == T, (out.shape, ref.shape, T)
            e = _rel(out.cpu(), ref)
            worst, n = max(worst, e), n + 1
            assert e < BLOCK_REL, (T, r, e)
    print(f"cpc conv {layer} scheme={scheme}: worst relative error over {n} lengths (T={_T}, every residue mod {s}): "
          f"{worst:.3e} (measured/bound {worst / BLOCK_REL:.3f})")


def test_cpc_conv_refusals(s3b_lib):
    x = torch.zeros(1, 400, 256, device="cuda")
    w = torch.zeros(256, 256, 8, device="cuda")
    v = torch.zeros(256, device="cuda")
    out = torch.zeros(1, 400, 256, device="cuda")
    for B, L, layer, want in ((1, 400, 5, b"layer"), (1, 400, -1, b"layer"), (0, 400, 1, b"batch"),
                              (1, 3, 1, b"too short"), (1, 3, 0, b"too short")):
        r = s3b_lib.s3b_cpc_conv_f32(_ptr(x), B, L, layer, _ptr(w), _ptr(v), _ptr(v), _ptr(v), -1, _ptr(out), None)
        assert r != 0 and want in s3b_lib.s3b_last_error(), (B, L, layer)


def _lstm_ref(x, sd, k):
    return CO.lstm_layer(x, *(sd[f"gAR.baseNet.{n}_l{k}"].double() for n in ("weight_ih", "weight_hh", "bias_ih",
                                                                             "bias_hh")))


def _cpc_lstm(s3b_lib, xg, whh, out_fmt=-1):
    from s3prl_b200 import lib

    B, T = xg.shape[0], xg.shape[1]
    out = torch.full((B, T, 256), float("nan"), device="cuda")
    planes = torch.full((B, T, 256), float("nan"), device="cuda") if out_fmt >= 0 else None
    lib.check(s3b_lib.s3b_cpc_lstm_f32(_ptr(xg), _ptr(whh), B, T, out_fmt, _ptr(out), _ptr(planes), _stream()))
    torch.cuda.synchronize()
    return out, planes


@pytest.mark.parametrize("B,T", [(1, 1), (4, 37), (5, 2000), (70, 300)])
def test_cpc_lstm_matches_fp64(s3b_lib, B, T):
    """One and two layers from xg = W_ih x + b_ih + b_hh, against the fp64 cell; B = 5 and 70 leave the last cluster's
    group of four partly filled."""
    from s3prl_b200.upstream.cpc import fabricate_cpc_state_dict

    n_active = C.c_int32()
    s3b_lib.s3b_cpc_lstm_max_active_clusters(C.byref(n_active))
    sd = fabricate_cpc_state_dict(4, 2)
    g = torch.Generator().manual_seed(B * 7 + T)
    x = torch.relu(torch.randn(B, T, 256, generator=g, dtype=torch.float64))
    worst = 0.0
    inp = x
    for k in range(2):
        xg = (inp.float() @ sd[f"gAR.baseNet.weight_ih_l{k}"].T + sd[f"gAR.baseNet.bias_ih_l{k}"]
              + sd[f"gAR.baseNet.bias_hh_l{k}"])
        out, planes = _cpc_lstm(s3b_lib, xg.cuda().contiguous(), sd[f"gAR.baseNet.weight_hh_l{k}"].cuda(), k)
        ref = _lstm_ref(inp, sd, k)
        e = _rel(out.cpu(), ref)
        worst = max(worst, e)
        assert e < BLOCK_REL, (k, e)
        assert _rel(planes, out) < 1e-4  # the operand planes hold the same values
        inp = out.cpu().double()
    print(f"cpc lstm B={B} T={T}: worst relative error over 2 layers {worst:.3e} (measured/bound "
          f"{worst / BLOCK_REL:.3f}); {n_active.value} clusters of 8 CTAs co-resident, {(B + 3) // 4} needed")


def test_cpc_lstm_bit_identical_in_any_slot(s3b_lib):
    from s3prl_b200.upstream.cpc import fabricate_cpc_state_dict

    sd = fabricate_cpc_state_dict(4)
    whh = sd["gAR.baseNet.weight_hh_l0"].cuda()
    g = torch.Generator().manual_seed(5)
    xg = torch.randn(11, 50, 1024, generator=g).cuda()
    full, _ = _cpc_lstm(s3b_lib, xg, whh)
    for i in (0, 3, 6, 10):
        alone, _ = _cpc_lstm(s3b_lib, xg[i : i + 1].contiguous(), whh)
        assert torch.equal(alone[0], full[i]), i
    perm = torch.randperm(11, generator=g)
    shuffled, _ = _cpc_lstm(s3b_lib, xg[perm].contiguous(), whh)
    assert torch.equal(shuffled, full[perm])


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _expert(scheme, **kw):
    from s3prl_b200.upstream.cpc import CpcExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        ex = CpcExpert(**kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


def _ckpt(tmp_path, over, seed):
    from s3prl_b200.upstream.cpc import cpc_config, fabricate_cpc_state_dict

    config = cpc_config(**over)
    sd = fabricate_cpc_state_dict(seed, config["nLevelsGRU"])
    path = tmp_path / "cpc.pt"
    torch.save({"config": config, "weights": sd}, path)
    return str(path), sd


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("fixture", ["cpc_ref", "cpc_ref_c2", "cpc_ref_variant"])
def test_matches_reference_golden(s3b_lib, tmp_path, fixture, scheme):
    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    path, _ = _ckpt(tmp_path, g["config"], g["weight_seed"])
    ex = _expert(scheme, ckpt=path)
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        wavs = [w.cuda() for w in _wavs(case["lens"], case["wav_seed"], case["wav_scale"])]
        res = ex(wavs)
        assert tuple(res["_hidden_states_info"]) == tuple(case["names"])
        hs = res["hidden_states"]
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            err = _rel(h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu(), case["sub"][l])
            print(f"cpc {fixture} lens={case['lens']} scheme={scheme or 'default'} state {l}: abs max "
                  f"{h.abs().max().item():.3f}, relative error {err:.3e} (measured/bound {err / REL_TOL:.3f})")
            assert err < REL_TOL


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("levels", [1, 2])
def test_matches_oracle_ragged(s3b_lib, tmp_path, scheme, levels):
    path, sd = _ckpt(tmp_path, {"nLevelsGRU": levels}, 2)
    ex = _expert(scheme, ckpt=path)
    lens = [48000, 159, 31234, 16001, 47999, 90, 9000]
    wavs = _wavs(lens, seed=11)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    ref = CO.forward(wavs, sd, levels)
    assert len(hs) == len(ref) == 2
    for l, (h, r) in enumerate(zip(hs, ref)):
        err = _rel(h.cpu(), r)
        print(f"cpc ragged levels={levels} scheme={scheme or 'default'} state {l}: abs max {r.abs().max().item():.3f}"
              f", relative error {err:.3e} (measured/bound {err / REL_TOL:.3f})")
        assert err < REL_TOL


def test_bit_identical_batch_shards_lanes_host_repeats(s3b_lib):
    from s3prl_b200.upstream.cpc import num_frames

    ex = _expert(None)
    lens = [int(v) for v in torch.randint(100, 160000, (32,), generator=torch.Generator().manual_seed(3))]
    lens[5] = 160000
    wavs = [w.cuda() for w in _wavs(lens, seed=21)]
    full = torch.stack(ex(wavs)["hidden_states"]).clone()
    # batch order at the same max_len
    perm = torch.randperm(32, generator=torch.Generator().manual_seed(4)).tolist()
    assert torch.equal(torch.stack(ex([wavs[i] for i in perm])["hidden_states"]), full[:, perm])
    # an utterance alone, padded to the batch's max_len, vs inside the batch of 32; shards of the batch
    ex.global_max_len = max(lens)
    for i in (0, 5, 17):
        alone = torch.stack(ex([wavs[i]])["hidden_states"])
        assert torch.equal(alone[:, 0], full[:, i]), i
    halves = [torch.stack(ex(wavs[s])["hidden_states"]) for s in (slice(0, 16), slice(16, 32))]
    assert torch.equal(torch.cat(halves, dim=1), full)
    ex.global_max_len = None
    # a different max_len: frames before an utterance's last one are unchanged
    for i in (0, 17, 30):
        alone = torch.stack(ex([wavs[i]])["hidden_states"])
        t = num_frames(lens[i]) - 1
        assert torch.equal(alone[:, 0, :t], full[:, i, :t]), i
    for lanes in (1, 2):
        ex.lanes = lanes
        assert torch.equal(torch.stack(ex(wavs)["hidden_states"]), full), lanes
    ex.lanes = 0
    host = ex.forward_host([w.cpu() for w in wavs[:8]])
    dev8 = torch.stack(ex(wavs[:8])["hidden_states"]).cpu()
    assert torch.equal(host, dev8)
    native = ex._native
    counts = []
    for i in range(10):
        c0 = native.lib.s3b_launch_count(native.handle)
        res = torch.stack(ex(wavs)["hidden_states"])
        counts.append(native.lib.s3b_launch_count(native.handle) - c0)
        assert torch.equal(res, full), f"call {i + 1} changed the result"
    assert len(set(counts)) == 1, counts
    # a long-lived model after a poisoned call larger than every probe (NaN, inf, 1e30 samples) and calls of other
    # shapes gives what a fresh one gives: no pad row of a reused workspace leaks into a result
    g = torch.Generator().manual_seed(8)
    poison = []
    for n in (170000, 165000, 150000, 170000):
        p = torch.randn(n, generator=g) * 1e30
        p[::7] = float("nan")
        p[3::11] = float("inf")
        poison.append(p.cuda())
    ex.lanes = 2
    bad = torch.stack(ex(poison)["hidden_states"])
    assert not torch.isfinite(bad[1]).all()
    ex.lanes = 0
    fresh = _expert(None)
    for probe in (wavs[3:9], wavs[:1], wavs):
        assert torch.equal(torch.stack(ex(probe)["hidden_states"]), torch.stack(fresh(probe)["hidden_states"]))
    print(f"cpc bit-identity: batch order and composition, max_len (frames before the last), shards, lanes 1/2, "
          f"forward_host, 10 repeats ({counts[0]} launches each), long-lived model after a poisoned call vs fresh")


@pytest.mark.parametrize("levels", [1, 3])
def test_launch_counts_profile_and_refusals(s3b_lib, tmp_path, levels):
    from s3prl_b200 import lib

    path, _ = _ckpt(tmp_path, {"nLevelsGRU": levels}, 1)
    ex = _expert(None, ckpt=path)
    ex.lanes = 1
    native = ex._native
    wavs = [w.cuda() for w in _wavs([16000, 8000], seed=1)]
    T = ex.num_frames(16000)
    out = torch.empty(2, 2, T, 256, device="cuda")
    ptrs = (C.c_void_p * 2)(*[w.data_ptr() for w in wavs])
    for field in ("ffn_out", "last_residual"):
        opts = lib.S3BForwardOpts(**{field: out.data_ptr()})
        r = native.lib.s3b_forward_ex(native.handle, ptrs, (C.c_int64 * 2)(16000, 8000), 2, 16000,
                                      C.c_void_p(out.data_ptr()), _stream(), C.byref(opts))
        assert r != 0 and field.encode() in native.lib.s3b_last_error()
    with pytest.raises(ValueError, match="159"):
        ex([torch.zeros(158, device="cuda"), torch.zeros(20, device="cuda")])
    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    c0 = native.lib.s3b_launch_count(native.handle)
    ex(wavs)
    total = native.lib.s3b_launch_count(native.handle) - c0
    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
    lib.check(native.lib.s3b_profile_read_ex(native.handle, 6, ms, fl, n, 1))
    lib.check(native.lib.s3b_profile_enable(native.handle, 0))
    # 4 conv GEMMs + 1 input GEMM per layer; conv 0; 4 norms; the wave pack; 1 recurrence per layer
    assert list(n) == [4 + levels, 0, 1, 4, 1, levels], list(n)
    assert total == 10 + 2 * levels, total
    # FLOPs with the real channels: conv i has 2 s_i taps of 256 channels
    L = [16000]
    for s, p in zip(CO.STRIDES, CO.PADDINGS):
        L.append((L[-1] + 2 * p - 2 * s) // s + 1)
    want = sum(2.0 * 2 * L[i + 1] * 256 * 256 * 2 * CO.STRIDES[i] for i in range(1, 5)) + levels * 2.0 * 2 * T * 1024 * 256
    assert abs(fl[0] / want - 1) < 1e-12, (fl[0], want)
    print(f"cpc profile ms (levels={levels}): gemm {ms[0]:.3f} conv0 {ms[2]:.3f} norm {ms[3]:.3f} "
          f"recurrence {ms[5]:.3f}")


def test_finalize_names_a_missing_tensor(s3b_lib):
    from s3prl_b200 import lib
    from s3prl_b200.upstream.cpc import CpcExpert

    ex = CpcExpert()
    ex._state_dict_host["gEncoder.batchNorm2.weight"] = torch.ones(256)  # not [1, 256, 1]
    with pytest.raises(lib.S3BError, match=r"gEncoder\.batchNorm2\.weight"):
        ex.to("cuda")([torch.randn(16000, device="cuda")])
