"""GPU tests of NPC (``npc``): the tap convolution at block level (``s3b_npc_conv_f32``) in both GEMM operand schemes,
per element against fp64 ``conv1d`` and against the scheme's emulated operand decomposition, the band of masked taps
left out bit-exactly, the neighbouring utterances of a batch never read, the whole model against the executed-reference
goldens (tests/golden/npc_ref*.pt) and the fp64 CPU oracle (tests/npc_oracle.py), bit-identical results across batch
composition, shards, lanes, ``forward_host``, repeated calls and a long-lived model, the launch counts, and the
library's refusal of a checkpoint whose conv_mask is not its config's.
Bounds: block per element, derived from the operands as in tests/test_gemm_layouts_gpu.py (_gemm_refs); model 2e-4
relative per hidden state. Every check prints measured / bound."""
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

import npc_oracle as NO  # noqa: E402
from test_gemm_layouts_gpu import _check, _epilogue, _gemm_refs, _operands  # noqa: E402
from test_port_shapes_gpu import LONG_K, _dropped_steps  # noqa: E402

pytestmark = pytest.mark.gpu

REL_TOL = 2e-4
TANH_ERR = 2.0**-22  # tanhf: at most 2 ulp of its result


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------------
# block level
# ------------------------------------------------------------------------------------------------
def _npc_conv(s3b_lib, x, w, k, mask, bias, res, act, res_first, scheme, pre=False):
    from s3prl_b200 import lib

    B, T, cin = x.shape
    out = torch.full((B, T, 512), float("nan"), device="cuda")
    out_pre = torch.full((B, T, 512), float("nan"), device="cuda") if pre else None
    lib.check(s3b_lib.s3b_npc_conv_f32(_ptr(x), B, T, cin, _ptr(w), k, mask, _ptr(bias), _ptr(res), act, res_first,
                                       scheme, _ptr(out), _ptr(out_pre), _stream()))
    torch.cuda.synchronize()
    return out, out_pre


def _unmasked_taps(k, mask):
    head = (k - mask) // 2
    return [j for j in range(k) if not head <= j < head + mask]


def _im2col(x, w, k, mask):
    """The GEMM the kernel runs, as fp32 matrices: row (b, t) of A is the unmasked taps x[b, t + j - (k - 1) / 2], zero
    outside [0, T), tap-major; W [512][u c_in] the same taps of w. Also which rows read a frame inside [0, T) for every
    tap (interior) and for none (empty: the output is act(bias) there)."""
    B, T, cin = x.shape
    taps = torch.tensor(_unmasked_taps(k, mask), device="cuda")
    h = (k - 1) // 2
    xp = F.pad(x, (0, 0, h, h))  # [B][T + k - 1][cin]
    idx = torch.arange(T, device="cuda")[:, None] + taps[None, :]  # padded frame of tap jj of output t
    a = xp[:, idx, :].reshape(B * T, len(taps) * cin)
    wk = w[:, :, taps].permute(0, 2, 1).reshape(512, len(taps) * cin)
    inside = ((idx - h >= 0) & (idx - h < T)).repeat(B, 1)
    return a, wk, inside.all(1), ~inside.any(1)


def _separation(what, a, w, e1, e2, interior, scheme):
    """The bounds' separation for _check. _gemm_refs counts every 16-wide k-step of K in the accumulation bound; rows
    with taps outside the utterance run fewer MMAs on non-zero operands, so their bounds are closer than the kernel's
    accumulation is, and the separation is taken over the interior rows (none: not checked). Where it is under 50x for
    f16q8 at K >= 5120 (tests/test_port_shapes_gpu.py), _dropped_steps checks what it stands for instead.
    Returns (gemm, apart_check) for _check."""
    if not interior.any():
        return (e1, e2), False
    gemm = (e1[interior], e2[interior])
    if scheme == 1 and a.shape[1] >= LONG_K and (gemm[0] / gemm[1]).median().item() < 50.0:
        _dropped_steps(what, a[interior], w, gemm[1])
        return gemm, False
    return gemm, True


def _act_epilogue(pre, e, bias, res, act, res_first):
    """fp64 epilogue of the NPC conv: v = pre + bias (+ residual if res_first); act; out_pre; (+ residual) and the
    propagated bounds (_epilogue: the fp32 bias and residual adds). ReLU is 1-Lipschitz and exact in fp32; tanh has
    slope <= 1, and tanhf adds at most 2 ulp (CUDA's documented maximum), bounded by TANH_ERR |tanh(v)|.
    Returns (out, bound, out_pre, bound_pre)."""
    v, ev = _epilogue(pre, e, bias, res=res if res_first else None)
    if act == 1:
        v = torch.relu(v)
    elif act == 2:
        v = torch.tanh(v)
        ev = ev + TANH_ERR * v.abs()
    if res_first:
        return v, ev, None, None
    out = v + res.double()
    return out, ev + 2.0**-24 * out.abs(), v, ev


# (c_in, k, mask): the served config's shapes — conv k = 3 on 80 and 512 channels, the 1x1 linear, the masked convs of
# kernel 15 / mask 5 (bands of 7, 9, 11, 13 taps) — and a kernel without a mask
_SHAPES = [(80, 3, 0), (512, 3, 0), (512, 1, 0), (512, 15, 7), (512, 15, 9), (512, 15, 11), (512, 15, 13),
           (512, 15, 0), (80, 9, 3)]
_T = [1, 2, 7, 8, 127, 128, 129, 998]
_UTT_SCALES = (1.0, 0.25, 0.5)  # per utterance of a batch of 3: a row read from the wrong utterance shows


def _conv_inputs(T, cin, k, mask, mag, seed):
    """x [3][T][c_in], w [512][c_in][k] at _operands' magnitudes (unit: w ~ 1 / sqrt(u c_in), the taps contracted;
    small: x 1e-3 of that, the f16q8 residuals in e4m3's subnormals; large: |x| up to 3000, |w| up to 40, where A_h8
    and W_h8 saturate, standing in for BatchNorm-folded weights and activations past fp8's range), the utterances at
    different scales; bias and residual at the scale of the convolution's output."""
    B, u = 3, k - mask
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, wr = _operands(B * T, 512 * k, cin, mag, g)  # x rows; one weight row per (tap, output channel)
    x = a.view(B, T, cin) * torch.tensor(_UTT_SCALES, device="cuda")[:, None, None]
    w = wr.view(k, 512, cin).permute(1, 2, 0).contiguous()
    if mag != "large":
        w = w / u**0.5  # _operands scales by 1 / sqrt(c_in); the conv contracts u taps of c_in
    y = 1.0 if mag == "unit" else 1e-3**2 if mag == "small" else 700 * 10 * (u * cin) ** 0.5
    bias = torch.randn(512, device="cuda", generator=g) * 0.1 * y
    res = torch.randn(B, T, 512, device="cuda", generator=g) * y
    return x, w, bias, res


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("cin,k,mask", _SHAPES)
def test_npc_conv_block_matches_fp64(s3b_lib, scheme, cin, k, mask):
    """The same-padded tap convolution of three utterances against two references per element (the module's bounds):
    the exact product in fp64, and the scheme's operand decomposition emulated in torch. Both run on the im2col view
    of the GEMM the kernel runs (_im2col), which must itself equal F.conv1d in fp64 with the band of masked taps
    zeroed. Epilogue: activation none, ReLU or tanh, with the residual added after the activation (out_pre checked
    too: the value before the add) or before it (res_first). At k = 15 and T <= 7 some frames have every unmasked tap
    outside the utterance: there the output is act(bias) exactly (act(bias + residual) with res_first)."""
    for mag, T in [(m, t) for m in ("unit", "small", "large") for t in _T]:
        what = f"npc conv c_in={cin} k={k} mask={mask} s{scheme} {mag} T={T}"
        x, w, bias, res = _conv_inputs(T, cin, k, mask, mag, T * 31 + k * 7 + mask + cin + 1000 * scheme + len(mag))
        a, wk, interior, empty = _im2col(x, w, k, mask)
        exact, emu, e1, e2 = _gemm_refs(a, wk, scheme)
        wm = w.double().clone()
        if mask:
            wm[:, :, (k - mask) // 2 : (k + mask) // 2] = 0
        conv = F.conv1d(x.double().transpose(1, 2), wm, padding=(k - 1) // 2).transpose(1, 2).reshape(-1, 512)
        assert ((conv - exact).abs() <= 1e-6 * e1).all()  # the im2col view is the convolution (to fp64 rounding)
        gemm, apart_check = _separation(what, a, wk, e1, e2, interior, scheme)
        r = res.view(-1, 512)
        for act in (0, 1, 2):
            for res_first in (0, 1):
                out, out_pre = _npc_conv(s3b_lib, x, w, k, mask, bias, res, act, res_first, scheme, pre=not res_first)
                out, tag = out.view(-1, 512), f"{what} act={act} res_first={res_first}"
                ref1, b1, pre1, bp1 = _act_epilogue(conv, e1, bias, r, act, res_first)
                ref2, b2, pre2, bp2 = _act_epilogue(emu, e2, bias, r, act, res_first)
                _check(tag, out, ref1, b1, ref2, b2, gemm, scheme, frob=mag == "unit", apart_check=apart_check)
                if not res_first:
                    _check(f"{tag} out_pre", out_pre.view(-1, 512), pre1, bp1, pre2, bp2, gemm, scheme,
                           frob=mag == "unit", apart_check=apart_check)
                    assert torch.equal(out, out_pre.view(-1, 512) + r), "out != out_pre + residual"
                if empty.any() and act != 2:  # no tap inside the utterance: the accumulator is exactly zero
                    v = bias.expand_as(r) + r if res_first else bias.expand_as(r)
                    v = torch.relu(v) if act == 1 else v
                    want = v if res_first else v + r
                    assert torch.equal(out[empty], want[empty]), (tag, "frames without a tap in the utterance")


@pytest.mark.parametrize("scheme", [0, 1])
def test_masked_band_is_left_out_bit_exactly(s3b_lib, scheme):
    """Rewriting the input rows inside output row t's masked band leaves output row t bit-identical: the band's taps
    are not contracted at all (a 0 * x product would still turn an inf or NaN input into NaN)."""
    k, mask, T, t = 15, 9, 200, 100
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, T, 512, generator=g).cuda()
    w = (torch.randn(512, 512, k, generator=g) / (512 * (k - mask)) ** 0.5).cuda()
    bias = (0.1 * torch.randn(512, generator=g)).cuda()
    a, _ = _npc_conv(s3b_lib, x, w, k, mask, bias, None, 2, 0, scheme)
    y = x.clone()
    r = (mask - 1) // 2
    y[:, t - r : t + r + 1] = torch.randn(2, 2 * r + 1, 512, generator=g).cuda() * 1e3
    y[0, t] = float("nan")
    b, _ = _npc_conv(s3b_lib, y, w, k, mask, bias, None, 2, 0, scheme)
    assert torch.equal(a[:, t], b[:, t])
    assert not torch.equal(a[:, t + 1], b[:, t + 1])  # one frame on, the band has moved off a rewritten row
    print(f"masked band scheme={scheme}: row {t} bit-identical after rewriting rows {t - r}..{t + r}")


@pytest.mark.parametrize("scheme", [0, 1])
@pytest.mark.parametrize("cin,k,mask,T", [(80, 3, 0, 129), (512, 3, 0, 1), (512, 15, 7, 7), (512, 15, 13, 129),
                                          (512, 15, 0, 8)])
def test_neighbours_are_never_read(s3b_lib, cin, k, mask, scheme, T):
    """Utterance 1 of a batch of 3 whose utterances 0 and 2 are all NaN is bit-identical to utterance 1 run alone: the
    halo of same padding reaches past both ends of every utterance at these lengths, and must read zeros there."""
    x, w, bias, res = _conv_inputs(T, cin, k, mask, "unit", T + k + mask + cin + scheme)
    alone, _ = _npc_conv(s3b_lib, x[1:2].contiguous(), w, k, mask, bias, res[1:2].contiguous(), 2, 0, scheme)
    x[0], x[2] = float("nan"), float("nan")
    res[0], res[2] = float("nan"), float("nan")
    out, _ = _npc_conv(s3b_lib, x, w, k, mask, bias, res, 2, 0, scheme)
    assert torch.isfinite(alone).all()
    assert torch.equal(out[1], alone[0])
    print(f"npc conv c_in={cin} k={k} mask={mask} T={T} s{scheme}: utterance 1 between NaN neighbours bit-identical")


def test_npc_conv_refusals(s3b_lib):
    x = torch.zeros(1, 4, 512, device="cuda")
    w = torch.zeros(512, 512, 15, device="cuda")
    out = torch.zeros(1, 4, 512, device="cuda")
    for cin, k, mask, act, rf, pre, want in ((256, 15, 0, 0, 0, False, b"c_in"), (512, 14, 0, 0, 0, False, b"k "),
                                             (512, 15, 4, 0, 0, False, b"mask"), (512, 15, 15, 0, 0, False, b"mask"),
                                             (512, 15, 0, 3, 0, False, b"act"), (512, 15, 0, 1, 1, True, b"out_pre")):
        r = s3b_lib.s3b_npc_conv_f32(_ptr(x), 1, 4, cin, _ptr(w), k, mask, None, _ptr(x), act, rf, -1, _ptr(out),
                                     _ptr(out) if pre else None, None)
        assert r != 0 and want in s3b_lib.s3b_last_error(), (cin, k, mask, act, rf, pre)


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _expert(scheme, **kw):
    from s3prl_b200.upstream.npc import NpcExpert

    saved = os.environ.get("S3B_GEMM_SCHEME")
    if scheme is not None:
        os.environ["S3B_GEMM_SCHEME"] = scheme
    try:
        ex = NpcExpert(**kw).to("cuda")
        ex._ensure_native(torch.device("cuda", torch.cuda.current_device()))  # the scheme is read here
        return ex
    finally:
        if scheme is not None:
            if saved is None:
                os.environ.pop("S3B_GEMM_SCHEME", None)
            else:
                os.environ["S3B_GEMM_SCHEME"] = saved


def _ckpt(tmp_path, over, seed):
    from s3prl_b200.upstream.npc import fabricate_npc_state_dict, npc_config

    config = npc_config(**over)
    sd = fabricate_npc_state_dict(seed, config["model"]["paras"])
    path = tmp_path / "npc.ckpt"
    torch.save({"config": config, "model": sd}, path)
    return str(path), sd


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("fixture", ["npc_ref", "npc_ref_c2", "npc_ref_variant"])
def test_matches_reference_golden(s3b_lib, tmp_path, fixture, scheme):
    g = torch.load(GOLDEN / f"{fixture}.pt", weights_only=False)
    path, _ = _ckpt(tmp_path, g["paras"], g["weight_seed"])
    ex = _expert(scheme, ckpt=path)
    cs, ts = g["channel_stride"], g["time_stride"]
    for case in g["cases"]:
        wavs = [w.cuda() for w in _wavs(case["lens"], case["wav_seed"])]
        res = ex(wavs)
        assert tuple(res["_hidden_states_info"]) == tuple(case["names"])
        hs = res["hidden_states"]
        assert len(hs) == case["num_hidden"] and tuple(hs[0].shape) == tuple(case["shape"])
        for l, h in enumerate(hs):
            err = _rel(h[:, (h.shape[1] - 1) % ts :: ts, ::cs].cpu(), case["sub"][l])
            print(f"npc {fixture} lens={case['lens']} scheme={scheme or 'default'} state {l}: abs max "
                  f"{h.abs().max().item():.3f}, relative error {err:.3e} (measured/bound {err / REL_TOL:.3f})")
            assert err < REL_TOL


_VARIANTS = [{}, {"activate": "tanh"}, {"residual": False}, {"batch_norm": False},
             {"n_blocks": 2, "kernel_size": 9, "mask_size": 3}, {"n_blocks": 1, "kernel_size": 7, "mask_size": 1}]


@pytest.mark.parametrize("scheme", [None, "bf16x3"])
@pytest.mark.parametrize("over", _VARIANTS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()) or "default")
def test_matches_oracle_ragged(s3b_lib, tmp_path, scheme, over):
    from s3prl_b200.upstream.npc import npc_config, validate_config

    path, sd = _ckpt(tmp_path, over, 2)
    paras = validate_config(npc_config(**over))
    ex = _expert(scheme, ckpt=path)
    lens = [48000, 560, 31234, 16001, 47999, 9000]
    wavs = _wavs(lens, seed=11)
    hs = ex([w.cuda() for w in wavs])["hidden_states"]
    ref, _ = NO.npc_forward(wavs, sd, paras)
    assert len(hs) == len(ref) == 2 * paras["n_blocks"] + 1
    for l, (h, r) in enumerate(zip(hs, ref)):
        err = _rel(h.cpu(), r)
        print(f"npc ragged {over or 'default'} scheme={scheme or 'default'} state {l}: abs max {r.abs().max().item():.3f}"
              f", relative error {err:.3e} (measured/bound {err / REL_TOL:.3f})")
        assert err < REL_TOL


def test_bit_identical_batch_shards_lanes_host_repeats(s3b_lib):
    ex = _expert(None)
    lens = [int(v) for v in torch.randint(560, 160000, (32,), generator=torch.Generator().manual_seed(3))]
    lens[5] = 160000
    wavs = [w.cuda() for w in _wavs(lens, seed=21)]
    full = torch.stack(ex(wavs)["hidden_states"]).clone()
    # an utterance alone, padded to the batch's max_len, vs inside the batch of 32
    ex.global_max_len = max(lens)
    for i in (0, 5, 17):
        alone = torch.stack(ex([wavs[i]])["hidden_states"])
        assert torch.equal(alone[:, 0], full[:, i]), i
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
    native = ex._native
    counts = []
    for i in range(10):
        c0 = native.lib.s3b_launch_count(native.handle)
        res = torch.stack(ex(wavs)["hidden_states"])
        counts.append(native.lib.s3b_launch_count(native.handle) - c0)
        assert torch.equal(res, full), f"call {i + 1} changed the result"
    assert len(set(counts)) == 1, counts
    # a long-lived model after calls of other shapes gives what a fresh one gives
    fresh = _expert(None)
    probe = wavs[3:9]
    assert torch.equal(torch.stack(ex(probe)["hidden_states"]), torch.stack(fresh(probe)["hidden_states"]))
    print(f"npc bit-identity: batch composition, shards, lanes 1/2, forward_host, 10 repeats ({counts[0]} launches "
          "each), long-lived vs fresh model")


def test_forward_ex_refusals_and_profile(s3b_lib):
    from s3prl_b200 import lib

    ex = _expert(None)
    native = ex._native
    wavs = [w.cuda() for w in _wavs([16000, 8000], seed=1)]
    T = ex.num_frames(16000)
    out = torch.empty(9, 2, T, 512, device="cuda")
    ptrs = (C.c_void_p * 2)(*[w.data_ptr() for w in wavs])
    for field in ("ffn_out", "last_residual"):
        opts = lib.S3BForwardOpts(**{field: out.data_ptr()})
        r = native.lib.s3b_forward_ex(native.handle, ptrs, (C.c_int64 * 2)(16000, 8000), 2, 16000,
                                      C.c_void_p(out.data_ptr()), _stream(), C.byref(opts))
        assert r != 0 and field.encode() in native.lib.s3b_last_error()
    with pytest.raises(ValueError, match="560"):
        ex([torch.zeros(559, device="cuda")])
    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    ex(wavs)
    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
    lib.check(native.lib.s3b_profile_read_ex(native.handle, 6, ms, fl, n, 1))
    lib.check(native.lib.s3b_profile_enable(native.handle, 0))
    assert list(n) == [12, 0, 2, 0, 0, 0], list(n)  # 3 GEMMs per block at 4 blocks, fbank + CMVN
    # FLOPs with the unpadded 80 channels and the unmasked taps only: 8 + 6 + 4 + 2 of the 15 taps
    M = 2 * T
    want = 2.0 * M * 512 * (80 * 3 + 3 * 512 * 3 + 4 * 512 + 512 * (8 + 6 + 4 + 2))
    assert abs(fl[0] / want - 1) < 1e-12, (fl[0], want)
    print(f"npc profile ms: gemm {ms[0]:.3f} front end {ms[2]:.3f}")


def test_finalize_refuses_a_conv_mask_that_is_not_the_configs(s3b_lib):
    from s3prl_b200 import lib
    from s3prl_b200.upstream.npc import NpcExpert

    ex = NpcExpert()
    ex._state_dict_host["masked_convs.2.conv_mask"] = torch.ones(512, 512, 15)  # nothing masked
    with pytest.raises(lib.S3BError, match=r"masked_convs\.2\."):
        ex.to("cuda")([torch.randn(16000, device="cuda")])
