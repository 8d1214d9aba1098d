"""The 128-bin fbank front ends of SSAST and MAE-AST per element against fp64, on structured audio, with every operand
plane read raw.

MAE-AST (mae_ast_fbank_kernel, as add_mae_ast_input launches it): kaldi fbank with the povey window and 128 bins, then
y = fma(log-mel, a, c), the eval batch norm times 0.5 folded by model.cu's mae_ast_bn_fold, stored at its unfolded
(token, column) position of the projection's operand. At every configuration (MAE_CONFIGS: frame | patch, operand
format 0 bf16 hi/lo | 1 f16q8) and batch-norm pair (BN_PAIRS), for every utterance of the corpus:
  y      : the fp32 output (s3b_mae_ast_fbank_f32) inside spectral_ref.mae_ast_bounds' interval (the fp64 log-mel
           interval through the fold: a64 df + |a32 - a64| |f| + |c32 - c64| + u |y|), compared after MO.unfold of the
           reference, so a misplaced element is orders of magnitude out; "y" over the energies the bound resolves,
           "y_floor" over those whose interval reaches the max(E, eps) floor. Where the fp64 energy sits above the
           floor by far more than the floor's own rounding margin and the kernel clamps to the floor (which the
           interval accepts), that ratio approaches 1 by construction; the floor value itself is pinned by bin 3
           (MAE-AST) and the silent windows (SSAST).
  padding: frames in [n_b, T' kt) exactly fp32 c; frames from T' kt on are not written (NaN guard rows stay NaN).
  bin 3  : the 128-bin bank's empty bin holds one value, bit for bit, in every computed frame of every utterance.
  planes : s3b_mae_ast_fbank_planes' raw planes (the forward's constants) are bit for bit the format's split of the fp32
           output: both bf16 planes, or the fp16, the e4m3 of the fp16 (the A_hi of the correction MMA, which decoding
           never reads) and the e4m3 of the residual; the bytes after the last plane stay 0xFF.
SSAST (ssast_fbank_kernel, then ssast_patches_kernel as add_ssast_frontend launches them), at every window length S of
test_ssast_blocks_gpu.SSAST_WINDOWS, the corpus cut into windows:
  y      : each window's normalised log-mel inside spectral_ref.ssast_bounds' interval on that zero-padded window
           ((f + 4.2677393) / 9.1379948, the sum and quotient rounded, the fp32 constants' error carried);
  silent : windows that start past an utterance's end hold one value, bit for bit, inside the floor's interval;
  rows   : rows m .. TL - 1 of every window exactly 0;
  planes : s3b_ssast_patch_planes' raw planes bit for bit the split of the kernel's own fp32 features, row for row
           (frame model) or through ssast_oracle.patch_operand's gather (patch model), at both formats.
The worst measured/bound per stage and input kind is printed (pytest -s)."""
import ctypes as C
import functools
import math
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import mae_ast_oracle as MO  # noqa: E402
import spectral_ref as R  # noqa: E402
import ssast_oracle as SO  # noqa: E402
from test_fbank_frontend_gpu import _bits, batches, split_planes  # noqa: E402
from test_spectral_gpu import Worst  # noqa: E402
from test_ssast_blocks_gpu import SSAST_WINDOWS  # noqa: E402

from s3prl_b200 import lib as L  # noqa: E402
from s3prl_b200.upstream import mae_ast, ssast  # noqa: E402

NMEL = 128
# (window, mel bins, normalisation, operand layout (the expert module's KINDS entry), operand format) of the front end
# a served model runs; the coverage guard (test_kernel_coverage_cpu) forms the served set from the hub entries
MAE_AST_NORM = "eval batch norm x 0.5"
SSAST_NORM = "(f + 4.2677393) / 9.1379948"
MAE_KINDS = [(kind, fmt) for kind in mae_ast.KINDS for fmt in (0, 1)]
MAE_CONFIGS = [("povey", NMEL, MAE_AST_NORM, mae_ast.KINDS[k], fmt) for k, fmt in MAE_KINDS]
SSAST_KINDS = [(kind, fmt) for kind in ssast.KINDS for fmt in (0, 1)]
SSAST_CONFIGS = [("hanning", NMEL, SSAST_NORM, ssast.KINDS[k], fmt) for k, fmt in SSAST_KINDS]
CONFIGS = MAE_CONFIGS + SSAST_CONFIGS
# (running_mean, running_var): the fabricated checkpoint's, a second moderate pair, and a small variance whose large
# a = 0.5 / sqrt(rv + 1e-5) (about 5) amplifies the log-mel's error
BN_PAIRS = [(-8.25, 12.5), (-7.5, 11.0), (-4.0, 0.01)]
WINDOW_S = sorted({ssast.geometry(w.kind, w.secs)["S"] for w in SSAST_WINDOWS})


def corpus():
    """Every utterance of test_fbank_frontend_gpu.batches(), as (kind, waveform)."""
    return [(kind, w) for items in batches().values() for kind, w in items]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptrs(dev):
    return (C.c_void_p * len(dev))(*[w.data_ptr() for w in dev])


def _unpack(raw, n, fmt, shape):
    if fmt == 0:
        planes = (raw[:2 * n].view(torch.bfloat16), raw[2 * n:4 * n].view(torch.bfloat16))
    else:
        planes = (raw[:2 * n].view(torch.float16), raw[2 * n:3 * n].view(torch.float8_e4m3fn),
                  raw[3 * n:4 * n].view(torch.float8_e4m3fn))
    return tuple(p.view(shape) for p in planes)


def _assert_planes(planes, y, fmt, what):
    for i, (p, e) in enumerate(zip(planes, split_planes(y, fmt))):
        bad = (_bits(p) != _bits(e)).nonzero()
        assert len(bad) == 0, (f"{what}: plane {i}: {len(bad)} elements differ from the split of the fp32 value, first "
                               f"{bad[0].tolist()}")


# ---- MAE-AST ----------------------------------------------------------------------------------------------------------
def mae_batches(kind):
    """batches(), a batch whose longest utterance has fewer samples than one patch of kind joined with a 2800-sample
    chirp (16 frames, one patch model patch)."""
    out = {}
    for name, items in batches().items():
        if max(len(w) for _, w in items) < mae_ast.min_batch_samples(kind):
            items = items + [("chirp_n2800", R.structured_wav("chirp", 2800))]
        out[name] = items
    return out


@functools.lru_cache(maxsize=None)
def _mae_refs(rm, rv):
    """(batch name, index) -> mae_ast_bounds of every utterance of mae_batches("patch"), which holds every batch of
    mae_batches("frame") as its leading utterances."""
    eps_w = R.bank_eps("kaldi", NMEL)
    return {(name, i): R.mae_ast_bounds(w, eps_w, rm, rv)
            for name, items in mae_batches("patch").items() for i, (_, w) in enumerate(items)}


def run_mae(lib, wavs, kind, rm, rv, fmt, guard=8):
    """(fp32 output [B, T' nv, 256] with `guard` NaN rows after it, raw planes, the raw buffer's guard bytes)."""
    lens = [len(w) for w in wavs]
    B, Lm = len(wavs), max(lens)
    N = mae_ast.num_frames(kind, Lm) * (NMEL // mae_ast.KINDS[kind][1])
    n = B * N * 256
    dev = [w.cuda() for w in wavs]
    out = torch.full((n + guard * 256,), float("nan"), device="cuda")
    raw = torch.full((4 * n + 64,), 0xFF, dtype=torch.uint8, device="cuda")
    c_lens = (C.c_int64 * B)(*lens)
    L.check(lib.s3b_mae_ast_fbank_f32(_ptrs(dev), c_lens, B, Lm, int(kind == "patch"), rm, rv, fmt,
                                      C.c_void_p(out.data_ptr()), None, _stream()))
    L.check(lib.s3b_mae_ast_fbank_planes(_ptrs(dev), c_lens, B, Lm, int(kind == "patch"), rm, rv, fmt,
                                         C.c_void_p(raw.data_ptr()), _stream()))
    torch.cuda.synchronize()
    out, raw = out.cpu(), raw.cpu()
    return out[:n].view(B, N, 256), out[n:], _unpack(raw, n, fmt, (B, N, 256)), raw[4 * n:]


def _frames(v, F, fill):
    """[m, 128] -> [F, 128]: the first min(m, F) frames, `fill` after."""
    out = torch.full((F, NMEL), fill, dtype=v.dtype)
    k = min(len(v), F)
    out[:k] = v[:k]
    return out


def check_mae_batch(lib, kind, fmt, rm, rv, name, items, worst, floor_bits):
    wavs = [w for _, w in items]
    y32, guard, planes, raw_guard = run_mae(lib, wavs, kind, rm, rv, fmt)
    assert torch.isfinite(y32).all(), f"{name}: output not finite"
    assert torch.isnan(guard).all(), f"{name}: rows past T' kt written"
    assert (raw_guard == 0xFF).all(), f"{name}: bytes past the last plane written"
    _assert_planes(planes, y32, fmt, f"{name} {kind} fmt {fmt}")
    kt = mae_ast.KINDS[kind][0]
    Fp = y32.shape[1] // (NMEL // mae_ast.KINDS[kind][1]) * kt  # T' kt frames
    _, _, _, c32 = R.bn_fold(rm, rv)
    refs = _mae_refs(rm, rv)
    bin3 = torch.zeros(Fp, NMEL, dtype=torch.bool)
    bin3[:, 3] = True
    for b, (ukind, w) in enumerate(items):
        s = refs[(name, b)]
        m = R.num_frames(len(w))
        unf = lambda v, fill: MO.unfold(_frames(v, Fp, fill)[None], kind)[0]  # noqa: E731
        pad = unf(torch.zeros(m, NMEL, dtype=torch.bool), True)
        got = y32[b]
        assert torch.all(got[pad] == c32), f"{name} {ukind}: padded frames not exactly fp32 c = {c32}"
        y, lo, hi = unf(s["y"], 0.0), unf(s["ylo"], 0.0), unf(s["yhi"], 0.0)
        resolved = unf(s["E"] - s["dE"] > R.FLOOR, False)
        ratio = R.interval_ratio(got, y, lo, hi)
        worst.add("y", ukind, ratio[resolved & ~pad])
        worst.add("y_floor", ukind, ratio[~resolved & ~pad])
        empty = MO.unfold(bin3[None], kind)[0] & ~pad
        floor_bits.update(got[empty].view(torch.int32).unique().tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("bn", BN_PAIRS, ids=[f"rm{rm:g}-rv{rv:g}" for rm, rv in BN_PAIRS])
@pytest.mark.parametrize("config", MAE_KINDS, ids=[f"{k}-fmt{f}" for k, f in MAE_KINDS])
def test_mae_ast_frontend_against_fp64(s3b_lib, config, bn):
    kind, fmt = config
    rm, rv = bn
    worst = Worst(f"MAE-AST {kind} front end fmt {fmt} rm {rm:g} rv {rv:g} vs fp64")
    floor_bits = set()
    for name, items in mae_batches(kind).items():
        check_mae_batch(s3b_lib, kind, fmt, rm, rv, name, items, worst, floor_bits)
    assert len(floor_bits) == 1, f"bin 3 holds {len(floor_bits)} values"
    v = torch.tensor([floor_bits.pop()], dtype=torch.int32).view(torch.float32).item()
    a, c, _, _ = R.bn_fold(rm, rv)
    y64 = a * math.log(R.FLOOR) + c
    ulp = 2.0 ** (math.floor(math.log2(abs(y64))) - 23)
    print(f"\nbin 3 (empty): {v!r} in every computed frame, {abs(v - y64) / ulp:.2f} ulp from fp64 {y64!r}")
    worst.report()


# ---- SSAST ------------------------------------------------------------------------------------------------------------
def run_ssast_fbank(lib, wavs, S):
    """s3b_ssast_fbank_f32 into a NaN-poisoned buffer: [B * nseg, TL, 128]."""
    lens = [len(w) for w in wavs]
    B, Lm = len(wavs), max(lens)
    nseg, TL = -(-Lm // S), S // R.SHIFT
    dev = [w.cuda() for w in wavs]
    out = torch.full((B * nseg, TL, NMEL), float("nan"), device="cuda")
    L.check(lib.s3b_ssast_fbank_f32(_ptrs(dev), (C.c_int64 * B)(*lens), B, Lm, S, C.c_void_p(out.data_ptr()),
                                    _stream()))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("S", WINDOW_S)
def test_ssast_fbank_against_fp64(s3b_lib, S):
    eps_w = R.bank_eps("kaldi", NMEL)
    floor = math.log(R.FLOOR)
    flo, fhi = R.ssast_interval(torch.tensor(floor - 2 * R.U * abs(floor), dtype=torch.float64),
                                torch.tensor(floor + 2 * R.U * abs(floor), dtype=torch.float64))
    floor_y = (floor + R.SSAST_SHIFT) / R.SSAST_SCALE
    worst = Worst(f"SSAST fbank S={S} vs fp64")
    m = R.num_frames(S)
    silent_bits = set()
    for name, items in batches().items():
        wavs = [w for _, w in items]
        got = run_ssast_fbank(s3b_lib, wavs, S)
        assert torch.isfinite(got).all(), f"{name}: features not finite"
        nseg = got.shape[0] // len(wavs)
        assert torch.count_nonzero(got[:, m:]) == 0 and not torch.isnan(got[:, m:]).any(), f"{name}: appended rows"
        for b, (kind, w) in enumerate(items):
            x = torch.zeros(nseg * S)
            x[:len(w)] = w
            for sg in range(nseg):
                g = got[b * nseg + sg, :m].double()
                if sg * S >= len(w):
                    silent_bits.update(got[b * nseg + sg, :m].view(torch.int32).unique().tolist())
                    worst.add("silent", kind, R.interval_ratio(g, torch.full_like(g, floor_y), flo, fhi))
                    continue
                s = R.ssast_bounds(x[sg * S:(sg + 1) * S], eps_w)
                ratio = R.interval_ratio(g, s["y"], s["ylo"], s["yhi"])
                resolved = s["E"] - s["dE"] > R.FLOOR
                worst.add("y", kind, ratio[resolved])
                worst.add("y_floor", kind, ratio[~resolved])
    assert len(silent_bits) <= 1, f"silent windows hold {len(silent_bits)} values"
    worst.report()


@functools.lru_cache(maxsize=4)
def _ssast_features(lib, S):
    return run_ssast_fbank(lib, [w for _, w in batches()["kinds"]], S)


@pytest.mark.gpu
@pytest.mark.parametrize("config", SSAST_KINDS, ids=[f"{k}-fmt{f}" for k, f in SSAST_KINDS])
def test_ssast_patch_planes_are_the_split_of_the_features(s3b_lib, config):
    """At every window of the kind: the raw operand planes s3b_ssast_patch_planes writes from the fbank kernel's own
    fp32 features, bit for bit the format's split of those features (frame model: row for row; patch model: through
    ssast_oracle.patch_operand's gather); the bytes after the last plane stay 0xFF."""
    kind, fmt = config
    for win in [w for w in SSAST_WINDOWS if w.kind == kind]:
        geo = ssast.geometry(kind, win.secs)
        feat = _ssast_features(s3b_lib, geo["S"])
        SB, TL = feat.shape[0], feat.shape[1]
        A = feat if kind == "frame" else SO.patch_operand(feat, "patch").contiguous()
        n = A.numel()
        raw = torch.full((4 * n + 64,), 0xFF, dtype=torch.uint8, device="cuda")
        fd = feat.cuda()
        L.check(s3b_lib.s3b_ssast_patch_planes(C.c_void_p(fd.data_ptr()), SB, TL, int(kind == "patch"), fmt,
                                               C.c_void_p(raw.data_ptr()), _stream()))
        torch.cuda.synchronize()
        raw = raw.cpu()
        assert (raw[4 * n:] == 0xFF).all(), f"{win}: bytes past the last plane written"
        _assert_planes(_unpack(raw, n, fmt, tuple(A.shape)), A, fmt, f"ssast {kind} {win.secs:g} s fmt {fmt}")
        print(f"ssast {kind} {win.secs:g} s (S={geo['S']}, TL={TL}) fmt {fmt}: {n} operand elements bit for bit")


def test_planes_entry_points_reject_bad_arguments(s3b_lib):
    """Checked before any device work."""
    dummy = torch.zeros(4)
    buf = C.c_void_p(dummy.data_ptr())
    ptrs = (C.c_void_p * 1)(dummy.data_ptr())
    lens = (C.c_int64 * 1)(16000)

    def refused(text, fn, *args):
        with pytest.raises(L.S3BError, match=text):
            L.check(fn(*args))

    mp, sp = s3b_lib.s3b_mae_ast_fbank_planes, s3b_lib.s3b_ssast_patch_planes
    refused("null argument", mp, ptrs, lens, 1, 16000, 0, 0.0, 1.0, 0, None, None)
    refused("4-byte aligned", mp, ptrs, lens, 1, 16000, 0, 0.0, 1.0, 0, C.c_void_p(dummy.data_ptr() + 2), None)
    refused("fmt must be 0", mp, ptrs, lens, 1, 16000, 0, 0.0, 1.0, 2, buf, None)
    refused("patch must be 0 or 1", mp, ptrs, lens, 1, 16000, 2, 0.0, 1.0, 0, buf, None)
    refused("out of range", mp, ptrs, (C.c_int64 * 1)(399), 1, 16000, 0, 0.0, 1.0, 0, buf, None)
    refused("null argument", sp, buf, 1, 100, 0, 0, None, None)
    refused("4-byte aligned", sp, buf, 1, 100, 0, 0, C.c_void_p(dummy.data_ptr() + 2), None)
    refused("fmt must be 0", sp, buf, 1, 100, 0, 2, buf, None)
    refused("patch must be 0 or 1", sp, buf, 1, 100, 2, 0, buf, None)
    refused("bad sizes", sp, buf, 1, 15, 1, 0, buf, None)
