"""The fbank front end of APC, VQ-APC, DeCoAR, decoar_layers, DeCoAR 2.0 and NPC per element against fp64, on
structured audio.

add_fbank_frontend runs launch_decoar2_features: fbank_frames_kernel<true, 80> (kaldi fbank with the hamming window
and 80 mel bins, no deltas) into an fp32 log-mel buffer, then decoar2_cmvn_kernel: CMVN over each utterance's m frames
(two-pass fp64 statistics over 16 frame lanes x 16 bins, unbiased std, 1e-10 + std), rows t < ceil(m / step) take
frame step * t, written as the first GEMM's operand planes [B * T][128]. s3b_fbank_cmvn_planes runs that step into
buffers of the test, poisoned with NaN first. At every served configuration (CONFIGS: step 1 | 2, operand format
0 bf16 hi/lo | 1 f16q8) and for every utterance:
  logmel : the frame kernel's log-mel inside spectral_ref's [lo, hi] with the hamming window, split as in
           test_spectral_gpu: "logmel" over the energies the bound resolves, "logmel_edge" over those whose interval
           reaches the max(E, eps) floor. The FFT bound is absolute per frame, so a bin far below its frame's peak gets
           the wide interval its fp32 spectrum needs (the 2 u sqrt(E_frame / E_bin) effect SSAST's fbank showed).
  cmvn   : the kernel's fp32 CMVN value within spectral_ref.cmvn_bound over all m frames, on the columns it conditions
           (s >= 10 max df); the others get test_spectral_gpu.check_cmvn's structural checks. The kernel keeps that
           value only in the planes: emulate_cmvn reproduces it bit for bit from the kernel's own log-mel, and the
           planes check below pins the reproduction.
  planes : every plane is the format's split of that fp32 value, bit for bit (bf16 hi / lo as split_pack2; fp16,
           e4m3 of the fp16, e4m3 of the residual x 2^11 as split_q8_pack2, including the e4m3 plane of the fp16 values
           that decoding never reads); the decoded value against fp64 within dz plus the format's representation
           error (ratio "planes"); s3b_apc_features_f32 / s3b_decoar2_features_f32 decode the same values.
  padding: every plane byte of rows t >= ceil(m / step) and of columns 80..127 is zero; log-mel rows t >= m keep
           the poison (decoar2_cmvn_kernel must not read them).
The worst measured/bound per stage and input kind is printed (pytest -s)."""
import ctypes as C
import math
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import spectral_ref as R  # noqa: E402
from test_spectral_gpu import Worst, check_cmvn  # noqa: E402

from s3prl_b200 import lib as L  # noqa: E402

U = R.U
NMEL, K = 80, 128  # mel bins; operand columns of the first GEMM (kDecoar2K)
MIN_SAMPLES = 560  # two frames: the unbiased std of one frame is NaN

# (window, mel bins, step, CMVN variant, operand format) of the front end a served model runs; the coverage guard
# (test_kernel_coverage_cpu) forms the served set from the model kinds
CMVN_ALL_FRAMES = "all frames, unbiased std, 1e-10 + std"
CONFIGS = [("hamming", NMEL, step, CMVN_ALL_FRAMES, fmt) for step in (1, 2) for fmt in (0, 1)]


# ---- inputs -----------------------------------------------------------------------------------------------------------
def few_bins(n: int) -> torch.Tensor:
    """A stationary comb of 300, 1200 and 5000 Hz (multiples of 100 Hz: every 160-sample hop sees the same samples, so
    the bins it fills are nearly constant over time) under a 3050 Hz tone on for 0.2 s of every 0.5 s: the tone's bins
    vary, the comb's barely do, and CMVN divides those by a tiny std."""
    t = torch.arange(n, dtype=torch.float64) / R.SR
    x = sum(0.05 * torch.sin(2 * math.pi * f * t + 0.4 * k) for k, f in enumerate((300.0, 1200.0, 5000.0)))
    gate = ((torch.arange(n) % 8000) < 3200).double()
    return (x + 0.3 * gate * torch.sin(2 * math.pi * 3050.0 * t)).float()


def one_frame(n: int, at: int = 8100) -> torch.Tensor:
    """Digital silence except one sample: the frames that hold it (the two of 160 t <= at < 160 t + 400 here) are the
    only ones above the floor, so their CMVN values sit at the Samuelson bound (m - 1) / sqrt(m)."""
    x = torch.zeros(n)
    x[at] = 0.5
    return x


def batches():
    """name -> [(kind, waveform)]. "kinds": every structured_wav kind and with_tail tail, 21 utterances (grid.x > 16) in
    unsorted lengths; "edges": lengths on frame edges, m = 2..5 (ceil(m / 2) reached from odd and even m); "long":
    20.5 s next to the shortest utterance served, so most of the short one's rows are padding."""
    w, t = R.structured_wav, R.with_tail
    kinds = [("chirp", w("chirp", 16000)), ("tone_fbank_bin", w("tone_fbank_bin", 12001)),
             ("tone_fbank_half+zeros", t(w("tone_fbank_half", 9000), "zeros")), ("tone_25", w("tone_25", 4001)),
             ("tone_7990", w("tone_7990", 3999)), ("bursts", w("bursts", 16000)), ("pink", w("pink", 16001, seed=1)),
             ("brown", w("brown", 8000, seed=2)), ("dc", w("dc", 880, seed=3)), ("clipped", w("clipped", 7000)),
             ("int16", w("int16", 6000)), ("tiny", w("tiny", 6000, seed=4)), ("zeros", w("zeros", 2000)),
             ("white", w("white", 560, seed=5)), ("chirp+negzeros", t(w("chirp", 5000), "negzeros")),
             ("pink+first_only", t(w("pink", 3000, seed=6), "first_only")), ("impulses", w("impulses", 3999)),
             ("few_bins", few_bins(16000)), ("one_frame", one_frame(16000)), ("tone_stft_half", w("tone_stft_half", 721)),
             ("few_bins_short", few_bins(1200))]
    edge_kinds = ["chirp", "pink", "tone_fbank_half", "impulses", "brown", "dc", "int16", "bursts"]
    edge_lens = [720, 560, 1040, 719, 881, 561, 1039, 880]
    edges = [(f"{k}_n{n}", w(k, n, seed=10 + i)) for i, (k, n) in enumerate(zip(edge_kinds, edge_lens))]
    long = [("chirp_20s", w("chirp", 328000)), ("tone_fbank_half_n560", w("tone_fbank_half", 560))]
    return {"kinds": kinds, "edges": edges, "long": long}


@pytest.fixture(scope="module")
def refs():
    """name -> (kinds, waveforms, fbank_cmvn_bounds of every waveform at step 1)."""
    eps_w = R.bank_eps("kaldi")
    out = {}
    for name, items in batches().items():
        wavs = [x for _, x in items]
        out[name] = ([k for k, _ in items], wavs, [R.fbank_cmvn_bounds(x, eps_w, 1) for x in wavs])
    return out


# ---- the kernel's arithmetic, restated --------------------------------------------------------------------------------
def _lane_sums(v: torch.Tensor) -> torch.Tensor:
    """decoar2_cmvn_kernel's fp64 reduction of v [m, n] over dim 0: lane r sums rows r, r + 16, ... in order, then the
    16 lane sums are added in lane order."""
    m = v.shape[0]
    rows = torch.cat([v, v.new_zeros((-m) % 16, v.shape[1])]).view(-1, 16, v.shape[1])
    lanes = torch.zeros(16, v.shape[1], dtype=torch.float64)
    for r in rows:  # adding the +0.0 padding changes no sum
        lanes = lanes + r
    a = torch.zeros(v.shape[1], dtype=torch.float64)
    for r in lanes:
        a = a + r
    return a


def emulate_cmvn(f32: torch.Tensor, step: int) -> torch.Tensor:
    """decoar2_cmvn_kernel's fp32 output [ceil(m / step), n] from the fp32 log-mel f32 [m, n] it reads: mean =
    fp32(sum / m), d = fp32(x - mean), sd = fp32(sqrt(sum d^2 / (m - 1))) (fp32 products are exact in fp64),
    y = fp32(fp32(x - mean) / fp32(1e-10f + sd)); every step-th row."""
    m = f32.shape[0]
    mean = (_lane_sums(f32.double()) / m).float()
    d = f32 - mean
    sd = (_lane_sums(d.double() * d.double()) / (m - 1)).sqrt().float()
    den = torch.tensor(1e-10, dtype=torch.float32) + sd
    return (d / den)[::step]


def split_planes(y: torch.Tensor, fmt: int):
    """The planes store_planes2 writes for fp32 y: (bf16 hi, bf16 lo) or (fp16, e4m3 of the fp16, e4m3 of the
    residual x 2^11), e4m3 saturating as cvt.rn.satfinite."""
    e4m3 = lambda v: v.clamp(-448.0, 448.0).to(torch.float8_e4m3fn)  # noqa: E731
    if fmt == 0:
        hi = y.bfloat16()
        return hi, (y - hi.float()).bfloat16()
    h16 = y.half()
    return h16, e4m3(h16.float()), e4m3((y - h16.float()) * 2048.0)


def decode_planes(planes, fmt: int) -> torch.Tensor:
    """load_planes2: hi + lo in fp32, or fma(l8, 2^-11, h16) (the product is exact)."""
    if fmt == 0:
        return planes[0].float() + planes[1].float()
    return planes[0].float() + planes[2].float() * 2.0**-11


def representation_error(z: torch.Tensor, fmt: int) -> torch.Tensor:
    """|y - decode(split(y))| for |y| <= z: hi + lo keeps 16 bits (2^-16 |y|); fp16 keeps 11 and the e4m3 residual 4
    more (2^-15 |y|), with e4m3's subnormal step 2^-9 scaled by 2^-11 as a floor (half of it: 2^-21)."""
    return 2.0**-16 * z if fmt == 0 else 2.0**-15 * z + 2.0**-21


# ---- running the front end ----------------------------------------------------------------------------------------------
def _ptrs(wavs):
    return (C.c_void_p * len(wavs))(*[w.data_ptr() for w in wavs])


def run_frontend(lib, wavs, step, fmt):
    """(log-mel [B][m][80], planes, decoded [B][T][80]) of s3b_fbank_cmvn_planes into NaN-poisoned buffers (planes as a
    tuple of [B][T][128] tensors of the format's plane dtypes) and of the model's features entry point."""
    B, lens = len(wavs), [len(w) for w in wavs]
    mf = R.num_frames(max(lens))
    T = -(-mf // step)
    n = B * T * K
    dev = [w.cuda() for w in wavs]
    logmel = torch.full((B, mf, NMEL), float("nan"), device="cuda")
    raw = torch.full((4 * n,), 0xFF, dtype=torch.uint8, device="cuda")  # NaN in bf16, fp16 and e4m3
    decoded = torch.full((B, T, NMEL), float("nan"), device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    c_lens = (C.c_int64 * B)(*lens)
    L.check(lib.s3b_fbank_cmvn_planes(_ptrs(dev), c_lens, B, step, fmt, C.c_void_p(logmel.data_ptr()),
                                      C.c_void_p(raw.data_ptr()), st))
    entry = lib.s3b_apc_features_f32 if step == 1 else lib.s3b_decoar2_features_f32
    L.check(entry(_ptrs(dev), c_lens, B, fmt, C.c_void_p(decoded.data_ptr()), st))
    torch.cuda.synchronize()
    raw = raw.cpu()
    if fmt == 0:
        planes = (raw[:2 * n].view(torch.bfloat16), raw[2 * n:].view(torch.bfloat16))
    else:
        planes = (raw[:2 * n].view(torch.float16), raw[2 * n:3 * n].view(torch.float8_e4m3fn),
                  raw[3 * n:].view(torch.float8_e4m3fn))
    planes = tuple(p.view(B, T, K) for p in planes)
    return logmel.cpu(), planes, decoded.cpu()


def _bits(p: torch.Tensor) -> torch.Tensor:
    return p.view(torch.uint8 if p.element_size() == 1 else torch.int16)


def check_batch(lib, step, fmt, kinds, wavs, bounds, worst):
    logmel, planes, decoded = run_frontend(lib, wavs, step, fmt)
    T = planes[0].shape[1]
    dec = decode_planes(planes, fmt)
    assert torch.equal(dec[..., :NMEL], decoded), "the features entry point decodes other values than the planes hold"
    for p in planes:  # columns 80..127 of every row, in every plane
        assert torch.count_nonzero(_bits(p[..., NMEL:])) == 0, "operand columns 80..127 not zero"
    for b, (kind, w, s) in enumerate(zip(kinds, wavs, bounds)):
        m = R.num_frames(len(w))
        tb = -(-m // step)
        g = logmel[b, :m].double()
        assert torch.isnan(logmel[b, m:]).all(), f"{kind}: log-mel rows past m were written"
        ratio, resolved = R.interval_ratio(g, s["f"], s["lo"], s["hi"]), s["E"] - s["dE"] > R.FLOOR
        worst.add("logmel", kind, ratio[resolved])
        worst.add("logmel_edge", kind, ratio[~resolved])
        # the kernel's fp32 CMVN value, and the planes it is written as
        y32 = emulate_cmvn(logmel[b, :m], step)
        for p, e in zip(planes, split_planes(y32, fmt)):
            got, want = _bits(p[b, :tb, :NMEL]), _bits(e)
            bad = (got != want).nonzero()
            assert len(bad) == 0, (f"{kind}: {len(bad)} plane elements differ from the split of the kernel's fp32 "
                                   f"value, first (row, col) {bad[0].tolist()}")
        for p in planes:
            assert torch.count_nonzero(_bits(p[b, tb:])) == 0, f"{kind}: rows t >= ceil(m / step) not zero"
        z64, dz, cond = s["z"][::step], s["dz"][::step], s["cond"]
        check_cmvn(y32.double(), (z64, dz, cond), m, kind, worst)
        if kind == "zeros":  # every frame at the floor: the fp32 statistics are exact, every value 0
            assert torch.count_nonzero(y32) == 0
        got = dec[b, :tb, :NMEL].double()
        rep = representation_error(z64.abs() + dz, fmt)
        worst.add("planes", kind, ((got - z64).abs() / (dz + rep))[:, cond])
    return T


@pytest.mark.gpu
@pytest.mark.parametrize("config", CONFIGS, ids=[f"step{c[2]}-fmt{c[4]}" for c in CONFIGS])
def test_fbank_frontend_against_fp64(s3b_lib, refs, config):
    _, _, step, _, fmt = config
    worst = Worst(f"fbank front end step {step} fmt {fmt} vs fp64")
    for name, (kinds, wavs, bounds) in refs.items():
        T = check_batch(s3b_lib, step, fmt, kinds, wavs, bounds, worst)
        assert T == -(-R.num_frames(max(len(w) for w in wavs)) // step), name
    worst.report()


def test_fbank_cmvn_planes_rejects_bad_arguments(s3b_lib):
    """Checked before any device work. 400 and 559 samples make one frame, whose unbiased std is NaN: refused at both
    steps, whatever else the batch holds."""
    dummy = torch.zeros(4)
    ptrs = (C.c_void_p * 1)(dummy.data_ptr())
    lens = (C.c_int64 * 1)(16000)
    buf = C.c_void_p(dummy.data_ptr())

    def refused(text, *args):
        with pytest.raises(L.S3BError, match=text):
            L.check(s3b_lib.s3b_fbank_cmvn_planes(*args))

    pair = (C.c_void_p * 2)(dummy.data_ptr(), dummy.data_ptr())
    for step in (1, 2):
        for n in (400, 559):
            refused(f"lens\\[1\\] = {n}: .* needs >= {MIN_SAMPLES} samples", pair, (C.c_int64 * 2)(16000, n), 2, step,
                    0, buf, buf, None)

    refused("step must be 1", ptrs, lens, 1, 3, 0, buf, buf, None)
    refused("step must be 1", ptrs, lens, 1, 0, 0, buf, buf, None)
    refused("out_fmt must be 0", ptrs, lens, 1, 1, 2, buf, buf, None)
    refused("null argument", ptrs, lens, 1, 1, 0, None, buf, None)
    refused("null argument", ptrs, lens, 1, 1, 0, buf, None, None)
    refused("4-byte aligned", ptrs, lens, 1, 1, 0, buf, C.c_void_p(dummy.data_ptr() + 2), None)
    refused("bad batch", ptrs, lens, 0, 1, 0, buf, buf, None)
