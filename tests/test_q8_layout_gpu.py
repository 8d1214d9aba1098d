"""GPU tests of the f16q8 operand's interleaved e4m3 plane (common.cuh: q8_off), where its layout meets the GEMM and the
C ABI: column slices of A on and off the 64-element k-block grid, partial last row tiles, every cluster size, and the
back-to-back plane layout the *_planes entry points document."""
import ctypes as C
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from s3prl_b200 import lib

    return lib


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _linear(a, w, b, M, N, K, **opts):
    lib = _lib()
    o = lib.S3BLinearOpts(scheme=1, **opts)
    out = torch.full((M, N), float("nan"), device="cuda")
    lib.check(lib.load().s3b_linear_ex(_ptr(a), _ptr(w), _ptr(b), None, M, N, K, 0, C.byref(o), _ptr(out), _stream()))
    torch.cuda.synchronize()
    assert o.scheme_used == 1
    return out


def _near_fp64(out, a, w, b):
    """Within f16q8's error of fp64. On these N(0, 1)-scaled operands the emulated f16q8 product is about 7e-6 off
    (relative Frobenius) and the fp16 product alone about 2e-4: a correction pass that adds nothing fails by 10x."""
    ref = a.double() @ w.double().T + b.double()
    rel = ((out.double() - ref).norm() / ref.norm()).item()
    assert rel < 2e-5, rel


@pytest.mark.parametrize("lda,a_off", [(3 * 768, 768), (1088, 64), (1088, 320), (1040, 16), (1024, 32), (800, 16)],
                         ids=["64_distiller", "64_a", "64_b", "16_a", "32", "16_b"])
def test_linear_slice(s3b_lib, lda, a_off):
    """f16q8 on the K-column slice at a_off of rows lda apart: on the 64-element grid the GEMM reads the q8 plane in
    place, off it the slice is split as dense rows. Either way bit for bit the dense slice; NaN outside the slice."""
    M, N, K = 499, 768, 768
    g = torch.Generator(device="cuda").manual_seed(lda + a_off)
    h = torch.full((M, lda), float("nan"), device="cuda")
    h[:, a_off:a_off + K] = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K**0.5
    b = torch.randn(N, device="cuda", generator=g)
    out = _linear(h, w, b, M, N, K, lda=lda, a_off=a_off)
    a = h[:, a_off:a_off + K].contiguous()
    assert torch.equal(out, _linear(a, w, b, M, N, K))
    _near_fp64(out, a, w, b)


@pytest.mark.parametrize("M", [499, 7984])
def test_clusters_bit_identical(s3b_lib, M):
    """Partial last row tiles at every cluster size: 128-wide tiles alone and in clusters of 2 and 4 that multicast
    the A boxes, the 256-wide cooperative kernel too; all bit for bit the same."""
    N, K = 1024, 768
    g = torch.Generator(device="cuda").manual_seed(M)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K**0.5
    b = torch.randn(N, device="cuda", generator=g)
    saved = os.environ.get("S3B_GEMM_CLUSTER")
    outs = {}
    try:
        for cn in ("1", "2", "4"):
            os.environ["S3B_GEMM_CLUSTER"] = cn
            outs[cn] = _linear(a, w, b, M, N, K, tile_n=128)
    finally:
        if saved is None:
            os.environ.pop("S3B_GEMM_CLUSTER", None)
        else:
            os.environ["S3B_GEMM_CLUSTER"] = saved
    outs["256"] = _linear(a, w, b, M, N, K, tile_n=256)
    for k, v in outs.items():
        assert torch.equal(v, outs["1"]), f"{k} differs from unclustered 128-wide tiles"
    _near_fp64(outs["1"], a, w, b)


# ---- the *_planes entry points: [fp16 | e4m3 of the fp16 | e4m3 of the residual x 2^11], one plane after another --
def _check_f16q8_planes(raw, n, y=None, y_approx=None):
    """raw: the entry point's bytes for n elements (fmt 1). y: the fp32 values (the planes must be their split bit for
    bit); y_approx: values within 2^-16 relative of them (the decode must be within the format's error)."""
    p16 = raw[:2 * n].view(torch.float16)
    h8 = raw[2 * n:3 * n]
    l8 = raw[3 * n:4 * n]
    assert torch.equal(h8, p16.float().clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)), "h8 != e4m3(fp16)"
    if y is not None:
        x16 = y.half()
        assert torch.equal(p16, x16), "fp16 plane"
        r = ((y - x16.float()) * 2.0**11).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8)
        assert torch.equal(l8, r), "l8 plane"
    if y_approx is not None:
        dec = p16.double() + l8.view(torch.float8_e4m3fn).double() * 2.0**-11
        err = (dec - y_approx.double()).abs()
        bound = 2.0**-14 * y_approx.double().abs() + 2.0**-20
        assert (err <= bound).all(), f"{int((err > bound).sum())} of {n} elements off"


def _wavs(B, n0):
    g = torch.Generator().manual_seed(B + n0)
    wavs = [torch.randn(n0 + 3217 * i, generator=g) * 0.1 for i in range(B)]
    dev = [w.cuda() for w in wavs]
    ptrs = (C.c_void_p * B)(*[w.data_ptr() for w in dev])
    lens = (C.c_int64 * B)(*[len(w) for w in wavs])
    return dev, ptrs, lens, max(len(w) for w in wavs)


def test_mae_ast_fbank_planes(s3b_lib):
    lib = _lib()
    L = lib.load()
    dev, ptrs, lens, Lm = _wavs(2, 16000)
    B, rm, rv = 2, -4.27, 4.57
    for patch in (0, 1):
        out = torch.full((1 << 22,), float("nan"), device="cuda")
        lib.check(L.s3b_mae_ast_fbank_f32(ptrs, lens, B, Lm, patch, rm, rv, 1, _ptr(out), None, _stream()))
        torch.cuda.synchronize()
        n = int((~torch.isnan(out)).sum())
        raw = torch.full((4 * n + 64,), 0xFF, dtype=torch.uint8, device="cuda")
        lib.check(L.s3b_mae_ast_fbank_planes(ptrs, lens, B, Lm, patch, rm, rv, 1, _ptr(raw), _stream()))
        torch.cuda.synchronize()
        assert (raw[4 * n:] == 0xFF).all(), "bytes past the last plane written"
        _check_f16q8_planes(raw[:4 * n], n, y=out[:n])


def test_ssast_patch_planes(s3b_lib):
    """The frame model's operand, which is the features row for row. Features that bf16 holds exactly: the bf16x3
    planes then give the values themselves (lo = 0)."""
    lib = _lib()
    L = lib.load()
    patch = 0
    for SB, TL in ((2, 64), (3, 100)):
        g = torch.Generator(device="cuda").manual_seed(TL)
        feat = torch.randn(SB, TL, 128, device="cuda", generator=g).bfloat16().float()
        n = SB * TL * 128
        raws = []
        for fmt in (0, 1):
            raw = torch.full((4 * n + 64,), 0xFF, dtype=torch.uint8, device="cuda")
            lib.check(L.s3b_ssast_patch_planes(_ptr(feat), SB, TL, patch, fmt, _ptr(raw), _stream()))
            torch.cuda.synchronize()
            assert (raw[4 * n:] == 0xFF).all(), "bytes past the last plane written"
            raws.append(raw[:4 * n])
        hi, lo = raws[0][:2 * n].view(torch.bfloat16), raws[0][2 * n:].view(torch.bfloat16)
        assert (lo == 0).all()
        _check_f16q8_planes(raws[1], n, y=hi.float())


def test_fbank_cmvn_planes(s3b_lib):
    """The f16q8 planes against the bf16x3 planes of the same call (hi + lo: within 2^-16 relative of the values)."""
    lib = _lib()
    L = lib.load()
    dev, ptrs, lens, Lm = _wavs(3, 8000)
    B = 3
    for step in (1, 2):
        raws = []
        for fmt in (0, 1):
            logmel = torch.empty(1 << 20, device="cuda")
            raw = torch.full((1 << 22,), 0xFF, dtype=torch.uint8, device="cuda")
            lib.check(L.s3b_fbank_cmvn_planes(ptrs, lens, B, step, fmt, _ptr(logmel), _ptr(raw), _stream()))
            torch.cuda.synchronize()
            raws.append(raw)
        frames = 1 + (Lm - 400) // 160
        n = B * (frames if step == 1 else (frames + 1) // 2) * 128  # [B][T][128]
        assert (raws[1][4 * n:] == 0xFF).all(), "bytes past the last plane written"
        y0 = raws[0][:2 * n].view(torch.bfloat16).double() + raws[0][2 * n:4 * n].view(torch.bfloat16).double()
        _check_f16q8_planes(raws[1][:4 * n], n, y_approx=y0)
