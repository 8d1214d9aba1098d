"""GPU tests of resource lifetime: models and building-block calls created and released over and over.

Each test runs its cycles in a child process (this file run as a script), so that the device memory NVML reports for
that process holds only what the cycles allocate. Model cycles: every model kind the runtime distinguishes (post-LN
transformer, WavLM with its relative-position table, Conformer, distiller with prediction heads, DeCoAR 2.0, APC,
DeCoAR) is created, finalized, run (two lanes where the model allows it, ``forward_host``, a profiled forward whose
profile is read, then one left unread) and destroyed, three times; every cycle's hidden states must equal the first
cycle's bit for bit. Block cycles: every block-level entry point that stages buffers of its own is called repeatedly.
Either way the process's device memory after the last cycle may exceed that after the first by at most MEM_SLACK_MIB.
Where NVML does not list the process (a PID namespace it cannot see into), the memory check is reported as not made;
device-wide free memory is no substitute on a shared device."""
import ctypes as C
import gc
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]

pytestmark = pytest.mark.gpu

MEM_SLACK_MIB = 4.0
MODEL_CYCLES = 3
BLOCK_CYCLES = 5
LENS = (24000, 16000, 9000, 20000)


def _process_mib():
    """Device memory NVML attributes to this process, in MiB, over all devices; None when NVML does not list it."""
    try:
        import pynvml

        pynvml.nvmlInit()
    except Exception:
        return None
    try:
        pid, total, seen = os.getpid(), 0, False
        for i in range(pynvml.nvmlDeviceGetCount()):
            for p in pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(i)):
                if p.pid == pid and p.usedGpuMemory is not None:
                    total, seen = total + p.usedGpuMemory, True
        return total / 2**20 if seen else None
    except pynvml.NVMLError:
        return None
    finally:
        pynvml.nvmlShutdown()


def _settled_mib():
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()  # torch's cached blocks are not the library's
    return _process_mib()


def _report_memory(what, first, last):
    if first is None or last is None:
        print(f"{what}: memory check not made (NVML does not list this process)")
        return
    print(f"{what}: process device memory {first:.1f} MiB after the first cycle, {last:.1f} MiB after the last")
    assert last - first <= MEM_SLACK_MIB, (what, first, last)


# ------------------------------------------------------------------------------------------------
# model cycles
# ------------------------------------------------------------------------------------------------
def _make(kind):
    from s3prl_b200.upstream.apc import ApcExpert
    from s3prl_b200.upstream.decoar import DecoarExpert
    from s3prl_b200.upstream.decoar2 import Decoar2Expert
    from s3prl_b200.upstream.expert import UpstreamExpert

    if kind == "decoar2":
        return Decoar2Expert()
    if kind == "apc":
        return ApcExpert()
    if kind == "decoar":
        return DecoarExpert(all_layers=True)
    return UpstreamExpert(name=kind, seed=0)


MODEL_KINDS = ["hubert_base", "wavlm_base_plus", "wav2vec2_conformer_rope", "distilhubert_base", "decoar2", "apc",
               "decoar"]


def _model_cycle(kind, host):
    """create -> finalize -> forwards -> destroy; the hidden states of each forward, on the host."""
    from s3prl_b200 import lib

    ex = _make(kind).to("cuda")
    wavs = [w.cuda() for w in host]
    ex.lanes = 2
    outs = [torch.stack(ex(wavs)["hidden_states"]).cpu()]
    ex.lanes = 0
    outs.append(ex.forward_host(host).clone())
    native = ex._native
    lib.check(native.lib.s3b_profile_enable(native.handle, 1))
    outs.append(torch.stack(ex(wavs)["hidden_states"]).cpu())
    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
    lib.check(native.lib.s3b_profile_read_ex(native.handle, 6, ms, fl, n, 1))
    assert sum(n) > 0, (kind, list(n))
    ex(wavs)  # timing events recorded and never read: the model releases them
    native.close()
    del ex, native, wavs
    return outs


def _run_models():
    g = torch.Generator().manual_seed(11)
    host = [torch.randn(n, generator=g) for n in LENS]
    first, mem = {}, []
    for cycle in range(MODEL_CYCLES):
        for kind in MODEL_KINDS:
            outs = _model_cycle(kind, host)
            if cycle == 0:
                first[kind] = outs
            else:
                for i, (a, b) in enumerate(zip(outs, first[kind])):
                    assert torch.equal(a, b), f"{kind}: output {i} of cycle {cycle} differs from cycle 0"
        mem.append(_settled_mib())
        print(f"model cycle {cycle} done")
    _report_memory("model cycles", mem[0], mem[-1])


# ------------------------------------------------------------------------------------------------
# block cycles
# ------------------------------------------------------------------------------------------------
def _block_calls(so, g):
    """One call of each block-level entry point that allocates buffers of its own, at a small shape, through the
    argument builders of the block tests."""
    import test_apc_gpu as APC
    import test_blocks_gpu as BLK
    import test_conformer_gpu as CONF
    import test_decoar_gpu as DEC
    import test_frontend_gpu as FE
    import test_gemm_layouts_gpu as GL
    from s3prl_b200 import lib as L

    def rnd(*shape, s=1.0):
        return torch.randn(*shape, device="cuda", generator=g) * s

    ptr, st = GL._ptr, GL._stream
    a, w = rnd(256, 512), rnd(768, 512, s=512**-0.5)
    GL._linear(a, w, rnd(768))
    GL._linear(a, w, None, out_fmt=1)
    GL._conv(rnd(2, 65, 512), rnd(512, 512, 3, s=1536**-0.5), rnd(512), 65, 3, True, -1, 1)
    x, pw, pb, _ = GL._pos_inputs(2, 40, 768, 16, 128, 3)
    GL._posconv(x, pw, pb, 16, 128, 4, 0)
    GL._posconv(x, pw, pb, 16, 128, 1, 0)

    B, T, H, hd = 2, 37, 4, 64
    D = H * hd
    q, k, vt = rnd(B, H, T, hd), rnd(B, H, T, hd), rnd(B, H, hd, (T + 7) // 8 * 8)
    L.check(so.s3b_qkv_hd_f32(ptr(rnd(B, T, D)), ptr(rnd(3 * D, D, s=D**-0.5)), ptr(rnd(3 * D)), B, T, H, hd, -1,
                              ptr(q), ptr(k), ptr(vt), st()))
    BLK._attention_ex(rnd(B, T, D), rnd(B, T, D), rnd(B, T, D), [T, 20], H)
    BLK._attention_ex(rnd(B, T, D), rnd(B, T, D), rnd(B, T, D), [T, 5], H, emb=rnd(BLK.NUM_BUCKETS, H),
                      gate=torch.rand(B, H, T, device="cuda", generator=g) + 0.5, table_frames=64, ctx_format=1)
    gate = torch.empty(B, H, T, device="cuda")
    L.check(so.s3b_wavlm_gate_f32(ptr(rnd(B, T, D)), B, T, H, ptr(rnd(8, 64, s=0.2)), ptr(rnd(8, s=0.2)),
                                  ptr(rnd(H, s=0.3) + 1), 1, ptr(gate), st()))
    bench = (C.c_float * 2)()
    L.check(so.s3b_gemm_bench(256, 768, 512, 1, 0, 2, bench))

    wavs = [rnd(n, s=0.1) for n in (16000, 9000)]
    FE._frontend(wavs, 16000, rnd(512, 10, s=0.3), rnd(512), rnd(512, s=0.1) + 1, rnd(512, s=0.1), 0, 1)
    FE._frontend(wavs, 16000, rnd(512, 10, s=0.3), rnd(512), rnd(512, s=0.1) + 1, rnd(512, s=0.1), 1, 0)
    ptrs = (C.c_void_p * 2)(*[t.data_ptr() for t in wavs])
    lens = (C.c_int64 * 2)(16000, 9000)
    feats = torch.empty(2, 99, 80, device="cuda")
    L.check(so.s3b_apc_features_f32(ptrs, lens, 2, 1, ptr(feats), st()))
    L.check(so.s3b_decoar2_features_f32(ptrs, lens, 2, 0, ptr(feats), st()))
    trimmed = (C.c_int64 * 2)()
    L.check(so.s3b_trimmed_lengths(ptrs, lens, 2, trimmed))

    APC._gru_block(so, rnd(3, 17, 1536), rnd(1536, 512, s=0.02), rnd(1536, s=0.1), None, [17, 5, 1], 1)
    hl = DEC.H
    DEC._lstm_block(so, [rnd(3, 9, 4 * hl)] * 2, [rnd(4 * hl, hl, s=0.2 / hl**0.5)] * 2, [None, rnd(4 * hl)],
                    [9, 4, 1], 0)
    CONF._conv_native(so, rnd(2, 33, 512), rnd(256, 1, 31, s=31**-0.5), *CONF._bn_params(256, g), 1)
    y, yr = torch.empty(2 * 33, 768, device="cuda"), torch.empty(2 * 33, 768, device="cuda")
    L.check(so.s3b_layernorm_rope_f32(ptr(rnd(2 * 33, 768)), 2 * 33, 33, 768, ptr(rnd(768, s=0.1) + 1),
                                      ptr(rnd(768, s=0.1)), None, 0, ptr(y), ptr(yr), st()))
    torch.cuda.synchronize()


def _run_blocks():
    from s3prl_b200 import lib

    so = lib.load()
    g = torch.Generator(device="cuda").manual_seed(5)
    mem = []
    for _ in range(BLOCK_CYCLES):
        _block_calls(so, g)
        mem.append(_settled_mib())
    print(f"{BLOCK_CYCLES} block cycles done")
    _report_memory("block cycles", mem[0], mem[-1])


# ------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------
def _child(what):
    r = subprocess.run([sys.executable, __file__, what], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    assert "memory check not made" in r.stdout or "process device memory" in r.stdout, r.stdout[-2000:]


def test_model_create_run_destroy_cycles(s3b_lib):
    _child("models")


def test_block_call_cycles(s3b_lib):
    _child("blocks")


if __name__ == "__main__":
    sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
    {"models": _run_models, "blocks": _run_blocks}[sys.argv[1]]()
