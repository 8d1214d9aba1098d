"""A forward must not depend on the calls before it.

Every model keeps its activations in per-lane workspace buffers that only grow and are zeroed once, when they are
allocated; launch plans are cached per (batch, max_len); the bookkeeping block is rewritten only when it changes; the
WavLM and rotary tables are rebuilt when a longer batch arrives. So from the second call on a forward runs over
whatever the earlier calls left behind. The property tested here, for every model kind whose workspace or plan differs:

    the output of a forward on a long-lived model is bit-identical (torch.equal) to the output of the same inputs on
    a freshly created model that has run nothing else, whatever the long-lived model ran before.

Each test plays a scripted history twice. The first pass computes the reference of every probe on a fresh native model
(one ``lanes = 1`` device forward, kept on the host); the second pass runs the history on one long-lived model and
compares every probe. The passes are kept apart because every allocation of any model moves the process-wide
allocation generation that the plan cache is keyed by: a fresh model created between two calls of the long-lived one
would turn each of its plan-cache hits into a rebuild. Models are cut to two encoder layers where the family allows it.
The numerical correctness of a fresh model is pinned by the golden and oracle tests; nothing here has a tolerance.

The poison step feeds waveforms made of NaN, +-inf and 1e30 (the fbank kinds: of +-1e30 .. 3e30, see ``_poison``).
That is arithmetic on non-finite data, not a fault: no kernel derives a loop bound, an index or a branch target from
waveform values (frame counts, lengths, the row mask and the recurrences' length order all come from ``lens`` on the
host; the fbank, normalisation and GroupNorm statistics are plain reductions), so it is used for every kind.
"""
import ctypes as C
from dataclasses import replace

import pytest
import torch

pytestmark = pytest.mark.gpu

# (kind, operand scheme): hubert_base and apc in both schemes, the rest in the default
KINDS = [
    ("hubert_base", None),           # GroupNorm conv 0, post-LN, pos_conv four-taps path (pos_z)
    ("hubert_base", "bf16x3"),
    ("wav2vec2_large_ll60k", None),  # per-frame conv LayerNorm (conv_f32 sized by L[1]), pre-LN, last_residual
    ("wavlm_base_plus", None),       # relative-position table, gate buffer
    ("data2vec_base_960", None),     # five positional conv blocks through pos_z, combine modes 1 / 2
    ("distilhubert_base", None),     # hs0, prediction heads, SplitLinear slices
    ("wav2vec2_conformer_rope", None),  # glu_f32, rotary table
    ("xls_r_hd80", None),            # 80-wide heads, D = 1280: TMA zero fill past the head width
    ("decoar2", None),               # fbank front end, 80 -> 128 column padding
    ("apc", None),                   # GRU state, length order
    ("apc", "bf16x3"),
    ("decoar", None),                # LSTM state exchange buffer, grid barrier counter
]
FBANK = ("decoar2", "apc", "decoar")
RECURRENT = ("apc", "decoar")

# frame counts of the probes: Tp - T (Tp = T rounded up to 8) from 0 to 7, one partial 64-row query tile, one key block
PROBE_T = (2, 9, 15, 63, 64, 65, 129)


# ------------------------------------------------------------------------------------------------
# models and inputs
# ------------------------------------------------------------------------------------------------
def _build(kind):
    from s3prl_b200.upstream.apc import ApcExpert
    from s3prl_b200.upstream.configs import ARCHS, XLS_R
    from s3prl_b200.upstream.decoar import DecoarExpert
    from s3prl_b200.upstream.decoar2 import DECOAR2, NUM_MEL_BINS, Decoar2Expert
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    if kind == "apc":
        return ApcExpert()
    if kind == "decoar":
        return DecoarExpert(all_layers=True)
    if kind == "decoar2":
        cfg = replace(DECOAR2, encoder_layers=2)
        sd = {k: v for k, v in fabricate_state_dict(cfg, 0).items() if k.startswith("encoder.")}
        g = torch.Generator().manual_seed(0)
        sd["post_extract_proj.weight"] = torch.randn(cfg.encoder_embed_dim, NUM_MEL_BINS, generator=g) / NUM_MEL_BINS**0.5
        sd["post_extract_proj.bias"] = torch.randn(cfg.encoder_embed_dim, generator=g) * 0.05

        class TwoLayerDecoar2(Decoar2Expert):  # Decoar2Expert's frame rule and length check on a two-layer encoder
            def __init__(self):
                UpstreamExpert.__init__(self, name="decoar2", arch=cfg, state_dict=sd)

        return TwoLayerDecoar2()
    if kind == "xls_r_hd80":
        return UpstreamExpert(name="wav2vec2_local", arch=replace(XLS_R["xls_r_1b"], encoder_layers=2))
    return UpstreamExpert(name=kind, arch=replace(ARCHS[kind], encoder_layers=2))


def _close(ex):
    if ex._native is not None:
        torch.cuda.synchronize()
        ex._native.close()
        ex._native = None


def _dims(ex):
    """(output slots, channels) of hidden_out."""
    if hasattr(ex, "arch"):
        return ex.arch.num_outputs, ex.arch.encoder_embed_dim
    return (ex.num_outputs if hasattr(ex, "num_outputs") else ex.num_layers), ex.hidden_size


def _min_len(kind):
    return 560 if kind in FBANK else 400


def _len_for(kind, frames):
    """The fewest samples that give `frames` output frames."""
    if kind in RECURRENT:
        return 400 + 160 * (frames - 1)
    if kind == "decoar2":
        return 400 + 160 * (2 * frames - 2)
    return 400 + 320 * (frames - 1)


def _lens(kind, B, T):
    """B ragged lengths whose longest (not the first utterance) gives T frames."""
    lens = [max(_min_len(kind), _len_for(kind, max(1, T * (B - i) // (B + 1))) + 7 * i) for i in range(1, B)]
    lens.insert(min(1, B - 1), _len_for(kind, T) + 13)
    return tuple(lens)


def _wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


def _valid(kind, ex, lens, max_len):
    if kind in RECURRENT:
        return [1 + (n - 400) // 160 for n in lens]
    return ex.valid_frames(list(lens), max_len)


def _forward(ex, dev, lanes=0, gml=None):
    ex.lanes, ex.global_max_len = lanes, gml
    try:
        return torch.stack(tuple(ex(dev)["hidden_states"])).cpu()
    finally:
        ex.lanes, ex.global_max_len = 0, None


def _forward_ex(ex, dev, out_ptr, layer_stride=0, ffn=None, last=None):
    """s3b_forward_ex with the options the experts do not expose."""
    from s3prl_b200 import lib

    native = ex._ensure_native(dev[0].device)
    B, lens = len(dev), [int(w.numel()) for w in dev]
    opts = lib.S3BForwardOpts(layer_stride=layer_stride)
    if ffn is not None:
        opts.ffn_out = ffn.data_ptr()
    if last is not None:
        opts.last_residual = last.data_ptr()
    lib.check(native.lib.s3b_forward_ex(native.handle, (C.c_void_p * B)(*[w.data_ptr() for w in dev]),
                                        (C.c_int64 * B)(*lens), B, max(lens), C.c_void_p(out_ptr),
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(opts)))


def _describe(got, ref, valid):
    """The first output slot that differs, and per utterance the frame range, split into valid and padded frames."""
    if got.shape != ref.shape:
        return f"shape {tuple(got.shape)} != {tuple(ref.shape)}"
    ne = (got != ref) & ~(torch.isnan(got) & torch.isnan(ref))
    if not ne.any():
        return "same values, NaN at the same places"
    slots = [i for i in range(got.shape[0]) if ne[i].any()]
    i = slots[0]
    parts = [f"first differing output slot {i} (of slots {slots})"]
    for b in range(got.shape[1]):
        frames = ne[i, b].any(dim=-1).nonzero().flatten()
        if frames.numel() == 0:
            continue
        v = valid[b] if valid is not None else got.shape[2]
        n_valid = int((frames < v).sum())
        nonfinite = int((~torch.isfinite(got[i, b])).sum())
        parts.append(f"utterance {b}: {frames.numel()} frames in [{int(frames[0])}, {int(frames[-1])}] "
                     f"({n_valid} valid, {frames.numel() - n_valid} padded; {v} valid of {got.shape[2]}), "
                     f"{int(ne[i, b].sum())} elements, {nonfinite} non-finite")
    return "; ".join(parts)


# ------------------------------------------------------------------------------------------------
# the two passes
# ------------------------------------------------------------------------------------------------
_REF = {}      # (kind, scheme, probe key) -> reference tensors on the host
_FACTORY = {}  # (kind, scheme) -> the expert whose native model is re-created for every reference


class _History:
    """One pass over a script: `live` None computes the references, otherwise runs the long-lived models."""

    def __init__(self, scheme, kinds, live):
        self.scheme, self.kinds, self.live, self.failures = scheme, kinds, live, []

    @property
    def reference_pass(self):
        return self.live is None

    def _reference(self, who, key, fn):
        kind = self.kinds[who]
        full = (kind, self.scheme, key)
        if full not in _REF:
            fk = (kind, self.scheme)
            if fk not in _FACTORY:
                _FACTORY[fk] = _build(kind).to("cuda").eval()
            fx = _FACTORY[fk]
            _close(fx)
            try:
                _REF[full] = fn(fx)
            finally:
                _close(fx)
        return _REF[full]

    def _compare(self, who, step, what, got, ref, valid=None):
        tag = f"{self.kinds[who]}[{self.scheme or 'default'}] {step}: {what}"
        if torch.equal(got, ref):
            print(f"{tag}: identical")
            return
        msg = f"{tag}: DIFFERS: {_describe(got, ref, valid)}"
        print(msg)
        self.failures.append(msg)

    def run(self, fn, who="A"):
        """A call of the history whose result is not compared."""
        if not self.reference_pass:
            fn(self.live[who])
            torch.cuda.synchronize()

    def probe(self, step, lens, seed, who="A", lanes=0, gml=None, dev=None, host_chunks=None, monkeypatch=None):
        """The long-lived model's result for (lens, seed) against a fresh model's single lanes = 1 device forward.
        dev: device tensors to run on (already holding the waveforms); host_chunks: through forward_host."""
        key = (tuple(lens), seed, gml)
        host = _wavs(lens, seed)
        if self.reference_pass:
            self._reference(who, key, lambda fx: _forward(fx, [w.cuda() for w in host], 1, gml))
            return
        ex, kind = self.live[who], self.kinds[who]
        what = f"B={len(lens)} max_len={gml or max(lens)} lanes={lanes}"
        if host_chunks is not None:
            monkeypatch.setenv("S3B_HOST_CHUNKS", str(host_chunks))
            torch.cuda.synchronize()
            ex.global_max_len = gml
            try:
                got = ex.forward_host(host).clone()
            finally:
                ex.global_max_len = None
                monkeypatch.delenv("S3B_HOST_CHUNKS")
            what += f" forward_host chunks={host_chunks}"
        else:
            got = _forward(ex, dev if dev is not None else [w.cuda() for w in host], lanes, gml)
        ref = _REF[(kind, self.scheme, key)]
        self._compare(who, step, what, got, ref, _valid(kind, ex, lens, gml or max(lens)))
        return got

    def probe_options(self, step, lens, seed, who="A"):
        """layer_stride into a NaN-filled larger buffer, then ffn_out / last_residual on, off, and on with other
        pointers, all at one (B, max_len): the plan is shared and these pointers are patched per call."""
        kind = self.kinds[who]
        host = _wavs(lens, seed)
        B = len(lens)
        extras = kind not in FBANK[1:] and kind not in ("wav2vec2_conformer_rope", "distilhubert_base")
        pre_ln = kind in ("wav2vec2_large_ll60k", "xls_r_hd80")

        def alloc(ex):
            n, D = _dims(ex)
            T = ex.num_frames(max(lens))
            nl = n - 1
            return n, nl, T, D

        def reference(fx):
            n, nl, T, D = alloc(fx)
            out = torch.empty(n, B, T, D, device="cuda")
            ffn = torch.empty(nl, B, T, D, device="cuda") if extras else None
            last = torch.empty(B, T, D, device="cuda") if extras and pre_ln else None
            _forward_ex(fx, [w.cuda() for w in host], out.data_ptr(), ffn=ffn, last=last)
            return tuple(None if t is None else t.cpu() for t in (out, ffn, last))

        key = (tuple(lens), seed, "options")
        if self.reference_pass:
            self._reference(who, key, reference)
            return
        ex = self.live[who]
        r_out, r_ffn, r_last = _REF[(kind, self.scheme, key)]
        valid = _valid(kind, ex, lens, max(lens))
        n, nl, T, D = alloc(ex)
        dev = [w.cuda() for w in host]
        nan = float("nan")
        # utterances 1 .. B of a [n][B + 2][T][D] buffer
        big = torch.full((n, B + 2, T, D), nan, device="cuda")
        _forward_ex(ex, dev, big[0, 1].data_ptr(), layer_stride=(B + 2) * T * D)
        big = big.cpu()
        self._compare(who, step, "layer_stride slice", big[:, 1:B + 1].contiguous(), r_out, valid)
        outside = torch.cat([big[:, :1], big[:, B + 1:]], dim=1)
        if not torch.isnan(outside).all():
            self.failures.append(f"{kind} {step}: layer_stride: {int((~torch.isnan(outside)).sum())} elements written "
                                 "outside the sub-batch's slice")
        if not extras:
            return
        bufs = []
        for turn, on in enumerate((True, False, True)):
            out = torch.full((n, B, T, D), nan, device="cuda")
            ffn = torch.full((nl, B, T, D), nan, device="cuda") if on else None
            last = torch.full((B, T, D), nan, device="cuda") if on and pre_ln else None
            for old in bufs:
                old.fill_(nan)
            _forward_ex(ex, dev, out.data_ptr(), ffn=ffn, last=last)
            self._compare(who, step, f"hidden, ffn_out {'on' if on else 'off'} (turn {turn})", out.cpu(), r_out, valid)
            if on:
                self._compare(who, step, f"ffn_out (turn {turn})", ffn.cpu(), r_ffn, valid)
                if last is not None:
                    self._compare(who, step, f"last_residual (turn {turn})", last.cpu()[None], r_last[None], valid)
            for old in bufs:  # the pointers of an earlier call must not be written again
                if not torch.isnan(old).all():
                    self.failures.append(f"{kind} {step}: turn {turn} wrote into an earlier call's ffn_out / last_residual")
            bufs += [t for t in (ffn, last) if t is not None]


def _play(script, scheme, kinds, monkeypatch):
    """script(h) twice: references on fresh models first, then the history on long-lived models."""
    if scheme is not None:
        monkeypatch.setenv("S3B_GEMM_SCHEME", scheme)  # read when a native model is created
    else:
        monkeypatch.delenv("S3B_GEMM_SCHEME", raising=False)
    script(_History(scheme, kinds, None))
    live = {who: _build(kind).to("cuda").eval() for who, kind in kinds.items()}
    h = _History(scheme, kinds, live)
    try:
        script(h)
    finally:
        for ex in live.values():
            _close(ex)
    assert not h.failures, "\n".join(h.failures)


def _poison(kind, lens):
    """Waveforms that are non-finite in different ways, utterance by utterance; the first two of each lane's half
    (whose workspace rows the small probes reuse) in the way that reaches every row. The fbank front end takes
    log(fmaxf(energy, eps)), and fmaxf drops a NaN, so a NaN or inf sample would come out as a finite constant frame:
    for the fbank kinds the same patterns are built from +-1e30 to 3e30, whose power spectrum overflows to inf."""
    g = torch.Generator().manual_seed(99)
    wavs = []
    for i, n in enumerate(lens):
        w = torch.randn(n, generator=g)
        how = (0, 0, 1, 2, 0, 0, 3, 1)[i % 8]
        if how == 0 and kind in FBANK:
            w *= 1e30
        elif how == 0:
            w.fill_(float("nan"))
        elif how == 1:
            w.fill_(1e30)
            w[::3] = -1e30
        elif how == 2:
            w[::7] = float("inf")
            w[3::11] = float("-inf")
        else:
            w[::5] = float("nan")
            w[1::2] *= 1e30
        if kind in FBANK:
            w = torch.nan_to_num(w, nan=1e30, posinf=3e30, neginf=-3e30)
        wavs.append(w)
    return wavs


BIG = (80000, 61234, 47000, 33333, 16000, 5000)                # B = 6, up to 5 s
BIGGER = (96000, 90001, 70000, 52345, 31000, 12000, 800)       # B = 7, up to 6 s: every buffer is reallocated
POISON = (104000, 104000, 99000, 90000, 104000, 101000, 95000, 88000)  # B = 8, 6.5 s: larger than every probe


def _history(kind, monkeypatch):
    from s3prl_b200 import lib

    def script(h):
        P = [(B, T) for T in PROBE_T for B in (1, 3)]

        def probes(step, which=P, **kw):
            for B, T in which:
                h.probe(f"{step} B={B} T={T}", _lens(kind, B, T), 100 * T + B, **kw)

        # 1. shrink: a large ragged batch, then small ones at the tile and padding edges
        h.probe("1 shrink: the large batch", BIG, 1)
        probes("1 shrink")
        if kind in FBANK:  # two-frame utterances next to a long one
            h.probe("1 shrink: 560 samples next to long", (_len_for(kind, 129), 560, 719, 20000), 2)
        # 2. grow back past the first size (reallocation: new generation, l8_off moves), then earlier shapes again
        h.probe("2 grow: the larger batch", BIGGER, 3)
        probes("2 after growth", [(3, 65), (1, 129), (3, 2)])
        h.probe("2 after growth: the first large batch", BIG, 1)
        # 3. same (B, max_len) on the same device tensors: new values, other inner lengths, then the same call again
        top = _len_for(kind, 71) + 5
        bufs = [torch.empty(top, device="cuda") for _ in range(3)]
        for turn, (inner, seed) in enumerate((((top, top - 4000, _min_len(kind)), 4), ((top - 9000, top, top - 321), 5),
                                              ((top - 9000, top, top - 321), 5))):
            dev = []
            for buf, w in zip(bufs, _wavs(inner, seed)):
                buf[: w.numel()].copy_(w)
                dev.append(buf[: w.numel()])
            h.probe(f"3 same shape, turn {turn}", inner, seed, dev=dev)
        # 4. six distinct (B, max_len) in a row, then the first again: the plan LRU holds four
        probes("4 eviction", P[:6] + P[:1])
        # 5. lanes 2 -> 1 -> 0 -> 2 over odd and even batches: lane 1's workspace sees sub-batches of changing size
        for i, (B, T, lanes) in enumerate(((5, 140, 2), (4, 97, 1), (3, 65, 0), (4, 97, 2), (5, 33, 2), (2, 129, 2))):
            h.probe(f"5 lanes, call {i}", _lens(kind, B, T), 100 * T + B, lanes=lanes)
        # 6. options at one shape; a larger global max_len and back; profiling on and off
        h.probe_options("6 options", _lens(kind, 2, 71), 6)
        small = _lens(kind, 3, 65)
        h.probe("6 global_max_len larger", small, 6503, gml=_len_for(kind, 90))
        h.probe("6 global_max_len back", small, 6503)

        def profile(on):
            def fn(ex):
                lib.check(ex._native.lib.s3b_profile_enable(ex._native.handle, int(on)))
                if not on:
                    ms, fl, n = (C.c_double * 6)(), (C.c_double * 6)(), (C.c_int64 * 6)()
                    lib.check(ex._native.lib.s3b_profile_read_ex(ex._native.handle, 6, ms, fl, n, 1))
            return fn

        h.run(profile(True))
        h.probe("6 profiling on, two lanes run in turn", _lens(kind, 4, 97), 9704, lanes=2)
        h.run(profile(False))
        h.probe("6 profiling off again", _lens(kind, 4, 97), 9704, lanes=2)
        # 7. the host path between device forwards
        for chunks in (1, 2, 3):
            h.probe("7 host path", _lens(kind, 5, 140), 14005, host_chunks=chunks, monkeypatch=monkeypatch)
            h.probe("7 device forward after the host path", _lens(kind, 3, 63), 6303)
        # 8. poison: one call, larger than every probe in B and T, on both lanes; then every probe again
        poison = _poison(kind, POISON)

        def run_poison(ex):
            out = _forward(ex, [w.cuda() for w in poison], lanes=2)
            assert not torch.isfinite(out[-1, [0, 1, 4, 5], :200]).any(), "the poison did not reach the last output"

        h.run(run_poison)
        for B, T in P:
            lens = _lens(kind, B, T)
            got = h.probe(f"8 after poison B={B} T={T}", lens, 100 * T + B)
            if got is not None and kind in RECURRENT:  # frames t >= m_b are exactly zero
                for b, m in enumerate(_valid(kind, None, lens, max(lens))):
                    if got[:, b, m:].count_nonzero() != 0:
                        h.failures.append(f"{kind} 8 after poison B={B} T={T}: utterance {b} is not zero from frame {m}")
        h.probe("8 after poison, two lanes", _lens(kind, 5, 140), 14005, lanes=2)
        h.probe("8 after poison, host path", _lens(kind, 5, 140), 14005, host_chunks=2, monkeypatch=monkeypatch)
        h.probe("8 after poison: the first large batch", BIG, 1)

    return script


# ------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,scheme", KINDS, ids=[f"{k}-{s or 'default'}" for k, s in KINDS])
def test_forward_is_independent_of_history(s3b_lib, monkeypatch, kind, scheme):
    """Steps 1 to 8 on one long-lived model: shrink, grow back, same shape with new content, plan eviction, lanes,
    options, the host path and a poisoned call. DeCoAR runs as one lane whatever ``lanes`` says, and every call here
    is complete (copied to the host) before the next starts, so no two recurrences are ever in flight."""
    _play(_history(kind, monkeypatch), scheme, {"A": kind}, monkeypatch)


@pytest.mark.slow
@pytest.mark.parametrize("kind", ["wavlm_base_plus", "wav2vec2_conformer_rope"])
def test_table_rebuild(s3b_lib, monkeypatch, kind):
    """One utterance longer than the table built at finalize (4096 frames): the relative-position table (WavLM) or the
    rotary table (Conformer) is rebuilt for twice its frames, and the short probes then run on the rebuilt table, whose
    centre and row stride have moved."""

    def script(h):
        h.probe("9 before the rebuild", _lens(kind, 3, 65), 6503)
        h.probe("9 4100 frames", (_len_for(kind, 4100),), 7)
        for T in PROBE_T:
            for B in (1, 3):
                h.probe(f"9 on the rebuilt table B={B} T={T}", _lens(kind, B, T), 100 * T + B)

    _play(script, None, {"A": kind}, monkeypatch)


def test_two_models_alive(s3b_lib, monkeypatch):
    """Two models of different kinds on one device, calls interleaved. C's first large call lands between two identical
    calls of A: it moves the allocation generation both share, so A's plan is rebuilt on unchanged buffers. Then C is
    destroyed and A called again."""
    lens_a, lens_c = _lens("hubert_base", 3, 65), _lens("apc", 3, 65)

    def script(h):
        h.probe("10 A first", lens_a, 6503)
        h.probe("10 A again (plan hit)", lens_a, 6503)
        h.probe("10 C's first large call", BIG, 1, who="C")
        h.probe("10 A after C allocated", lens_a, 6503)
        h.probe("10 C small", lens_c, 6503, who="C")
        h.probe("10 A larger", _lens("hubert_base", 4, 97), 9704)
        h.probe("10 C after A allocated", lens_c, 6503, who="C")
        h.run(_close, who="C")
        h.probe("10 A after C was destroyed", lens_a, 6503)

    _play(script, None, {"A": "hubert_base", "C": "apc"}, monkeypatch)
