"""GPU parity of the full upstream forward (through UpstreamExpert -> C ABI -> sm_90a kernels).

  * against the golden vectors produced by executing the reference (tests/golden/*.pt)
  * against the CPU oracle on other seeded inputs (ragged batches, the survey's parity set)
Tolerance (north_star): hidden states within 1e-3 relative (fp32); we assert 2e-4 relative Frobenius per
layer (measured ~1e-5) and an elementwise bound of 1e-3 of the layer's absolute maximum.
The frame padding bookkeeping is asserted bit-exact in tests/test_oracle_cpu.py.
"""
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
GOLDEN = ROOT / "tests" / "golden"

pytestmark = pytest.mark.gpu

REL_TOL = 2e-4
ABS_FRAC = 1e-3


def _wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


_EXPERTS = {}


def _expert(name):
    from s3prl_b200.upstream.expert import UpstreamExpert

    if name not in _EXPERTS:
        _EXPERTS.clear()  # one resident model at a time
        _EXPERTS[name] = UpstreamExpert(name=name, seed=0).to("cuda")
    return _EXPERTS[name]


def _compare(got, ref, what):
    rel = ((got.double() - ref.double()).norm() / ref.double().norm()).item()
    mx = (got.double() - ref.double()).abs().max().item()
    assert torch.isfinite(got).all(), what
    assert rel < REL_TOL, (what, rel)
    assert mx < ABS_FRAC * ref.abs().max().item(), (what, mx)
    return rel


from s3prl_b200.upstream.configs import ARCHS  # noqa: E402

GOLDEN_MODELS = sorted(p.stem for p in GOLDEN.glob("*.pt") if p.stem in ARCHS)
# BASELINE.json sizes on a batch the CPU reference affords (oracle/make_golden.py FULL_SIZE): wav2vec2_large at
# T = 999 (C3, both variants), wavlm_base_plus at T = 499 incl. a ragged pair (C4)
FULL_SIZE = sorted(p.stem for p in GOLDEN.glob("c[0-9]_*.pt"))


@pytest.mark.parametrize("name", GOLDEN_MODELS + FULL_SIZE)
def test_matches_reference_golden(s3b_lib, name):
    fx = torch.load(GOLDEN / f"{name}.pt", weights_only=False)
    expert = _expert(fx["arch"])
    cs, ts = fx["channel_stride"], fx.get("time_stride", 1)
    worst = 0.0
    for case in fx["cases"]:
        wavs = [w.cuda() for w in _wavs(case["lens"], case["wav_seed"])]
        res = expert(wavs)
        hs = res["hidden_states"]
        assert len(hs) == case["num_hidden"]
        assert tuple(hs[0].shape) == tuple(case["shape"])
        assert res["last_hidden_state"] is hs[-1]
        for l, h in enumerate(hs):
            sub = h[:, (h.shape[1] - 1) % ts :: ts, ::cs]
            worst = max(worst, _compare(sub.cpu(), case["sub"][l], f"{name} case lens={case['lens']} layer {l}"))
            nrm = h.double().norm().item()
            assert abs(nrm - case["norms"][l].item()) < REL_TOL * case["norms"][l].item()
    print(f"{name}: worst per-layer relative error vs reference golden = {worst:.3e}")


@pytest.mark.parametrize(
    "name,lens",
    [
        ("hubert_base", [160000, 123457, 80000, 16000, 800]),  # the survey's ragged parity set
        ("hubert_base", [32000, 32000, 32000]),                # no padding
        ("wav2vec2_base_960", [48000, 31999, 1200]),
        ("wav2vec2_base_960", [16000, 50, 399, 5]),  # shorter than the receptive field: the reference's mask index wraps
        ("wavlm_base_plus", [40000, 33333, 900]),
        ("distilhubert_base", [40000, 33333, 900]),  # feat_final + 2 layer outputs + 3 prediction heads
        ("data2vec_base_960", [40000, 33333, 900]),  # five conv blocks as positional encoder, nothing re-masked between
        ("data2vec_base_960", [16000, 50, 399]),     # them; wav2vec 2.0 mask rule incl. the wrap-around of short inputs
    ],
)
def test_matches_oracle_ragged(s3b_lib, name, lens):
    import upstream_oracle as O
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = ARCHS[name]
    sd = fabricate_state_dict(cfg, seed=0)
    wavs = _wavs(lens, seed=1234)
    with torch.no_grad():
        ref, pad = O.upstream_forward(wavs, sd, cfg)
    expert = _expert(name)
    hs = expert([w.cuda() for w in wavs])["hidden_states"]
    assert len(hs) == len(ref)
    worst = 0.0
    for l, (h, r) in enumerate(zip(hs, ref)):
        assert h.shape == r.shape
        worst = max(worst, _compare(h.cpu(), r, f"{name} lens={lens} layer {l}"))
    valid = expert.valid_frames(lens)
    assert valid == O.valid_frames(cfg.family, lens, max(lens))
    print(f"{name} lens={lens}: worst per-layer relative error vs oracle = {worst:.3e}")


@pytest.mark.parametrize("depth,conv_pos,dim", [(2, 95, 768), (4, 96, 768), (5, 95, 1024), (3, 9, 768)])
def test_positional_conv_block_variants(s3b_lib, depth, conv_pos, dim):
    """pos_conv_depth > 1 (make_conv_block, wav2vec2_model.py:2995-3026) beyond the published data2vec shape: k = 47
    (rounded up to 48 taps), an EVEN k = 24 (SamePad drops the last frame), 64 channels per group, and the k = 3 floor
    of max(3, conv_pos // depth); two-layer encoders against the oracle, ragged batch."""
    import dataclasses

    import upstream_oracle as O
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = dataclasses.replace(ARCHS["data2vec_base_960"], encoder_layers=2, pos_conv_depth=depth, conv_pos=conv_pos,
                              encoder_embed_dim=dim, encoder_attention_heads=dim // 64, encoder_ffn_embed_dim=4 * dim)
    sd = fabricate_state_dict(cfg, seed=3)
    lens = [24000, 17777, 1000]
    wavs = _wavs(lens, seed=77)
    with torch.no_grad():
        ref, _pad = O.upstream_forward(wavs, sd, cfg)
    _EXPERTS.clear()
    expert = UpstreamExpert(arch=cfg, state_dict=sd, name="data2vec_variant").to("cuda")
    hs = expert([w.cuda() for w in wavs])["hidden_states"]
    assert len(hs) == len(ref) == 3
    for l, (h, r) in enumerate(zip(hs, ref)):
        _compare(h.cpu(), r, f"pos_conv depth={depth} conv_pos={conv_pos} D={dim} layer {l}")


@pytest.mark.slow
def test_wavlm_rel_table_rebuild(s3b_lib):
    """WavLM's relative-position table is built at finalize for 4096 frames (82 s) and rebuilt for 2T frames when a
    longer batch arrives. A two-layer wavlm_base_plus: one 82.5 s utterance (T = 4124 > 4096) against the oracle,
    then, on the same model and its rebuilt table (centre 2 * 4124 - 1), a short ragged batch. The oracle's
    [H, T, T] bias and scores take a few GB of host memory at this length."""
    import dataclasses

    import upstream_oracle as O
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = dataclasses.replace(ARCHS["wavlm_base_plus"], encoder_layers=2)
    sd = fabricate_state_dict(cfg, seed=11)
    _EXPERTS.clear()
    expert = UpstreamExpert(arch=cfg, state_dict=sd, name="wavlm_two_layers").to("cuda")
    for lens in ([1_320_000], [40000, 33333, 900]):
        wavs = _wavs(lens, seed=len(lens))
        assert len(lens) > 1 or O.conv_output_length(lens[0]) > 4096
        with torch.no_grad():
            ref, _pad = O.upstream_forward(wavs, sd, cfg)
        hs = expert([w.cuda() for w in wavs])["hidden_states"]
        assert len(hs) == len(ref) == 3
        worst = 0.0
        for l, (h, r) in enumerate(zip(hs, ref)):
            worst = max(worst, _compare(h.cpu(), r, f"wavlm two layers lens={lens} layer {l}"))
        del ref, hs
        print(f"wavlm two layers lens={lens}: worst per-layer relative error vs oracle = {worst:.3e}")


def test_forward_host_matches_device(s3b_lib):
    expert = _expert("hubert_base")
    wavs = _wavs([16000, 9000], seed=5)
    dev = torch.stack(expert([w.cuda() for w in wavs])["hidden_states"]).cpu()
    host = expert.forward_host(wavs)
    assert torch.equal(dev, host)


def test_forward_host_chunked_matches_device(s3b_lib):
    """Chunked host forward (chunk c+1's conv stack overlaps chunk c's device->host copies) is bit-identical."""
    expert = _expert("hubert_base")
    wavs = _wavs([16000, 9000, 12000, 4000, 16000], seed=6)
    dev = torch.stack(expert([w.cuda() for w in wavs])["hidden_states"]).cpu()
    for chunks in ("2", "3", "5", "9"):
        os.environ["S3B_HOST_CHUNKS"] = chunks
        try:
            host = expert.forward_host(wavs)
        finally:
            os.environ.pop("S3B_HOST_CHUNKS", None)
        assert torch.equal(dev, host), chunks


def test_short_utterances(s3b_lib):
    """0.05 s inputs (T = 2 frames), the reference's _test_forward_backward sizes (test/test_upstream.py:192-200)."""
    import upstream_oracle as O
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = ARCHS["hubert_base"]
    sd = fabricate_state_dict(cfg, seed=0)
    expert = _expert("hubert_base")
    for lens in ([800], [800, 800], [800, 5000, 16000]):
        wavs = _wavs(lens, seed=9)
        with torch.no_grad():
            ref, _ = O.upstream_forward(wavs, sd, cfg)
        hs = expert([w.cuda() for w in wavs])["hidden_states"]
        for l, (h, r) in enumerate(zip(hs, ref)):
            _compare(h.cpu(), r, f"short lens={lens} layer {l}")


def test_lanes_are_bit_identical(s3b_lib):
    """Two utterance micro-batches on two streams (the default) == one lane, bit for bit, also for odd / ragged batches."""
    expert = _expert("hubert_base")
    for lens in ([32000] * 4, [24000, 17000, 9000, 16000, 800], [16000, 12000]):
        wavs = [w.cuda() for w in _wavs(lens, seed=77)]
        outs = []
        for lanes in (1, 2):
            expert.lanes = lanes
            try:
                outs.append(torch.stack(expert(wavs)["hidden_states"]).clone())
            finally:
                expert.lanes = 0
        assert torch.equal(outs[0], outs[1]), lens
        assert torch.equal(torch.stack(expert(wavs)["hidden_states"]), outs[0])


def test_wav2vec2_feature_selection_and_hooks(s3b_lib):
    """feature_selection of the wav2vec2 expert (wav2vec2/expert.py:35-39,81-93) and custom UpstreamBase hooks
    (interfaces.py:74-131) against the oracle: layer outputs, fc2 outputs before the residual add."""
    import torch.nn.functional as F
    import upstream_oracle as O
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    for name in ("wav2vec2_base_960", "wav2vec2_large_ll60k"):
        cfg = ARCHS[name]
        sd = fabricate_state_dict(cfg, seed=0)
        wavs = _wavs([9000, 6000], seed=21)
        with torch.no_grad():
            ref, pad = O.upstream_forward(wavs, sd, cfg)
        NL = cfg.encoder_layers
        _EXPERTS.clear()
        fl = UpstreamExpert(name=name, seed=0, feature_selection="fairseq_layers").to("cuda")
        got = fl([w.cuda() for w in wavs])["hidden_states"]
        assert len(got) == NL
        for l in range(NL - 1):
            _compare(got[l].cpu(), ref[l + 1], f"{name} fairseq_layers {l}")
        if cfg.layer_norm_first:  # last entry is the stream BEFORE encoder.layer_norm
            ln = F.layer_norm(got[-1].cpu(), (got[-1].shape[-1],), sd["encoder.layer_norm.weight"],
                              sd["encoder.layer_norm.bias"], 1e-5)
            _compare(ln, ref[NL], f"{name} fairseq_layers last (re-normalised)")
        else:
            _compare(got[-1].cpu(), ref[NL], f"{name} fairseq_layers last")
        del fl
        br = UpstreamExpert(name=name, seed=0, feature_selection="fairseq_layers_before_residual").to("cuda")
        pre = br([w.cuda() for w in wavs])["hidden_states"]
        assert len(pre) == NL
        if cfg.layer_norm_first:  # residual stream: h_{l+1} = r + fc2_out, r = h_l + attention(...): check the last step
            hk = UpstreamExpert(
                name=name, seed=0,
                hooks=[(f"self.model.encoder.layers[{NL - 2}]", lambda i, o: (o[0] - o[1][1]).transpose(0, 1))],
            ).to("cuda")
            r = hk([w.cuda() for w in wavs])["hidden_states"][0]
            _compare((r + pre[NL - 2]).cpu(), ref[NL - 1], f"{name} r + fc2 == hidden state")
            del hk
        else:  # post-LN: h_{l+1} = LN2(x1 + fc2_out) with x1 = LN1(h_l + attn): verify through the oracle pieces
            p = f"encoder.layers.{NL - 1}"
            h = ref[NL - 1]
            a = O.self_attention(h, {k: v.float() for k, v in sd.items()}, f"{p}.self_attn", cfg.encoder_attention_heads, pad)
            x1 = F.layer_norm(h + a, (h.shape[-1],), sd[f"{p}.self_attn_layer_norm.weight"], sd[f"{p}.self_attn_layer_norm.bias"], 1e-5)
            f2 = F.linear(F.gelu(F.linear(x1, sd[f"{p}.fc1.weight"], sd[f"{p}.fc1.bias"])), sd[f"{p}.fc2.weight"], sd[f"{p}.fc2.bias"])
            _compare(pre[NL - 1].cpu(), f2, f"{name} fairseq_layers_before_residual last")
        del br
    with pytest.raises(TypeError):
        UpstreamExpert(name="hubert_base", feature_selection="fairseq_layers")
    with pytest.raises(ValueError):
        UpstreamExpert(name="hubert_base", hooks=[("self.model.feature_extractor", lambda i, o: o)])


def test_local_checkpoint_entries(s3b_lib, tmp_path):
    """*_local hub entries read a converted reference checkpoint of each layout (hubert/convert.py:37-56,
    wav2vec2/convert.py:26-39, wavlm/expert.py:37-40) and reproduce the named entry bit for bit."""
    from s3prl_b200 import hub
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.convert import save_converted_checkpoint
    from s3prl_b200.upstream.weights import fabricate_state_dict

    wavs = [w.cuda() for w in _wavs([12000, 7001], seed=3)]
    for name, local in (("hubert_base", "hubert_local"), ("wav2vec2_base_960", "wav2vec2_local"),
                        ("wavlm_base_plus", "wavlm_local"), ("unispeech_sat_base_plus", "unispeech_sat_local"),
                        ("distilhubert_base", "distiller_local"), ("data2vec_base_960", "data2vec_local")):
        path = tmp_path / f"{name}.pt"
        save_converted_checkpoint(path, ARCHS[name], fabricate_state_dict(ARCHS[name], 0))
        _EXPERTS.clear()
        a = torch.stack(hub.ENTRIES[name]().to("cuda")(wavs)["hidden_states"])
        b = torch.stack(hub.ENTRIES[local](str(path)).to("cuda")(wavs)["hidden_states"])
        assert torch.equal(a, b), name


@pytest.mark.parametrize("name", ["hubert_base", "wav2vec2_large_ll60k", "wavlm_base_plus", "wavlm_large"])
def test_forward_is_bit_identical_across_calls_and_lanes(s3b_lib, name):
    """A forward is bit-reproducible from call to call and across one / two lanes, for post-LN and pre-LN encoders,
    the per-frame conv LayerNorm + GELU and WavLM's relative-position bias."""
    expert = _expert(name)
    wavs = [w.cuda() for w in _wavs([20000, 16001, 5000], seed=31)]
    ref = torch.stack(expert(wavs)["hidden_states"]).clone()
    for lanes in (1, 2):
        expert.lanes = lanes
        try:
            got = torch.stack(expert(wavs)["hidden_states"])
        finally:
            expert.lanes = 0
        assert torch.equal(got, ref), (name, lanes)


@pytest.mark.parametrize("name", ["hubert_base", "wav2vec2_large_ll60k", "wavlm_base_plus"])
def test_operand_schemes_agree(s3b_lib, name):
    """The two tensor-core operand schemes of the conv / linear GEMMs — bf16 hi/lo with 3 MMAs per product, and fp16 with
    two e4m3 correction products (2 MMA slots, S3B_GEMM_SCHEME=f16q8) — both reproduce the oracle within the parity
    tolerance and agree with each other to well inside it."""
    import upstream_oracle as O
    from s3prl_b200.upstream.configs import ARCHS
    from s3prl_b200.upstream.expert import UpstreamExpert
    from s3prl_b200.upstream.weights import fabricate_state_dict

    cfg = ARCHS[name]
    wavs = _wavs([24000, 17003], seed=77)
    with torch.no_grad():
        ref, _ = O.upstream_forward(wavs, fabricate_state_dict(cfg, 0), cfg)
    outs = {}
    _EXPERTS.clear()
    for scheme in ("bf16x3", "f16q8"):
        os.environ["S3B_GEMM_SCHEME"] = scheme
        try:
            e = UpstreamExpert(name=name, seed=0).to("cuda")
            outs[scheme] = [h.cpu() for h in e([w.cuda() for w in wavs])["hidden_states"]]
            del e
        finally:
            os.environ.pop("S3B_GEMM_SCHEME", None)
        worst = max(_compare(h, r, f"{name} {scheme} layer {l}") for l, (h, r) in enumerate(zip(outs[scheme], ref)))
        print(f"{name} {scheme}: worst per-layer relative error vs oracle = {worst:.3e}")
    for a, b in zip(outs["bf16x3"], outs["f16q8"]):
        assert ((a.double() - b.double()).norm() / b.double().norm()).item() < 1e-4


def test_repeated_calls_are_bit_identical(s3b_lib):
    """10 identical calls after a first one give its result bit for bit and each adds the same launch count."""
    from s3prl_b200.upstream.expert import UpstreamExpert

    g = torch.Generator().manual_seed(5)
    wavs = [torch.randn(n, generator=g).cuda() for n in (24000, 16000, 9000, 20000)]
    e = UpstreamExpert(name="wavlm_base_plus", seed=0).to("cuda")
    ref = torch.stack(e(wavs)["hidden_states"]).clone()
    native = e._native
    counts = []
    for i in range(10):
        c0 = native.lib.s3b_launch_count(native.handle)
        res = e(wavs)
        counts.append(native.lib.s3b_launch_count(native.handle) - c0)
        assert torch.equal(torch.stack(res["hidden_states"]), ref), f"call {i + 1} changed the result"
    assert len(set(counts)) == 1, counts
