"""TEST INFRASTRUCTURE — generates tests/golden/*.pt by EXECUTING THE REFERENCE (s3prl @ /root/reference).

Run in the build container only (the reference does not travel to the GPU box):

    PYTHONPATH=/root/reference python oracle/make_golden.py [--only hubert_base]

For every architecture it
  1. fabricates the deterministic checkpoint (s3prl_b200.upstream.weights.fabricate_state_dict, seed 0),
  2. writes it in the reference's converted-checkpoint format and loads it with the reference's own
     ``UpstreamExpert`` (s3prl/upstream/{hubert,wav2vec2,wavlm}/expert.py) — reference constructors, reference
     ``load_state_dict``, reference forward and hooks,
  3. runs ``expert(wavs)`` on seeded waveforms (equal-length and ragged batches, incl. a 0.05 s utterance),
  4. stores a strided sub-sample of every hidden state plus per-layer norms (fixtures stay < 1 MB each).
Integer rules (frame masks, WavLM buckets, Featurizer lengths) are recorded exhaustively, and the host logic of
s3prl.nn (Featurizer, UpstreamDownstreamModel, S3PRLUpstream bookkeeping) on fake upstreams.
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))
GOLDEN = ROOT / "tests" / "golden"

from s3prl_b200.upstream.configs import ARCHS, CONV_LAYERS  # noqa: E402
from s3prl_b200.upstream.weights import fabricate_state_dict  # noqa: E402

# (architecture, list of waveform lengths per case, channel stride of the stored sub-sample)
CASES = {
    "hubert_base": ([[16000, 12345, 800], [8000, 8000]], 14),
    "wav2vec2_base_960": ([[16000, 12345, 800], [8000, 8000]], 14),
    "wavlm_base_plus": ([[16000, 12345, 800], [8000, 8000]], 14),
    "wav2vec2_large_ll60k": ([[12000, 7001]], 13),
    "wav2vec2_large_960": ([[12000, 7001]], 13),
    "wavlm_large": ([[12000, 7001]], 13),
    "hubert_large_ll60k": ([[12000, 7001]], 13),
    "unispeech_sat_base_plus": ([[16000, 12345, 800], [8000, 8000]], 14),
    "unispeech_sat_large": ([[12000, 7001]], 13),
    "distilhubert_base": ([[16000, 12345, 3200], [8000, 8000]], 7),
    "data2vec_base_960": ([[16000, 12345, 800], [8000, 8000]], 14),
    "data2vec_large_ll60k": ([[12000, 7001]], 13),
}


# BASELINE.json sizes on a batch
# the CPU reference can afford: fixture name -> (architecture, cases, channel stride, time stride of the sub-sample)
FULL_SIZE = {
    "c3_wav2vec2_large_960": ("wav2vec2_large_960", [[320000, 320000]], 26, 16),
    "c3_wav2vec2_large_ll60k": ("wav2vec2_large_ll60k", [[320000, 271828]], 26, 16),
    "c4_wavlm_base_plus": ("wavlm_base_plus", [[160000, 160000], [160000, 100003]], 14, 8),
}


def seeded_wavs(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in lens]


from ref_runtime import reference_expert  # noqa: E402  (the reference itself on a fabricated checkpoint)


def make_model_fixture(name: str, fixture: str = None):
    if fixture is None:
        (lens_cases, cstride), tstride, fixture = CASES[name], 1, name
    else:
        name, lens_cases, cstride, tstride = FULL_SIZE[fixture]
    sd = fabricate_state_dict(ARCHS[name], seed=0)
    expert = reference_expert(name, sd)
    out = {"arch": name, "weight_seed": 0, "channel_stride": cstride, "time_stride": tstride, "cases": []}
    for ci, lens in enumerate(lens_cases):
        wavs = seeded_wavs(lens, seed=100 + ci)
        with torch.no_grad():
            res = expert(wavs)
        hs = [h.float() for h in res["hidden_states"]]
        out["cases"].append(
            {
                "lens": lens,
                "wav_seed": 100 + ci,
                "shape": tuple(hs[0].shape),
                "num_hidden": len(hs),
                # time sub-sample anchored at the LAST frame so that the end of the sequence is always covered
                "sub": torch.stack([h[:, (h.shape[1] - 1) % tstride :: tstride, ::cstride].contiguous() for h in hs]),
                "norms": torch.tensor([h.double().norm().item() for h in hs]),
                "abs_max": torch.tensor([h.abs().max().item() for h in hs]),
            }
        )
        print(f"{fixture} case {ci}: lens={lens} -> {len(hs)} x {tuple(hs[0].shape)}", flush=True)
    torch.save(out, GOLDEN / f"{fixture}.pt")


def make_integer_fixture():
    """Frame-mask rules, WavLM buckets and length rules straight from the reference code."""
    from s3prl.upstream.hubert.hubert_model import HubertModel
    from s3prl.upstream.interfaces import Featurizer  # noqa: F401  (rule restated below, see tolist)
    from s3prl.upstream.wav2vec2.wav2vec2_model import Wav2Vec2Config, Wav2Vec2Model
    from s3prl.upstream.wavlm.modules import MultiheadAttention as WavLMAttention

    g = torch.Generator().manual_seed(7)
    batches, short_batches = [], []
    w2v = Wav2Vec2Model(Wav2Vec2Config(encoder_layers=1, quantize_targets=False))
    # 60 random batches, then batches holding utterances SHORTER than the 400-sample receptive field (the wav2vec2
    # rule's unclamped floor arithmetic goes to 0 / negative there and the mask index wraps around)
    short = [[16000, 50], [16000, 5], [8000, 399, 55, 56, 57, 1], [16000, 400, 401, 719, 720, 721], [4000, 10, 9, 14, 15, 16]]
    g2 = torch.Generator().manual_seed(11)
    for _ in range(12):
        short.append([int(torch.randint(2000, 40000, (1,), generator=g2))] + torch.randint(1, 400, (4,), generator=g2).tolist())
    for it in range(60 + len(short)):
        if it >= 60:
            lens = short[it - 60]
            B = len(lens)
        else:
            B = int(torch.randint(1, 7, (1,), generator=g))
            lens = torch.randint(400, 170000, (B,), generator=g).tolist()
            if torch.rand(1, generator=g).item() < 0.3:
                lens = [max(lens)] * B  # no padding at all
        Lmax = max(lens)
        pad = ~torch.lt(torch.arange(Lmax).unsqueeze(0), torch.tensor(lens).unsqueeze(1))
        n = Lmax
        for _d, k, s in CONV_LAYERS:
            n = (n - k) // s + 1
        T = n
        feats = torch.zeros(B, T, 1)
        hub_mask = HubertModel.forward_padding_mask(None, feats, pad)
        # wav2vec2 rule: replay the statements of Wav2Vec2Model.forward (wav2vec2_model.py:2652-2671)
        if pad.any():
            input_lengths = (1 - pad.long()).sum(-1)
            output_lengths = w2v._get_feat_extract_output_lengths(input_lengths)
            m = torch.zeros((B, T), dtype=torch.float32)
            m[(torch.arange(B), output_lengths - 1)] = 1
            w2v_mask = (1 - m.flip([-1]).cumsum(-1).flip([-1])).bool()
            w2v_valid = [int((~r).sum()) for r in w2v_mask]
        else:
            w2v_valid = [T] * B
        (batches if it < 60 else short_batches).append(
            {
                "lens": lens,
                "T": T,
                "hubert_valid": [int((~r).sum()) for r in hub_mask],
                "hubert_prefix": bool(all((r[: int((~r).sum())] == False).all() for r in hub_mask)),  # noqa: E712
                "wav2vec2_valid": w2v_valid,
                "featurizer_len": [round(n_ / 320) for n_ in lens],
                "s3prl_upstream_len": [(n_ - 1) // 320 + 1 for n_ in lens],
            }
        )
    att = WavLMAttention(768, 12, has_relative_attention_bias=True, num_buckets=320, max_distance=800)
    rel = torch.arange(-2100, 2101, dtype=torch.long)
    buckets = att._relative_positions_bucket(rel.unsqueeze(0), bidirectional=True)[0]
    torch.save({"batches": batches, "short_batches": short_batches, "wavlm_rel": rel, "wavlm_bucket": buckets},
               GOLDEN / "integer_rules.pt")
    print(f"integer rules: {len(batches)} + {len(short_batches)} batches, {len(rel)} relative positions")


def make_fbank_fixture():
    """s3prl.upstream.baseline fbank (config 1: 4 x 1 s, seed 0) + a ragged batch."""
    from s3prl.upstream.baseline.hubconf import fbank

    expert = fbank()
    expert.eval()
    out = {"cases": []}
    torch.manual_seed(0)
    c1 = [torch.randn(16000) for _ in range(4)]  # BASELINE.json config C1
    for name, wavs in (("c1_4x1s_seed0", c1), ("ragged", seeded_wavs([16000, 9999, 4000, 480], 321))):
        with torch.no_grad():
            hs = expert(wavs)["hidden_states"][0]
        out["cases"].append({"name": name, "lens": [len(w) for w in wavs], "out": hs.float().clone()})
        print(f"fbank {name}: {tuple(hs.shape)}")
    torch.save(out, GOLDEN / "fbank.pt")


def make_spectrogram_fixture():
    """s3prl.upstream.baseline mel / linear entries (torch.stft path) on equal-length and ragged batches."""
    from s3prl.upstream.baseline.hubconf import linear, mel

    out = {"cases": []}
    for name, factory in (("mel", mel), ("linear", linear)):
        expert = factory()
        expert.eval()
        torch.manual_seed(0)
        c1 = [torch.randn(16000) for _ in range(4)]
        ragged = seeded_wavs([16000, 9999, 4000, 1234], 654)
        ragged[1][-37:] = 0.0  # trailing exact zeros exercise the non-zero trimming rule
        for cname, wavs in (("4x1s_seed0", c1), ("ragged", ragged)):
            with torch.no_grad():
                hs = expert(wavs)["hidden_states"][0]
            out["cases"].append({"feat": name, "name": cname, "lens": [len(w) for w in wavs], "out": hs.float().clone()})
            print(f"{name} {cname}: {tuple(hs.shape)}")
    torch.save(out, GOLDEN / "spectrogram.pt")


# structured inputs (recipes in tests/spectral_ref.py): each keeps a specific error alive through CMVN
SPECTRAL_FBANK = [("chirp", 6400, "none"), ("pink", 6401, "none"), ("bursts", 4800, "none"), ("dc", 2000, "none"),
                  ("tone_fbank_half", 720, "none"), ("impulses", 560, "none"), ("brown", 401, "none"),
                  ("int16", 400, "none")]
SPECTRAL_STFT = [("tone_stft_half", 4321, "none"), ("chirp", 6400, "zeros"), ("pink", 6000, "negzeros"),
                 ("brown", 5000, "none"), ("tone_25", 3000, "first_only")]


def spectral_wavs(spec):
    sys.path.insert(0, str(ROOT / "tests"))
    import spectral_ref as R

    return [R.with_tail(R.structured_wav(kind, n), tail) for kind, n, tail in spec]


def make_spectral_fixture():
    """fbank, fbank_no_cmvn, mel and linear of the reference on structured audio (tones, chirp, bursts, tilted noise,
    DC, impulses, int16 scale, trailing zeros / -0.0, 1-frame utterances). The waveforms are stored as recipes plus
    their fp32 checksums."""
    from s3prl.upstream.baseline.hubconf import fbank, fbank_no_cmvn, linear, mel

    out = {"fbank_spec": SPECTRAL_FBANK, "stft_spec": SPECTRAL_STFT, "cases": {}}
    for spec, entries in ((SPECTRAL_FBANK, (("fbank", fbank), ("fbank_no_cmvn", fbank_no_cmvn))),
                          (SPECTRAL_STFT, (("mel", mel), ("linear", linear)))):
        wavs = spectral_wavs(spec)
        out["checksum_" + ("fbank" if spec is SPECTRAL_FBANK else "stft")] = torch.stack(
            [w.double().sum() for w in wavs] + [w.double().abs().sum() for w in wavs])
        for name, factory in entries:
            expert = factory()
            expert.eval()
            with torch.no_grad():
                hs = expert(wavs)["hidden_states"][0]
            out["cases"][name] = hs.float().clone()
            print(f"spectral {name}: {tuple(hs.shape)}")
    torch.save(out, GOLDEN / "spectral_structured.pt")


class _FakeLayers:
    """Only the layer facts a Featurizer reads (five 16-wide layers, stride 320)."""

    def __init__(self, n):
        self.num_layers, self.hidden_sizes, self.downsample_rates = n, [16] * n, [320] * n


def make_nn_fixture():
    """The reference's s3prl.nn host logic on fake upstreams (no model): Featurizer (layer selections, normalize,
    weights and their gradient, single-layer pass-through), UpstreamDownstreamModel, and S3PRLUpstream's length
    bookkeeping (s3prl/nn/upstream.py:166-384). tests/test_host_cpu.py replays the same inputs through s3prl_b200.nn."""
    import ref_runtime

    ref_runtime.activate()
    from s3prl.nn.upstream import Featurizer, S3PRLUpstream, UpstreamDownstreamModel

    g = torch.Generator().manual_seed(0)
    hs = [torch.randn(3, 7, 16, generator=g) for _ in range(5)]
    lens = torch.tensor([7, 5, 2])
    featurizer = []
    for sel, norm in ((None, False), ([4, 0, 2], False), (None, True), ([1, 3], True)):
        f = Featurizer(_FakeLayers(5), sel, norm)
        w = torch.randn(len(f.weights), generator=g)
        with torch.no_grad():
            f.weights.copy_(w)
        out, out_len = f(hs, [lens] * 5)
        out.square().sum().backward()
        featurizer.append({"sel": sel, "norm": norm, "weights": w, "layer_selections": list(f.layer_selections),
                           "out": out.detach().clone(), "out_len": out_len.clone(), "grad": f.weights.grad.clone(),
                           "output_size": f.output_size, "downsample_rate": f.downsample_rate})
    one = Featurizer(_FakeLayers(1))
    single = {"has_weights": hasattr(one, "weights"), "passthrough": one(hs[:1], [lens])[0] is hs[0]}

    class Up(torch.nn.Module):
        num_layers, hidden_sizes, downsample_rates = 5, [16] * 5, [320] * 5

        def forward(self, wav, wav_len):
            return hs, [lens] * 5

    class Down(torch.nn.Module):
        output_size = 3

        def forward(self, h, h_len, scale=1.0):
            return h.mean(-1) * scale, h_len

    m = UpstreamDownstreamModel(Up(), Featurizer(Up()), Down())
    out, out_len = m(None, None, scale=2.0)
    udm = {"out": out.detach().clone(), "out_len": out_len.clone(),
           "sizes": (m.input_size, m.downsample_rate, m.output_size)}

    class Fake(torch.nn.Module):  # three layers, the conv stack's frame rule, values independent of the waveform
        def forward(self, wavs):
            frames = max((len(w) - 400) // 320 + 1 if len(w) >= 400 else 0 for w in wavs)
            base = torch.arange(len(wavs) * frames * 2, dtype=torch.float32).view(len(wavs), frames, 2)
            return {"hidden_states": [base + k for k in range(3)]}

    up = S3PRLUpstream.__new__(S3PRLUpstream)
    torch.nn.Module.__init__(up)
    up.upstream, up.normalize = Fake(), False
    up._hidden_sizes, up._downsample_rates, up._num_layers = [2] * 3, [320] * 3, 3
    bookkeeping = []
    g = torch.Generator().manual_seed(0)
    for wav_lens in ([16000, 9000, 3200], [16001, 480], [700, 500], [32000, 31999], [1281, 1280, 1279], [48000]):
        for normalize in (False, True):
            up.normalize = normalize
            width = max(wav_lens) + 37  # the padded tensor may be wider than the longest utterance
            wavs = torch.zeros(len(wav_lens), width)
            for i, n in enumerate(wav_lens):
                wavs[i, :n] = torch.randn(n, generator=g)
            for channel_dim in (False, True):
                h, h_len = up(wavs.unsqueeze(-1) if channel_dim else wavs, torch.tensor(wav_lens))
                bookkeeping.append({"lens": wav_lens, "normalize": normalize, "width": width, "channel_dim": channel_dim,
                                    "hs": [x.clone() for x in h], "hs_len": [x.clone() for x in h_len]})
    refused = []
    for wav_lens in ([960, 961], [1000, 900]):  # 2 frames from the conv rule where ceil(L / 320) = 4
        try:
            up(torch.zeros(len(wav_lens), max(wav_lens)), torch.tensor(wav_lens))
            refused.append((wav_lens, False))
        except AssertionError:
            refused.append((wav_lens, True))
    torch.save({"hs": hs, "lens": lens, "featurizer": featurizer, "single": single, "udm": udm,
                "bookkeeping": bookkeeping, "refused": refused}, GOLDEN / "nn_upstream.pt")
    print(f"nn: {len(featurizer)} featurizer cases, {len(bookkeeping)} bookkeeping cases")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    args = ap.parse_args()
    GOLDEN.mkdir(parents=True, exist_ok=True)
    torch.manual_seed(0)
    if args.only in (None, "integer"):
        make_integer_fixture()
    if args.only in (None, "fbank"):
        make_fbank_fixture()
    if args.only in (None, "spectrogram"):
        make_spectrogram_fixture()
    if args.only in (None, "spectral"):
        make_spectral_fixture()
    if args.only in (None, "nn"):
        make_nn_fixture()
    for name in CASES:
        if args.only in (None, name):
            make_model_fixture(name)
    for fixture in FULL_SIZE:
        if args.only in (None, fixture, "full_size"):
            make_model_fixture(None, fixture)


if __name__ == "__main__":
    main()
