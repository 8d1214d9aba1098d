"""fp64 CPU restatement of MAE-AST's forward (s3prl/upstream/mae_ast/{expert,mae_ast}.py) on the tensors the library
reads (s3prl_b200.upstream.mae_ast.prepare_mae_ast_tensors): per utterance kaldi fbank (DC removal, pre-emphasis 0.97
with the first sample replicated, povey window hann(400, periodic=False) ** 0.85, 512-point power spectrum, 128 mel
bins 20 Hz..Nyquist, log(max(E, float eps))), zero-padded to the longest; (x - running_mean) / sqrt(running_var +
1e-5) * 0.5 on every element; unfold into (kt, kc) patches; post_extract_proj; sinusoidal positions on the valid
tokens; the wav2vec 2.0 encoder layers (post-LN with encoder.layer_norm on the input, or pre-LN without a final norm)
under a key mask of valid_b = min(ceil(n_b / kt), T') * nv tokens; each layer's output as [B, T', nv * 768]."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from ssast_oracle import FLOOR, NFFT, SHIFT, WIN, mel_banks

KINDS = {"frame": (2, 128), "patch": (16, 16)}


def povey_window() -> torch.Tensor:
    return torch.hann_window(WIN, periodic=False, dtype=torch.float64).pow(0.85)


def fbank(wav: torch.Tensor) -> torch.Tensor:
    """kaldi.fbank(num_mel_bins=128, use_energy=False) of one utterance: [n, 128] (fp64), n = 1 + (L - 400) // 160."""
    n = 1 + (len(wav) - WIN) // SHIFT
    frames = wav.double().unfold(0, WIN, SHIFT)[:n]
    d = frames - frames.mean(dim=1, keepdim=True)
    prev = torch.cat([d[:, :1], d[:, :-1]], dim=1)
    y = (d - 0.97 * prev) * povey_window()
    P = torch.fft.rfft(F.pad(y, (0, NFFT - WIN))).abs().pow(2)
    return (P @ mel_banks().T).clamp(min=FLOOR).log()


def padded_fbank(wavs: Sequence[torch.Tensor]) -> torch.Tensor:
    """[B, F, 128]: each utterance's frames, zero rows up to the longest's F."""
    feats = [fbank(w) for w in wavs]
    Fm = max(f.shape[0] for f in feats)
    return torch.stack([F.pad(f, (0, 0, 0, Fm - f.shape[0])) for f in feats])


def normalise(x: torch.Tensor, sd: Dict[str, torch.Tensor]) -> torch.Tensor:
    rm, rv = sd["batch_norm.running_mean"].double(), sd["batch_norm.running_var"].double()
    return (x - rm) / torch.sqrt(rv + 1e-5) * 0.5


def unfold(x: torch.Tensor, kind: str) -> torch.Tensor:
    """[B, F, 128] -> [B, T' nv, kt kc]: token t * nv + fi, column i * kc + j (frames past T' kt dropped)."""
    kt, kc = KINDS[kind]
    B, Fm, C = x.shape
    T = Fm // kt
    p = x[:, : T * kt].reshape(B, T, kt, C // kc, kc).permute(0, 1, 3, 2, 4)
    return p.reshape(B, T * (C // kc), kt * kc)


def frontend(wavs: Sequence[torch.Tensor], sd: Dict[str, torch.Tensor], kind: str) -> torch.Tensor:
    """The patch GEMM's A operand [B, T' nv, 256] (fp64)."""
    return unfold(normalise(padded_fbank(wavs), sd), kind)


def valid_tokens(lens: Sequence[int], kind: str, T: int) -> List[int]:
    kt, kc = KINDS[kind]
    nv = 128 // kc
    return [min(-(-(1 + (n - WIN) // SHIFT) // kt), T) * nv for n in lens]


def layer(x: torch.Tensor, sd: Dict[str, torch.Tensor], l: int, key_valid: torch.Tensor, pre: bool,
          heads: int = 12) -> torch.Tensor:
    """TransformerSentenceEncoderLayer; key_valid [B, N] bool."""
    p = f"encoder.layers.{l}."
    g = lambda k: sd[p + k].double()  # noqa: E731
    B, N, C = x.shape
    hd = C // heads
    ln = lambda v, n: F.layer_norm(v, (C,), g(n + ".weight"), g(n + ".bias"), 1e-5)  # noqa: E731

    def attn(h):
        q = F.linear(h, g("self_attn.q_proj.weight"), g("self_attn.q_proj.bias")) * hd ** -0.5
        k = F.linear(h, g("self_attn.k_proj.weight"), g("self_attn.k_proj.bias"))
        v = F.linear(h, g("self_attn.v_proj.weight"), g("self_attn.v_proj.bias"))
        q, k, v = (t.reshape(B, N, heads, hd).transpose(1, 2) for t in (q, k, v))
        s = (q @ k.transpose(-2, -1)).masked_fill(~key_valid[:, None, None, :], float("-inf"))
        a = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, N, C)
        return F.linear(a, g("self_attn.out_proj.weight"), g("self_attn.out_proj.bias"))

    def ffn(h):
        return F.linear(F.gelu(F.linear(h, g("fc1.weight"), g("fc1.bias"))), g("fc2.weight"), g("fc2.bias"))

    if pre:
        x = x + attn(ln(x, "self_attn_layer_norm"))
        return x + ffn(ln(x, "final_layer_norm"))
    x = ln(x + attn(x), "self_attn_layer_norm")
    return ln(x + ffn(x), "final_layer_norm")


def embed(a: torch.Tensor, sd: Dict[str, torch.Tensor], cfg: Dict, valid: Sequence[int]) -> torch.Tensor:
    """post_extract_proj, positions on the valid tokens, and (post-LN) encoder.layer_norm: layer 0's input (fp64)."""
    x = F.linear(a.double(), sd["post_extract_proj.weight"].double(), sd["post_extract_proj.bias"].double())
    B, N, C = x.shape
    if cfg["enc_sine_pos"]:
        pe = sd["enc_sine_pos_embed.pe"][0, :N].double()
        keep = torch.arange(N)[None, :] < torch.tensor(list(valid))[:, None]
        x = x + pe[None] * keep[..., None]
    if not cfg["layer_norm_first"]:
        x = F.layer_norm(x, (C,), sd["encoder.layer_norm.weight"].double(), sd["encoder.layer_norm.bias"].double(), 1e-5)
    return x


def mae_ast_forward(wavs: Sequence[torch.Tensor], sd: Dict[str, torch.Tensor], cfg: Dict,
                    layers: Optional[int] = None) -> List[torch.Tensor]:
    """The hidden states (fp64) of the reference expert: [B, T', nv * 768] per encoder layer."""
    kind = cfg["kind"]
    a = frontend(wavs, sd, kind)
    B, N, _ = a.shape
    nv = 128 // KINDS[kind][1]
    valid = valid_tokens([len(w) for w in wavs], kind, N // nv)
    key_valid = torch.arange(N)[None, :] < torch.tensor(valid)[:, None]
    x = embed(a, sd, cfg, valid)
    out = []
    for l in range(cfg["layers"] if layers is None else layers):
        x = layer(x, sd, l, key_valid, cfg["layer_norm_first"])
        out.append(x.reshape(B, N // nv, nv * x.shape[-1]))
    return out
