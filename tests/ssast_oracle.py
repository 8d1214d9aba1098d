"""fp64 CPU restatement of SSAST's forward (s3prl/upstream/ssast/{expert,audio,ast_models}.py) on the tensors the
library reads (s3prl_b200.upstream.ssast.prepare_ssast_tensors: timm names, positional table re-gridded to the
window): every utterance zero-padded to nseg windows, kaldi fbank of each window (DC removal, pre-emphasis 0.97 with
the first sample replicated, hann(400, periodic=False), 512-point power spectrum, 128 mel bins 20 Hz..Nyquist,
log(max(E, float eps))), (y + 4.2677393) / 9.1379948, zero rows up to target_length; the patch embedding, class tokens
and positional table; 12 pre-LN DeiT blocks with LayerNorm eps 1e-6; each block's output without the class tokens,
frequency patches folded into channels, trimmed to the reference's frame count."""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

WIN, SHIFT, NFFT, NMEL, SR = 400, 160, 512, 128, 16000
FLOOR = torch.finfo(torch.float32).eps


def mel_banks(dtype=torch.float64) -> torch.Tensor:
    """get_mel_banks(128 bins, 512-point FFT, 16 kHz, low 20 Hz, high = Nyquist) -> [128, 257]."""
    mel_low, mel_high = 1127.0 * math.log(1.0 + 20.0 / 700.0), 1127.0 * math.log(1.0 + 8000.0 / 700.0)
    delta = (mel_high - mel_low) / (NMEL + 1)
    b = torch.arange(NMEL, dtype=dtype).unsqueeze(1)
    left, center, right = mel_low + b * delta, mel_low + (b + 1.0) * delta, mel_low + (b + 2.0) * delta
    mel = 1127.0 * (1.0 + (SR / NFFT) * torch.arange(NFFT // 2, dtype=dtype) / 700.0).log()
    w = torch.min((mel - left) / (center - left), (right - mel) / (right - center)).clamp(min=0.0)
    return F.pad(w, (0, 1))


def window_fbank(seg: torch.Tensor, TL: int) -> torch.Tensor:
    """The normalised features [TL, 128] of one window of S samples (fp64)."""
    m = 1 + (len(seg) - WIN) // SHIFT
    frames = seg.double().unfold(0, WIN, SHIFT)[:m]
    d = frames - frames.mean(dim=1, keepdim=True)
    prev = torch.cat([d[:, :1], d[:, :-1]], dim=1)
    y = (d - 0.97 * prev) * torch.hann_window(WIN, periodic=False, dtype=torch.float64)
    P = torch.fft.rfft(F.pad(y, (0, NFFT - WIN))).abs().pow(2)
    f = (P @ mel_banks().T).clamp(min=FLOOR).log()
    f = (f + 4.2677393) / (4.5689974 * 2)
    return F.pad(f, (0, 0, 0, TL - m))


def fbank_windows(wavs: Sequence[torch.Tensor], S: int, max_len: int) -> torch.Tensor:
    """[B * nseg, TL, 128], row block b * nseg + s = window s of utterance b."""
    nseg = len(range(0, max_len, S))
    out = []
    for w in wavs:
        x = torch.zeros(nseg * S, dtype=torch.float64)
        x[: len(w)] = w.double()
        out += [window_fbank(x[s * S:(s + 1) * S], S // SHIFT) for s in range(nseg)]
    return torch.stack(out)


def patch_operand(feat: torch.Tensor, kind: str) -> torch.Tensor:
    """The patch GEMM's A rows: frame model [SB, TL, 128] itself; patch model [SB, P, 256], row fi * tdim + ti,
    column kf * 16 + kt = feat[sb, 10 ti + kt, 10 fi + kf]."""
    if kind == "frame":
        return feat
    x = feat.transpose(1, 2).unsqueeze(1)  # [SB, 1, 128, TL]
    cols = F.unfold(x, kernel_size=(16, 16), stride=(10, 10))  # [SB, 256, P], P in (f, t) row-major
    return cols.transpose(1, 2)


def embed(feat: torch.Tensor, sd: Dict[str, torch.Tensor]) -> torch.Tensor:
    """[cls, dist, patch_embed(x)] + pos_embed: [SB, 2 + P, 768] (fp64)."""
    x = feat.double().transpose(1, 2).unsqueeze(1)
    w = sd["patch_embed.proj.weight"].double()
    stride = (128, 1) if w.shape[2] == 128 else (10, 10)
    p = F.conv2d(x, w, sd["patch_embed.proj.bias"].double(), stride=stride).flatten(2).transpose(1, 2)
    SB = p.shape[0]
    tok = torch.cat([sd["cls_token"].double().expand(SB, -1, -1), sd["dist_token"].double().expand(SB, -1, -1), p], 1)
    return tok + sd["pos_embed"].double()


def block(x: torch.Tensor, sd: Dict[str, torch.Tensor], l: int, heads: int = 12) -> torch.Tensor:
    p = f"blocks.{l}."
    g = lambda k: sd[p + k].double()  # noqa: E731
    SB, N, C = x.shape
    h = F.layer_norm(x, (C,), g("norm1.weight"), g("norm1.bias"), 1e-6)
    qkv = F.linear(h, g("attn.qkv.weight"), g("attn.qkv.bias")).reshape(SB, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    a = ((qkv[0] @ qkv[1].transpose(-2, -1)) * (C // heads) ** -0.5).softmax(-1)
    x = x + F.linear((a @ qkv[2]).transpose(1, 2).reshape(SB, N, C), g("attn.proj.weight"), g("attn.proj.bias"))
    h = F.layer_norm(x, (C,), g("norm2.weight"), g("norm2.bias"), 1e-6)
    return x + F.linear(F.gelu(F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias"))), g("mlp.fc2.weight"), g("mlp.fc2.bias"))


def fold(x: torch.Tensor, B: int, f_dim: int, T: int) -> torch.Tensor:
    """[B * nseg, 2 + P, D] -> [B, T, f_dim * D]: class tokens dropped, (f, t) patches to (t, f * D), trimmed."""
    SB, N, D = x.shape
    nseg = SB // B
    h = x[:, 2:, :].reshape(SB, f_dim, -1, D).transpose(1, 2).flatten(2)  # [SB, tdim, f_dim * D]
    return h.reshape(B, nseg * h.shape[1], f_dim * D)[:, :T]


def ssast_forward(wavs: Sequence[torch.Tensor], sd: Dict[str, torch.Tensor], kind: str, window_secs: float,
                  max_len: int = None) -> List[torch.Tensor]:
    """The 12 hidden states (fp64) of the reference's SSAST expert."""
    from s3prl_b200.upstream.ssast import geometry

    g = geometry(kind, window_secs)
    L = max_len or max(len(w) for w in wavs)
    T = min(len(range(0, L, g["S"])) * g["t_dim"], len(range(0, L, g["rate"])))
    x = embed(fbank_windows(wavs, g["S"], L), sd)
    hidden = []
    for l in range(12):
        x = block(x, sd, l)
        hidden.append(fold(x, len(wavs), g["f_dim"], T))
    return hidden
