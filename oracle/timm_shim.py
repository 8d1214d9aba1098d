"""TEST INFRASTRUCTURE — a minimal stand-in for timm 0.4.5, so that the reference's SSAST (s3prl/upstream/ssast/
ast_models.py) can be executed where timm is not installed. Written from the published architecture of the DeiT models
(Touvron et al., "Training data-efficient image transformers & distillation through attention", 2021) and timm's public
interface, not from timm's sources.

``install()`` registers the modules ``timm``, ``timm.models``, ``timm.models.layers`` and
``timm.models.vision_transformer`` only when ``import timm`` fails, and returns whether it did. They expose what
ASTModel uses: ``__version__ == "0.4.5"``, ``create_model`` for the DeiT names it asks for, ``to_2tuple`` /
``trunc_normal_`` and ``PatchEmbed`` (which ASTModel replaces with its own before calling ``create_model``: the model
looks the class up at construction time, as timm's does). A block is x + attn(norm1(x)), then x + mlp(norm2(x)):
LayerNorm eps 1e-6, one qkv Linear with bias whose output splits as (3, heads, head_dim), softmax(q k^T / sqrt(head_dim))
v, proj; mlp = fc1 -> exact GELU -> fc2 at 4x width. Nothing in the product package imports this module.
"""
from __future__ import annotations

import collections.abc
import math
import sys
import types
from functools import partial

import torch
import torch.nn as nn


def to_2tuple(x):
    if isinstance(x, collections.abc.Iterable) and not isinstance(x, str):
        return tuple(x)
    return (x, x)


def trunc_normal_(tensor: torch.Tensor, mean: float = 0.0, std: float = 1.0, a: float = -2.0, b: float = 2.0):
    with torch.no_grad():
        return nn.init.trunc_normal_(tensor, mean=mean, std=std, a=a, b=b)


class PatchEmbed(nn.Module):
    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768):
        super().__init__()
        img_size, patch_size = to_2tuple(img_size), to_2tuple(patch_size)
        self.img_size, self.patch_size = img_size, patch_size
        self.num_patches = (img_size[0] // patch_size[0]) * (img_size[1] // patch_size[1])
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class Attention(nn.Module):
    def __init__(self, dim, num_heads):
        super().__init__()
        self.num_heads = num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.proj = nn.Linear(dim, dim)

    def forward(self, x):
        B, N, C = x.shape
        qkv = self.qkv(x).reshape(B, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        attn = ((q @ k.transpose(-2, -1)) * self.scale).softmax(dim=-1)
        return self.proj((attn @ v).transpose(1, 2).reshape(B, N, C))


class Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1, self.act, self.fc2 = nn.Linear(dim, hidden), nn.GELU(), nn.Linear(hidden, dim)

    def forward(self, x):
        return self.fc2(self.act(self.fc1(x)))


class Block(nn.Module):
    def __init__(self, dim, num_heads, norm_layer):
        super().__init__()
        self.norm1, self.attn = norm_layer(dim), Attention(dim, num_heads)
        self.norm2, self.mlp = norm_layer(dim), Mlp(dim, 4 * dim)

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


class VisionTransformer(nn.Module):
    """DeiT (distilled: a dist_token and a head_dist next to the class token and its head)."""

    def __init__(self, img_size, embed_dim, depth, num_heads, distilled, num_classes=1000):
        super().__init__()
        norm_layer = partial(nn.LayerNorm, eps=1e-6)
        self.patch_embed = sys.modules[__name__ + ".vision_transformer"].PatchEmbed(
            img_size=img_size, patch_size=16, in_chans=3, embed_dim=embed_dim)
        ntok = 2 if distilled else 1
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.dist_token = nn.Parameter(torch.zeros(1, 1, embed_dim)) if distilled else None
        self.pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches + ntok, embed_dim))
        self.pos_drop = nn.Dropout(p=0.0)
        self.blocks = nn.ModuleList([Block(embed_dim, num_heads, norm_layer) for _ in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.head = nn.Linear(embed_dim, num_classes)
        self.head_dist = nn.Linear(embed_dim, num_classes) if distilled else None
        for p in (self.cls_token, self.pos_embed) + ((self.dist_token,) if distilled else ()):
            trunc_normal_(p, std=0.02)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)


# name -> (img_size, embed_dim, depth, num_heads, distilled): the DeiT models ASTModel asks for
_MODELS = {
    "vit_deit_tiny_distilled_patch16_224": (224, 192, 12, 3, True),
    "vit_deit_small_distilled_patch16_224": (224, 384, 12, 6, True),
    "vit_deit_base_distilled_patch16_384": (384, 768, 12, 12, True),
    "vit_deit_base_patch16_384": (384, 768, 12, 12, False),
}


def create_model(name: str, pretrained: bool = False, **kwargs):
    if pretrained:
        raise RuntimeError("timm_shim: pretrained weights are not available")
    if name not in _MODELS:
        raise KeyError(f"timm_shim: unknown model {name!r}")
    img, dim, depth, heads, distilled = _MODELS[name]
    return VisionTransformer(img, dim, depth, heads, distilled)


def install() -> bool:
    """Register the stand-in as ``timm`` when timm cannot be imported. Returns True when the stand-in is in use."""
    try:
        import timm  # noqa: F401
    except ImportError:
        pass
    else:
        return getattr(sys.modules.get("timm"), "__shim__", False)
    timm = types.ModuleType("timm")
    timm.__version__ = "0.4.5"
    timm.__shim__ = True
    timm.create_model = create_model
    models = types.ModuleType("timm.models")
    layers = types.ModuleType("timm.models.layers")
    layers.to_2tuple, layers.trunc_normal_ = to_2tuple, trunc_normal_
    vt = types.ModuleType("timm.models.vision_transformer")
    vt.PatchEmbed = PatchEmbed
    vt.VisionTransformer = VisionTransformer
    models.layers, models.vision_transformer = layers, vt
    timm.models = models
    sys.modules.update({"timm": timm, "timm.models": models, "timm.models.layers": layers,
                        "timm.models.vision_transformer": vt})
    # VisionTransformer looks PatchEmbed up here, where ASTModel's replacement lands
    sys.modules[__name__ + ".vision_transformer"] = vt
    return True
