"""Torch restatement of guided_diffusion/unet.py::EncoderUNetModel.forward (unet.py:684-895) for the variant create_classifier
builds for imagenet_256_cc.yml (use_scale_shift_norm, resblock_updown, legacy attention in the blocks, AttentionPool2d with
QKVAttention, or the adaptive head), and of the cond_fn the runner builds from it with autograd (diffusion.py:183-189).
Functional over a state dict in the reference checkpoint layout; any dtype (the tests use float64)."""
import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F


@dataclass
class ClassifierConfig:
    image_size: int = 256
    model_channels: int = 128
    out_channels: int = 1000
    num_res_blocks: int = 2
    attention_resolutions: tuple = (8, 16, 32)   # downsample rates
    channel_mult: tuple = (1, 1, 2, 2, 4, 4)
    num_head_channels: int = 64
    pool: str = "attention"

    @staticmethod
    def tiny():
        return ClassifierConfig(32, 64, 1000, 1, (2, 4), (1, 2, 2), 64, "attention")

    @staticmethod
    def imagenet_256():
        return ClassifierConfig()

    def kwargs(self):
        """keyword arguments of EncoderUNetModel (the reference class and ddnm_b200.model.EncoderUNetModel)"""
        return dict(image_size=self.image_size, in_channels=3, model_channels=self.model_channels, out_channels=self.out_channels,
                    num_res_blocks=self.num_res_blocks, attention_resolutions=self.attention_resolutions, channel_mult=self.channel_mult,
                    num_head_channels=self.num_head_channels, use_scale_shift_norm=True, resblock_updown=True, pool=self.pool)


def _up(x):
    """x in at least fp32 (GroupNorm32 / the attention softmax of a fp16 torso)"""
    return x.to(torch.promote_types(x.dtype, torch.float32))


def _gn(x, sd, p):
    return F.group_norm(_up(x), 32, sd[p + ".weight"], sd[p + ".bias"], 1e-5).to(x.dtype)


def _res(sd, p, x, emb, down):
    h = F.silu(_gn(x, sd, p + ".in_layers.0"))
    if down:
        h, x = F.avg_pool2d(h, 2), F.avg_pool2d(x, 2)
    h = F.conv2d(h, sd[p + ".in_layers.2.weight"], sd[p + ".in_layers.2.bias"], padding=1)
    e = F.linear(F.silu(emb), sd[p + ".emb_layers.1.weight"], sd[p + ".emb_layers.1.bias"])
    scale, shift = e[:, :, None, None].to(h.dtype).chunk(2, dim=1)
    h = _gn(h, sd, p + ".out_layers.0") * (1 + scale) + shift
    h = F.conv2d(F.silu(h), sd[p + ".out_layers.3.weight"], sd[p + ".out_layers.3.bias"], padding=1)
    if p + ".skip_connection.weight" in sd:
        x = F.conv2d(x, sd[p + ".skip_connection.weight"], sd[p + ".skip_connection.bias"])
    return x + h


def _attn(sd, p, x, ch):
    b, c, H, W = x.shape
    qkv = F.conv1d(_gn(x, sd, p + ".norm").reshape(b, c, -1), sd[p + ".qkv.weight"], sd[p + ".qkv.bias"])
    heads = c // ch
    q, k, v = qkv.reshape(b * heads, 3 * ch, -1).split(ch, dim=1)      # QKVAttentionLegacy (unet.py:337-354)
    s = 1 / math.sqrt(math.sqrt(ch))
    w = torch.softmax(_up(torch.einsum("bct,bcs->bts", q * s, k * s)), dim=-1).to(q.dtype)
    a = torch.einsum("bts,bcs->bct", w, v).reshape(b, -1, H * W)
    h = F.conv1d(a, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])
    return x + h.reshape(b, c, H, W)


_CONV = (".in_layers.2.", ".out_layers.3.", ".skip_connection.", ".qkv.", ".proj_out.", "input_blocks.0.0.")


def forward(sd, x, t, cfg, torso_dtype=None):
    """torso_dtype: run input_blocks + middle_block with their convolutions in that dtype (convert_to_fp16, unet.py:859-864 with
    fp16_util.convert_module_to_f16: only Conv layers are cast; GroupNorm32 and the attention softmax compute in fp32)"""
    if torso_dtype is not None:
        sd = {k: v.to(torso_dtype) if k.startswith(("input_blocks", "middle_block")) and any(c in k for c in _CONV) else v
              for k, v in sd.items()}
    return _forward(sd, x, t, cfg, torso_dtype)


def _forward(sd, x, t, cfg, torso_dtype):
    mc = cfg.model_channels
    half = mc // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float64) / half).to(x)
    args = t.to(x.dtype)[:, None] * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    emb = F.linear(F.silu(F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    h = F.conv2d(x.to(torso_dtype or x.dtype), sd["input_blocks.0.0.weight"], sd["input_blocks.0.0.bias"], padding=1)
    ds, idx, ch = 1, 1, cfg.num_head_channels
    for level, _ in enumerate(cfg.channel_mult):
        for _ in range(cfg.num_res_blocks):
            h = _res(sd, f"input_blocks.{idx}.0", h, emb, False)
            if ds in cfg.attention_resolutions:
                h = _attn(sd, f"input_blocks.{idx}.1", h, ch)
            idx += 1
        if level != len(cfg.channel_mult) - 1:
            h = _res(sd, f"input_blocks.{idx}.0", h, emb, True)
            idx += 1
            ds *= 2
    h = _res(sd, "middle_block.0", h, emb, False)
    h = _attn(sd, "middle_block.1", h, ch)
    h = _res(sd, "middle_block.2", h, emb, False).to(x.dtype)
    h = F.silu(_gn(h, sd, "out.0"))
    b, c = h.shape[:2]
    if cfg.pool == "adaptive":
        return F.conv2d(h.mean(dim=(2, 3), keepdim=True), sd["out.3.weight"], sd["out.3.bias"]).flatten(1)
    # AttentionPool2d (unet.py:20-50) with QKVAttention (unet.py:357-393)
    h = h.reshape(b, c, -1)
    h = torch.cat([h.mean(dim=-1, keepdim=True), h], dim=-1) + sd["out.2.positional_embedding"][None].to(h.dtype)
    qkv = F.conv1d(h, sd["out.2.qkv_proj.weight"], sd["out.2.qkv_proj.bias"])
    heads, T = c // ch, h.shape[-1]
    q, k, v = qkv.chunk(3, dim=1)
    s = 1 / math.sqrt(math.sqrt(ch))
    w = torch.softmax(torch.einsum("bct,bcs->bts", (q * s).reshape(b * heads, ch, T), (k * s).reshape(b * heads, ch, T)), dim=-1)
    a = torch.einsum("bts,bcs->bct", w, v.reshape(b * heads, ch, T)).reshape(b, -1, T)
    return F.conv1d(a, sd["out.2.c_proj.weight"], sd["out.2.c_proj.bias"])[:, :, 0]


def cond_fn(sd, cfg, scale, torso_dtype=None):
    """the reference's cond_fn(x, t, y) (diffusion.py:183-189) over this restatement"""
    if torso_dtype is not None:
        sd = {k: v.to(torso_dtype) if k.startswith(("input_blocks", "middle_block")) and any(c in k for c in _CONV) else v
              for k, v in sd.items()}
    def fn(x, t, y):
        with torch.enable_grad():
            x_in = x.detach().requires_grad_(True)
            logits = _forward(sd, x_in, t, cfg, torso_dtype)
            selected = F.log_softmax(logits, dim=-1)[range(len(logits)), y.view(-1)]
            return torch.autograd.grad(selected.sum(), x_in)[0] * scale
    return fn
