"""Oracle for the rest of guided-diffusion's ImageNet UNet family (the 64 / 128 base models and the SuperResModel upsamplers):
oracle/unet_openai.py's UNetModel restatement extended with the two attention settings those networks use,
  QKVAttention (unet.py:361-389): q, k, v split before the heads (use_new_attention_order=True), and
  a fixed head count per block (unet.py:277-283, 452-453): with num_head_channels == -1 the input and middle blocks use
  num_heads heads and the output blocks num_heads_upsample (-1: num_heads).
Functional over a reference-layout state dict (oracle.unet_openai.init_state_dict: the parameter shapes do not depend on the
attention settings); any floating dtype (the tap tests run it in float64).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from oracle import unet_openai as UO


@dataclass
class ZooConfig(UO.OpenAIUNetConfig):
    num_heads: int = 1
    num_heads_upsample: int = -1
    use_new_attention_order: bool = False
    small_size: int = 0          # > 0: SuperResModel conditioned on a [B, 3, small_size, small_size] image (in_channels = 6)

    def heads(self, channels, upsample):
        """AttentionBlock.__init__'s head count (unet.py:277-283) for a block of the output path (upsample) or not"""
        if self.num_head_channels != -1:
            assert channels % self.num_head_channels == 0
            return channels // self.num_head_channels
        n = self.num_heads_upsample if upsample and self.num_heads_upsample != -1 else self.num_heads
        assert channels % n == 0
        return n

    def reference_kwargs(self):
        """keyword arguments of the reference UNetModel / SuperResModel (whose in_channels is the image's: 3)"""
        return dict(image_size=self.image_size, in_channels=3 if self.small_size else self.in_channels,
                    model_channels=self.model_channels, out_channels=self.out_channels, num_res_blocks=self.num_res_blocks,
                    attention_resolutions=self.attention_ds, dropout=0.0, channel_mult=self.channel_mult,
                    num_classes=self.num_classes, use_checkpoint=False, use_fp16=False, num_heads=self.num_heads,
                    num_head_channels=self.num_head_channels, num_heads_upsample=self.num_heads_upsample,
                    use_scale_shift_norm=True, resblock_updown=True, use_new_attention_order=self.use_new_attention_order)


def _gn(sd, name, x):
    return F.group_norm(x, 32, sd[name + ".weight"], sd[name + ".bias"], 1e-5)


def _resblock(sd, p, x, emb, up=False, down=False):
    # unet.py:236-256 with use_scale_shift_norm=True
    h = F.silu(_gn(sd, p + ".in_layers.0", x))
    if up:
        h, x = F.interpolate(h, scale_factor=2, mode="nearest"), F.interpolate(x, scale_factor=2, mode="nearest")
    elif down:
        h, x = F.avg_pool2d(h, 2, 2), F.avg_pool2d(x, 2, 2)
    h = F.conv2d(h, sd[p + ".in_layers.2.weight"], sd[p + ".in_layers.2.bias"], padding=1)
    emb_out = F.linear(F.silu(emb), sd[p + ".emb_layers.1.weight"], sd[p + ".emb_layers.1.bias"])[..., None, None]
    scale, shift = torch.chunk(emb_out, 2, dim=1)
    h = _gn(sd, p + ".out_layers.0", h) * (1 + scale) + shift
    h = F.conv2d(F.silu(h), sd[p + ".out_layers.3.weight"], sd[p + ".out_layers.3.bias"], padding=1)
    if (p + ".skip_connection.weight") in sd:
        x = F.conv2d(x, sd[p + ".skip_connection.weight"], sd[p + ".skip_connection.bias"])
    return x + h


def attention(sd, p, x, n_heads, new_order):
    """AttentionBlock._forward (unet.py:299-305) with QKVAttention (new_order) or QKVAttentionLegacy (:337-354)"""
    b, c, hh, ww = x.shape
    xf = x.reshape(b, c, -1)
    qkv = F.conv1d(_gn(sd, p + ".norm", xf), sd[p + ".qkv.weight"], sd[p + ".qkv.bias"])
    bs, width, length = qkv.shape
    ch = width // (3 * n_heads)
    if new_order:
        q, k, v = (t.reshape(bs * n_heads, ch, length) for t in qkv.chunk(3, dim=1))
    else:
        q, k, v = qkv.reshape(bs * n_heads, ch * 3, length).split(ch, dim=1)
    scale = 1 / math.sqrt(math.sqrt(ch))
    weight = torch.softmax(torch.einsum("bct,bcs->bts", q * scale, k * scale), dim=-1)
    a = torch.einsum("bts,bcs->bct", weight, v).reshape(bs, -1, length)
    h = F.conv1d(a, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])
    return (xf + h).reshape(b, c, hh, ww)


def forward(sd, x, t, cfg: ZooConfig, taps=None, y=None, low_res=None):
    """UNetModel.forward (unet.py:635-664), or SuperResModel.forward (:667-681) when cfg.small_size > 0, in the dtype of x"""
    dt = x.dtype
    sd = {k: v.to(device=x.device, dtype=dt) for k, v in sd.items()}
    if cfg.small_size:
        up = F.interpolate(low_res.to(dt), x.shape[2:], mode="bilinear", align_corners=False)
        x = torch.cat([x, up], dim=1)
    inp, mid, out, _ = UO.block_plan(cfg)
    half = cfg.model_channels // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32) / half).to(device=x.device, dtype=dt)
    args = t.to(dt)[:, None] * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    emb = F.linear(emb, sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    assert (y is not None) == (cfg.num_classes is not None)
    if cfg.num_classes is not None:
        emb = emb + sd["label_emb.weight"][y.long()]

    def tap(name, v):
        if taps is not None:
            taps[name] = v.detach().clone()
        return v

    def run(prefix, layers, h, upsample):
        for j, (kind, _cin, _cout) in enumerate(layers):
            p = f"{prefix}.{j}"
            if kind == "conv":
                h = F.conv2d(h, sd[p + ".weight"], sd[p + ".bias"], padding=1)
            elif kind == "attn":
                h = attention(sd, p, h, cfg.heads(h.shape[1], upsample), cfg.use_new_attention_order)
            else:
                h = _resblock(sd, p, h, emb, up=(kind == "res_up"), down=(kind == "res_down"))
        return h

    hs = []
    h = x
    for i, layers in enumerate(inp):
        h = tap(f"in.{i}", run(f"input_blocks.{i}", layers, h, False))
        hs.append(h)
    h = tap("mid", run("middle_block", mid, h, False))
    for i, layers in enumerate(out):
        h = tap(f"out.{i}", run(f"output_blocks.{i}", layers, torch.cat([h, hs.pop()], dim=1), True))
    h = F.silu(_gn(sd, "out.0", h))
    return F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)


def attention_blocks(cfg: ZooConfig):
    """[(tap name, resolution, channels, heads)] of every block that ends in an attention layer"""
    inp, mid, out, _ = UO.block_plan(cfg)
    res, found = cfg.image_size, []
    for i, layers in enumerate(inp):
        if layers[-1][0] == "attn":
            found.append((f"in.{i}", res, layers[-1][1], cfg.heads(layers[-1][1], False)))
        if layers[-1][0] == "res_down":
            res //= 2
    for i, layers in enumerate(out):
        if layers[-1][0] == "attn":
            found.append((f"out.{i}", res, layers[-1][1], cfg.heads(layers[-1][1], True)))
        if layers[-1][0] == "res_up":
            res *= 2
    return found
