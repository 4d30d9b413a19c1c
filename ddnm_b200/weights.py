"""Synthetic (random-init) weights in the reference checkpoint layout, for benchmarks and smoke runs where the real
CelebA-HQ checkpoint cannot be downloaded.  Parameters are drawn exactly as ``torch.manual_seed(seed); Model(config)``
would draw them (same torch.nn layer types constructed in the order of guided_diffusion/models.py:216-299), so the
result equals the reference model's own ``state_dict()`` for that seed."""
import torch
import torch.nn as nn


def random_state_dict(config, seed=1234):
    m = config.model
    ch, out_ch, mult = int(m.ch), int(m.out_ch), tuple(int(v) for v in m.ch_mult)
    nrb, attn_res = int(m.num_res_blocks), tuple(int(v) for v in m.attn_resolutions)
    res = int(config.data.image_size)
    tch = 4 * ch
    sd = {}
    torch.manual_seed(seed)

    def take(prefix, module):
        for k, v in module.state_dict().items():
            sd[f"{prefix}.{k}"] = v.detach().clone()

    def res_block(prefix, cin, cout):
        take(prefix + ".norm1", nn.GroupNorm(32, cin, eps=1e-6))
        take(prefix + ".conv1", nn.Conv2d(cin, cout, 3, padding=1))
        take(prefix + ".temb_proj", nn.Linear(tch, cout))
        take(prefix + ".norm2", nn.GroupNorm(32, cout, eps=1e-6))
        take(prefix + ".conv2", nn.Conv2d(cout, cout, 3, padding=1))
        if cin != cout:
            take(prefix + ".nin_shortcut", nn.Conv2d(cin, cout, 1))

    def attn_block(prefix, c):
        take(prefix + ".norm", nn.GroupNorm(32, c, eps=1e-6))
        for leaf in ("q", "k", "v", "proj_out"):
            take(f"{prefix}.{leaf}", nn.Conv2d(c, c, 1))

    take("temb.dense.0", nn.Linear(ch, tch))
    take("temb.dense.1", nn.Linear(tch, tch))
    take("conv_in", nn.Conv2d(int(m.in_channels), ch, 3, padding=1))
    widths = [ch * v for v in mult]
    prev = [ch] + widths[:-1]
    cur = ch
    for lv, w in enumerate(widths):
        cur = prev[lv]
        for ib in range(nrb):
            res_block(f"down.{lv}.block.{ib}", cur, w)
            cur = w
            if res in attn_res:
                attn_block(f"down.{lv}.attn.{ib}", cur)
        if lv + 1 < len(widths):
            take(f"down.{lv}.downsample.conv", nn.Conv2d(cur, cur, 3, stride=2))
            res //= 2
    res_block("mid.block_1", cur, cur)
    attn_block("mid.attn_1", cur)
    res_block("mid.block_2", cur, cur)
    for lv in range(len(widths) - 1, -1, -1):
        w = widths[lv]
        for ib in range(nrb + 1):
            skip = prev[lv] if ib == nrb else w
            res_block(f"up.{lv}.block.{ib}", cur + skip, w)
            cur = w
            if res in attn_res:
                attn_block(f"up.{lv}.attn.{ib}", cur)
        if lv > 0:
            take(f"up.{lv}.upsample.conv", nn.Conv2d(cur, cur, 3, padding=1))
            res *= 2
    take("norm_out", nn.GroupNorm(32, cur, eps=1e-6))
    take("conv_out", nn.Conv2d(cur, out_ch, 3, padding=1))
    return sd


def random_state_dict_openai(model, seed=1234, zero_std=0.02):
    """Random-init weights for ``ddnm_b200.model.UNetModel`` in the reference checkpoint layout, drawn as
    ``torch.manual_seed(seed); create_model(...)`` draws them (layer construction order of unet.py:472-617).  The
    tensors the reference zero-initialises (ResBlock out conv, attention proj_out, final conv: unet.py:210-212,294,616)
    are re-drawn from N(0, zero_std) with generator seed+1, otherwise a random-init net would output exactly 0."""
    mc, tdim = model.model_channels, model.model_channels * 4
    sd, zero_keys = {}, []
    torch.manual_seed(seed)

    def take(prefix, module, zero=False):
        for k, v in module.state_dict().items():
            sd[f"{prefix}.{k}"] = v.detach().clone()
            if zero:
                zero_keys.append(f"{prefix}.{k}")

    def res_block(p, cin, cout):
        take(p + ".in_layers.0", nn.GroupNorm(32, cin))
        take(p + ".in_layers.2", nn.Conv2d(cin, cout, 3, padding=1))
        take(p + ".emb_layers.1", nn.Linear(tdim, 2 * cout))
        take(p + ".out_layers.0", nn.GroupNorm(32, cout))
        take(p + ".out_layers.3", nn.Conv2d(cout, cout, 3, padding=1), zero=True)
        if cin != cout:
            take(p + ".skip_connection", nn.Conv2d(cin, cout, 1))

    def attention(p, c):
        take(p + ".norm", nn.GroupNorm(32, c))
        take(p + ".qkv", nn.Conv1d(c, 3 * c, 1))
        take(p + ".proj_out", nn.Conv1d(c, c, 1), zero=True)

    take("time_embed.0", nn.Linear(mc, tdim))
    take("time_embed.2", nn.Linear(tdim, tdim))
    ch = int(model.channel_mult[0] * mc)
    first = ch
    take("input_blocks.0.0", nn.Conv2d(model.in_channels, ch, 3, padding=1))
    skip_chans, ds, idx = [ch], 1, 1
    nlev = len(model.channel_mult)
    for level, mult in enumerate(model.channel_mult):
        for _ in range(model.num_res_blocks):
            res_block(f"input_blocks.{idx}.0", ch, int(mult * mc))
            ch = int(mult * mc)
            if ds in model.attention_resolutions:
                attention(f"input_blocks.{idx}.1", ch)
            skip_chans.append(ch)
            idx += 1
        if level != nlev - 1:
            res_block(f"input_blocks.{idx}.0", ch, ch)
            skip_chans.append(ch)
            idx += 1
            ds *= 2
    res_block("middle_block.0", ch, ch)
    attention("middle_block.1", ch)
    res_block("middle_block.2", ch, ch)
    idx = 0
    for level in range(nlev - 1, -1, -1):
        mult = model.channel_mult[level]
        for i in range(model.num_res_blocks + 1):
            ich = skip_chans.pop()
            res_block(f"output_blocks.{idx}.0", ch + ich, int(mc * mult))
            ch = int(mc * mult)
            j = 1
            if ds in model.attention_resolutions:
                attention(f"output_blocks.{idx}.{j}", ch)
                j += 1
            if level and i == model.num_res_blocks:
                res_block(f"output_blocks.{idx}.{j}", ch, ch)
                ds //= 2
            idx += 1
    take("out.0", nn.GroupNorm(32, ch))
    take("out.2", nn.Conv2d(first, model.out_ch, 3, padding=1), zero=True)
    g = torch.Generator().manual_seed(seed + 1)
    for k in zero_keys:
        sd[k] = torch.randn(sd[k].shape, generator=g) * zero_std
    return sd


def random_state_dict_classifier(model, seed=1234, zero_std=0.02):
    """Random-init weights for ``ddnm_b200.model.EncoderUNetModel`` in the reference checkpoint layout, drawn in the layer
    construction order of unet.py:714-871 after ``torch.manual_seed(seed)``.  As in ``random_state_dict_openai``, the tensors the
    reference zero-initialises (ResBlock out conv, attention proj_out, the adaptive head's conv) are re-drawn from N(0, zero_std)
    with generator seed+1: with the reference's own init the input gradient of a random net is degenerate (max |d/dx| ~ 7e-6 at 256^2)."""
    mc, tdim = model.model_channels, model.model_channels * 4
    sd, zero_keys = {}, []
    torch.manual_seed(seed)

    def take(prefix, module, zero=False):
        for k, v in module.state_dict().items():
            sd[f"{prefix}.{k}"] = v.detach().clone()
            if zero:
                zero_keys.append(f"{prefix}.{k}")

    def res_block(p, cin, cout):
        take(p + ".in_layers.0", nn.GroupNorm(32, cin))
        take(p + ".in_layers.2", nn.Conv2d(cin, cout, 3, padding=1))
        take(p + ".emb_layers.1", nn.Linear(tdim, 2 * cout))
        take(p + ".out_layers.0", nn.GroupNorm(32, cout))
        take(p + ".out_layers.3", nn.Conv2d(cout, cout, 3, padding=1), zero=True)
        if cin != cout:
            take(p + ".skip_connection", nn.Conv2d(cin, cout, 1))

    def attention(p, c):
        take(p + ".norm", nn.GroupNorm(32, c))
        take(p + ".qkv", nn.Conv1d(c, 3 * c, 1))
        take(p + ".proj_out", nn.Conv1d(c, c, 1), zero=True)

    take("time_embed.0", nn.Linear(mc, tdim))
    take("time_embed.2", nn.Linear(tdim, tdim))
    ch = int(model.channel_mult[0] * mc)
    take("input_blocks.0.0", nn.Conv2d(model.in_channels, ch, 3, padding=1))
    ds, idx = 1, 1
    for level, mult in enumerate(model.channel_mult):
        for _ in range(model.num_res_blocks):
            res_block(f"input_blocks.{idx}.0", ch, int(mult * mc))
            ch = int(mult * mc)
            if ds in model.attention_resolutions:
                attention(f"input_blocks.{idx}.1", ch)
            idx += 1
        if level != len(model.channel_mult) - 1:
            res_block(f"input_blocks.{idx}.0", ch, ch)
            idx += 1
            ds *= 2
    res_block("middle_block.0", ch, ch)
    attention("middle_block.1", ch)
    res_block("middle_block.2", ch, ch)
    take("out.0", nn.GroupNorm(32, ch))
    if model.pool == "attention":
        T = (model.image_size // ds) ** 2 + 1
        sd["out.2.positional_embedding"] = torch.randn(ch, T) / ch ** 0.5
        take("out.2.qkv_proj", nn.Conv1d(ch, 3 * ch, 1))
        take("out.2.c_proj", nn.Conv1d(ch, model.out_channels, 1))
    else:
        take("out.3", nn.Conv2d(ch, model.out_channels, 1), zero=True)
    g = torch.Generator().manual_seed(seed + 1)
    for k in zero_keys:
        sd[k] = torch.randn(sd[k].shape, generator=g) * zero_std
    return sd
