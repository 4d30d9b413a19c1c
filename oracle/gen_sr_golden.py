"""Super-resolution UNet (guided_diffusion/unet.py::SuperResModel, :667-681) fixtures: writes tests/golden/superres.npz with the
outputs of the UNMODIFIED reference module (fp32, CPU) for random weights (oracle.unet_openai.init_state_dict, seed 1234) at small
channel counts, 32 -> 64 and 64 -> 128, unconditional and class-conditional.  Inputs (x, t, low_res, labels) are regenerated from
seeds by ``inputs`` below.  Also asserts that ``forward`` (the torch restatement) agrees with the reference.

The reference module is imported from the copy ``__graft_entry__.build()`` makes under oracle/_ref/ (oracle/make_ref.py), or from
the reference checkout given on the command line:

    python -m oracle.gen_sr_golden [/path/to/reference]

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

from oracle import unet_openai as UO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_COPY = os.path.join(ROOT, "oracle", "_ref")


def config(large, small, class_cond, out_channels):
    """a small SuperResModel: 64 channels, one ResBlock per level, attention at 16 x 16; in_channels = 6 (x + upsampled low_res)"""
    mult = (1, 2, 2) if large == 64 else (1, 1, 2, 2)
    cfg = UO.OpenAIUNetConfig(image_size=large, model_channels=64, num_res_blocks=1, channel_mult=mult, attention_resolutions=(16,),
                              num_head_channels=64, out_channels=out_channels, in_channels=6,
                              num_classes=1000 if class_cond else None)
    cfg.small_size = small
    return cfg


# (fixture key, config, batch, input seed, t, labels or None)
def cases():
    return [("sr32", config(64, 32, False, 6), 2, 41, (20.0, 640.0), None),
            ("sr32_cc", config(64, 32, True, 3), 2, 42, (300.0, 999.0), (951, 7)),
            ("sr64", config(128, 64, False, 6), 1, 43, (450.0,), None),
            ("sr64_cc", config(128, 64, True, 3), 1, 44, (90.0,), (388,))]


def inputs(cfg, B, seed):
    """(x_t [B,3,L,L], low_res [B,3,s,s]) regenerated from the seed"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=g)
    low = torch.rand(B, 3, cfg.small_size, cfg.small_size, generator=g) * 2 - 1
    return x, low


def state_dict(cfg, seed=1234):
    return UO.init_state_dict(cfg, seed)


def forward(sd, x, t, low_res, cfg, y=None):
    """SuperResModel.forward restated: cat([x, interpolate(low_res, x.shape[2:], bilinear)]) into the UNetModel of cfg"""
    up = F.interpolate(low_res, x.shape[2:], mode="bilinear", align_corners=False)
    return UO.forward(sd, torch.cat([x, up.to(x.dtype)], dim=1), t, cfg, y=y)


def reference_class(ref_root=None):
    """guided_diffusion.unet.SuperResModel of the reference copy (oracle/_ref by default)"""
    root = ref_root or REF_COPY
    if not os.path.isfile(os.path.join(root, "guided_diffusion", "unet.py")):
        raise FileNotFoundError(f"no reference guided_diffusion/unet.py under {root}: run __graft_entry__.build() first")
    if root not in sys.path:
        sys.path.insert(0, root)
    from guided_diffusion.unet import SuperResModel
    return SuperResModel


def reference_kwargs(cfg):
    return dict(image_size=cfg.image_size, in_channels=3, model_channels=cfg.model_channels, out_channels=cfg.out_channels,
                num_res_blocks=cfg.num_res_blocks, attention_resolutions=cfg.attention_ds, dropout=0.0, channel_mult=cfg.channel_mult,
                num_classes=cfg.num_classes, use_checkpoint=False, use_fp16=False, num_heads=4, num_head_channels=cfg.num_head_channels,
                num_heads_upsample=-1, use_scale_shift_norm=True, resblock_updown=True)


def main(ref_root=None):
    SuperResModel = reference_class(ref_root)
    out = {}
    for key, cfg, B, seed, t, labels in cases():
        ref = SuperResModel(**reference_kwargs(cfg)).eval()
        sd = state_dict(cfg)
        ref.load_state_dict(sd)
        x, low = inputs(cfg, B, seed)
        tt = torch.tensor(t)
        y = None if labels is None else torch.tensor(labels)
        with torch.no_grad():
            r = ref(x, tt, low_res=low) if y is None else ref(x, tt, low_res=low, y=y)
            o = forward(sd, x, tt, low, cfg, y=y)
        err = (o - r).abs().max().item()
        assert torch.allclose(o, r, rtol=1e-4, atol=1e-5), err
        out[key + "_t"] = np.array(t, np.float32)
        if y is not None:
            out[key + "_labels"] = np.array(labels, np.int64)
        out[key + "_out"] = r.numpy()
        print(key, tuple(r.shape), "max|out|", r.abs().max().item(), "oracle-ref", err)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "superres.npz"), **out)


if __name__ == "__main__":
    if len(sys.argv) > 2:
        sys.exit(__doc__)
    sys.path.insert(0, ROOT)
    main(sys.argv[1] if len(sys.argv) == 2 else None)
