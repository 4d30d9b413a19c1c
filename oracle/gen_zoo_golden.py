"""Fixtures for guided-diffusion's ImageNet UNet family: runs the UNMODIFIED reference UNetModel / SuperResModel / EncoderUNetModel
(fp32, CPU) with seeded random weights and writes
  tests/golden/zoo.npz            reduced-width nets, one per attention variant (new order; fixed heads of width 96, 48, 40 and
                                  80; num_heads_upsample != num_heads; 3 ResBlocks per level with a x3 level; class-conditional or
                                  not; head widths 128 and 192), B = 2; and the logits of the 64x64 and 128x128 classifiers
  tests/golden/zoo_published*.npz the four published shapes at B = 1 and full width: the 64x64 base (new attention order), the
                                  128x128 base (4 heads), the 64 -> 256 upsampler (4 heads: width 96 at 32 x 32) and the
                                  128 -> 512 upsampler (a fixed crop of its output).  Each file stays under 1 MB: the 64 -> 256
                                  output is stored as the top and bottom halves of its rows in two part files; ``load_published``
                                  puts them back together
Weights: oracle.unet_openai.init_state_dict(cfg, 1234) / ddnm_b200.weights.random_state_dict_classifier(shape, 1234).  Inputs are
regenerated from seeds by ``inputs`` below.  The reduced nets also check oracle/unet_zoo.py against the reference.

The reference modules come from the copy ``__graft_entry__.build()`` makes under oracle/_ref/, or from the reference checkout
given on the command line:

    python -m oracle.gen_zoo_golden [/path/to/reference]

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import os
import sys

import numpy as np
import torch

from oracle import unet_openai as UO
from oracle.unet_zoo import ZooConfig, forward

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_COPY = os.path.join(ROOT, "oracle", "_ref")
CROP = (slice(None), slice(None), slice(192, 320), slice(192, 320))   # of the 512 x 512 upsampler output
GOLDEN = os.path.join(ROOT, "tests", "golden")
# the published-shape fixtures: the main file, then the row halves of the 64 -> 256 upsampler's output
PUBLISHED_FILES = ("zoo_published.npz", "zoo_published.part1.npz", "zoo_published.part2.npz")
HALVES = ("up256_out_top", "up256_out_bottom")


def load_published(golden=GOLDEN):
    """the published-shape fixtures as one dict (key + "_t", "_labels", "_out")"""
    d = {}
    for f in PUBLISHED_FILES:
        d.update(np.load(os.path.join(golden, f)))
    d["up256_out"] = np.concatenate([d.pop(h) for h in HALVES], axis=2)
    return d


def _z(image_size, mc, nrb, mult, attn, head_ch=-1, heads=1, heads_up=-1, new=False, classes=None, out=6, small=0):
    return ZooConfig(image_size=image_size, model_channels=mc, num_res_blocks=nrb, channel_mult=mult, attention_resolutions=attn,
                     num_head_channels=head_ch, out_channels=out, in_channels=6 if small else 3, num_classes=classes,
                     num_heads=heads, num_heads_upsample=heads_up, use_new_attention_order=new, small_size=small)


# (fixture key, config, batch, input seed, t, labels or None)
def reduced_cases():
    return [("new64", _z(32, 64, 1, (1, 2, 2), (16, 8), head_ch=64, new=True), 2, 51, (20.0, 640.0), None),
            # 2 heads of 96 at 16 x 16 (tensor cores: a full then a partial k-block / N tile) and 8 x 8 (CUDA cores)
            ("h96", _z(32, 64, 1, (1, 3, 3), (16, 8), heads=2), 2, 52, (300.0, 999.0), None),
            # the same in the new order, output blocks with 4 heads of 48 (one partial k-block / N tile)
            ("h96_new_cc", _z(32, 64, 1, (1, 3, 3), (16, 8), heads=2, heads_up=4, new=True, classes=1000, out=3), 2, 53,
             (5.0, 450.0), (951, 7)),
            # 8 heads of 40 at 16 x 16, output blocks 4 heads of 80
            ("h40", _z(32, 64, 1, (1, 5), (16,), heads=8, heads_up=4), 2, 54, (120.0, 870.0), None),
            ("h40_new_cc", _z(32, 64, 1, (1, 5), (16,), heads=8, new=True, classes=1000), 2, 55, (700.0, 1.0), (388, 0)),
            # num_res_blocks 3 and a x3 level (192 channels: 6 per GroupNorm group)
            ("res3_cc", _z(32, 64, 3, (1, 2, 3), (16, 8), head_ch=64, classes=1000), 2, 56, (250.0, 30.0), (1, 999)),
            # one head of 128 at 32 x 32 and of 192 at 16 x 16, new order
            ("wide_new", _z(32, 64, 1, (2, 3), (32, 16), heads=1, new=True), 2, 57, (60.0, 930.0), None)]


def published_cases():
    return [("base64", _z(64, 192, 3, (1, 2, 3, 4), (32, 16, 8), head_ch=64, new=True, classes=1000), 1, 61, (500.0,), (88,)),
            ("base128", _z(128, 256, 2, (1, 1, 2, 3, 4), (32, 16, 8), heads=4, classes=1000), 1, 62, (500.0,), (207,)),
            ("up256", _z(256, 192, 2, (1, 1, 2, 2, 4, 4), (32, 16, 8), heads=4, classes=1000, small=64), 1, 63, (400.0,), (279,)),
            ("up512", _z(512, 192, 2, (1, 1, 2, 2, 4, 4), (32, 16), head_ch=64, classes=1000, small=128), 1, 64, (400.0,), (979,))]


def classifier_cases():
    """(key, ClassifierConfig, batch, input seed, t): create_classifier(64 | 128, width 128, depth 4 | 2, "32,16,8", attention pool)"""
    from oracle.classifier import ClassifierConfig
    return [("cls64", ClassifierConfig(64, 128, 1000, 4, (2, 4, 8), (1, 2, 3, 4), 64, "attention"), 1, 71, (300.0,)),
            ("cls128", ClassifierConfig(128, 128, 1000, 2, (4, 8, 16), (1, 1, 2, 3, 4), 64, "attention"), 1, 72, (300.0,))]


def inputs(cfg, B, seed):
    """(x_t [B,3,R,R], low_res [B,3,s,s] or None) regenerated from the seed"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=g)
    low = torch.rand(B, 3, cfg.small_size, cfg.small_size, generator=g) * 2 - 1 if cfg.small_size else None
    return x, low


def state_dict(cfg, seed=1234):
    return UO.init_state_dict(cfg, seed)


def _reference(ref_root):
    root = ref_root or REF_COPY
    if not os.path.isfile(os.path.join(root, "guided_diffusion", "unet.py")):
        raise FileNotFoundError(f"no reference guided_diffusion/unet.py under {root}: run __graft_entry__.build() first")
    if root not in sys.path:
        sys.path.insert(0, root)
    from guided_diffusion import unet
    return unet


def _run_ref(unet, cfg, sd, x, t, low, y):
    cls = unet.SuperResModel if cfg.small_size else unet.UNetModel
    ref = cls(**cfg.reference_kwargs()).eval()
    ref.load_state_dict(sd)
    kw = {} if low is None else {"low_res": low}
    if y is not None:
        kw["y"] = y
    with torch.no_grad():
        return ref(x, t, **kw)


def main(ref_root=None):
    unet = _reference(ref_root)
    torch.set_num_threads(os.cpu_count() or 1)
    out = {}
    for key, cfg, B, seed, t, labels in reduced_cases():
        sd = state_dict(cfg)
        x, low = inputs(cfg, B, seed)
        tt, y = torch.tensor(t), None if labels is None else torch.tensor(labels)
        r = _run_ref(unet, cfg, sd, x, tt, low, y)
        with torch.no_grad():
            o = forward(sd, x, tt, cfg, y=y, low_res=low)
        err = (o - r).abs().max().item()
        assert torch.allclose(o, r, rtol=1e-4, atol=1e-5), err
        out[key + "_t"] = np.array(t, np.float32)
        if y is not None:
            out[key + "_labels"] = np.array(labels, np.int64)
        out[key + "_out"] = r.numpy()
        print(key, tuple(r.shape), "max|out|", r.abs().max().item(), "oracle-ref", err, flush=True)
    from ddnm_b200.weights import random_state_dict_classifier
    from oracle.gen_classifier_golden import shape
    for key, cfg, B, seed, t in classifier_cases():
        ref = unet.EncoderUNetModel(**cfg.kwargs()).eval()
        ref.load_state_dict(random_state_dict_classifier(shape(cfg), 1234))
        x = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(seed))
        with torch.no_grad():
            logits = ref(x, torch.tensor(t))
        out[key + "_t"], out[key + "_logits"] = np.array(t, np.float32), logits.numpy()
        print(key, "max|logits|", logits.abs().max().item(), flush=True)
    np.savez_compressed(os.path.join(GOLDEN, "zoo.npz"), **out)
    pub = {}
    for key, cfg, B, seed, t, labels in published_cases():
        sd = state_dict(cfg)
        x, low = inputs(cfg, B, seed)
        r = _run_ref(unet, cfg, sd, x, torch.tensor(t), low, torch.tensor(labels))
        pub[key + "_t"], pub[key + "_labels"] = np.array(t, np.float32), np.array(labels, np.int64)
        pub[key + "_out"] = (r[CROP] if key == "up512" else r).numpy()
        print(key, tuple(r.shape), "max|out|", r.abs().max().item(), flush=True)
        del sd, r
    up = pub.pop("up256_out")
    rows = up.shape[2] // 2
    np.savez_compressed(os.path.join(GOLDEN, PUBLISHED_FILES[0]), **pub)
    np.savez_compressed(os.path.join(GOLDEN, PUBLISHED_FILES[1]), **{HALVES[0]: up[:, :, :rows]})
    np.savez_compressed(os.path.join(GOLDEN, PUBLISHED_FILES[2]), **{HALVES[1]: up[:, :, rows:]})


if __name__ == "__main__":
    if len(sys.argv) > 2:
        sys.exit(__doc__)
    sys.path.insert(0, ROOT)
    main(sys.argv[1] if len(sys.argv) == 2 else None)
