"""Writes tests/golden/classifier.npz: logits and cond_fn gradients of the UNMODIFIED reference EncoderUNetModel (unet.py:684-895,
fp32, CPU) with ddnm_b200.weights.random_state_dict_classifier(seed 1234) weights: the tiny classifier config (every layer kind:
skip conv, down ResBlock, tensor-core and CUDA-core attention sizes, T = 65 attention pool) at B = 2 with two t / label sets, the
same with the adaptive pool, and the imagenet_256_cc.yml classifier at B = 1 (its gradient in classifier.part1.npz, under 1 MB).  Inputs are regenerated from seeds
by ``inputs`` below.  Also asserts that oracle/classifier.py agrees with the reference.

    python -m oracle.gen_classifier_golden /path/to/reference"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def inputs(B, seed, size=32):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, size, size, generator=g)


def shape(cfg):
    """the attributes random_state_dict_classifier reads"""
    class Shape:
        model_channels, channel_mult, in_channels, num_res_blocks = cfg.model_channels, cfg.channel_mult, 3, cfg.num_res_blocks
        attention_resolutions, pool, image_size, out_channels = cfg.attention_resolutions, cfg.pool, cfg.image_size, cfg.out_channels
    return Shape


# (fixture key, config, batch, input seed, t, labels, scale)
def cases():
    from oracle.classifier import ClassifierConfig
    tiny = ClassifierConfig.tiny()
    adaptive = ClassifierConfig.tiny()
    adaptive.pool = "adaptive"
    return [("s11", tiny, 2, 11, (10.0, 700.0), (3, 951), 2.0),
            ("s12", tiny, 2, 12, (500.0, 500.0), (951, 0), 1.0),
            ("adaptive", adaptive, 2, 13, (250.0, 900.0), (951, 42), 1.0),
            ("full", ClassifierConfig.imagenet_256(), 1, 31, (600.0,), (951,), 10.0)]


def main(ref_root):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, ref_root)
    from guided_diffusion.unet import EncoderUNetModel
    from ddnm_b200.weights import random_state_dict_classifier
    from oracle import classifier as OC

    out, parts = {}, {}
    for key, cfg, B, seed, t, labels, scale in cases():
        ref = EncoderUNetModel(**cfg.kwargs()).eval()
        sd = random_state_dict_classifier(shape(cfg), 1234)
        ref.load_state_dict(sd)
        x = inputs(B, seed, cfg.image_size)
        tt, y = torch.tensor(t), torch.tensor(labels)
        with torch.enable_grad():
            x_in = x.detach().requires_grad_(True)
            logits = ref(x_in, tt)
            sel = torch.log_softmax(logits, dim=-1)[range(B), y]
            grad = torch.autograd.grad(sel.sum(), x_in)[0] * scale
        sd64 = {k: v.double() for k, v in sd.items()}
        with torch.no_grad():
            ol = OC.forward(sd64, x.double(), tt.double(), cfg)
        og = OC.cond_fn(sd64, cfg, scale)(x.double(), tt.double(), y)
        assert torch.allclose(ol, logits.double(), rtol=1e-4, atol=1e-5), (ol - logits).abs().max()
        assert torch.allclose(og, grad.double(), rtol=1e-3, atol=1e-4 * grad.abs().max().item()), (og - grad).abs().max()
        out[key + "_t"], out[key + "_labels"], out[key + "_scale"] = np.array(t, np.float32), np.array(labels, np.int64), np.float32(scale)
        out[key + "_logits"] = logits.detach().numpy()
        (parts if cfg.image_size > 32 else out)[key + "_grad"] = grad.numpy()   # full-size gradient: its own part file
        print(key, "max|grad|", grad.abs().max().item(), "oracle(fp64)-ref", (og - grad).abs().max().item(),
              "logits", (ol - logits).abs().max().item())
    for i, (k, v) in enumerate(sorted(parts.items())):
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", f"classifier.part{i + 1}.npz"), **{k: v})
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "classifier.npz"), **out)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
