"""Pin the oracle to the reference and write the committed fixtures under tests/golden/.

Runs ONLY in the build container (needs /root/reference).  For every fixture it (1) executes the
UNMODIFIED reference code (imported from /root/reference, with ``.to('cuda')`` redirected to CPU and
``torch.randn_like`` fed from a noise tape), (2) asserts the oracle restatement agrees, (3) stores the
reference's outputs.  tests/test_oracle_golden.py re-checks the oracle against these files everywhere;
tests/test_gpu_*.py check the CUDA engine against them on the H100.

    python -m oracle.gen_golden
"""
import os
import sys
import types

import numpy as np
import torch

REF = "/root/reference"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

from oracle import operators as O          # noqa: E402
from oracle import sampler as S            # noqa: E402
from oracle import schedule as SCH         # noqa: E402
from oracle import unet_simple as U        # noqa: E402
from oracle import unet_openai as UO       # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def save_split(stem, out, limit=950_000):
    """out as stem.npz (+ stem.part1.npz, ...): keys in order, a new file whenever the compressed size would pass `limit` bytes
    (tests/conftest.py merges the parts)."""
    import glob
    import io
    for old in glob.glob(stem + ".part*.npz"):
        os.remove(old)
    parts, cur = [], {}
    for k, v in out.items():
        cur[k] = v
        buf = io.BytesIO()
        np.savez_compressed(buf, **cur)
        if buf.tell() > limit and len(cur) > 1:
            del cur[k]
            parts.append(cur)
            cur = {k: v}
    parts.append(cur)
    for i, p in enumerate(parts):
        np.savez_compressed(stem + (".npz" if i == 0 else f".part{i}.npz"), **p)


def ns(**k):
    return types.SimpleNamespace(**k)


def ref_model(cfg, seed):
    from guided_diffusion.models import Model
    c = ns(model=ns(type="simple", ch=cfg.ch, out_ch=cfg.out_ch, ch_mult=list(cfg.ch_mult),
                    num_res_blocks=cfg.num_res_blocks, attn_resolutions=list(cfg.attn_resolutions), dropout=0.0,
                    in_channels=cfg.in_channels, resamp_with_conv=True),
           data=ns(image_size=cfg.resolution), diffusion=ns(num_diffusion_timesteps=1000))
    torch.manual_seed(seed)
    return Model(c).eval()


from oracle.ref_shim import cpu_shim      # noqa: E402,F401  (the .to('cuda') / randn_like redirection)


def close(a, b, tol, what):
    d = (a - b).abs().max().item()
    assert d <= tol, f"{what}: oracle deviates from reference by {d}"
    return d


# --------------------------------------------------------------------------------------------------
def unet_fixtures():
    out = {}
    for name, cfg, B in (("tiny", U.SimpleUNetConfig.tiny(), 2), ("celeba", U.SimpleUNetConfig.celeba_hq(), 1)):
        m = ref_model(cfg, 1234)
        sd = U.init_state_dict(cfg, 1234)
        assert all(torch.equal(sd[k], v) for k, v in m.state_dict().items()), "weight init differs"
        g = torch.Generator().manual_seed(99)
        x = torch.randn(B, 3, cfg.resolution, cfg.resolution, generator=g)
        t = torch.tensor([417.0, 3.0][:B])
        with torch.no_grad():
            r = m(x, t)
            taps = {}
            o = U.forward(sd, x, t, cfg, taps=taps)
        close(o, r, 0.0, f"unet {name}")
        out[f"{name}_t"] = t.numpy()
        if name == "tiny":
            out["tiny_x"] = x.numpy()
            out["tiny_out"] = r.numpy()
            for k in ("conv_in", "down.0.0", "down.0.ds", "down.1.0", "mid.attn_1", "up.1.us", "up.0.1"):
                out["tiny_tap_s2_" + k] = taps[k][:, :, ::2, ::2].contiguous().numpy()   # strided sample keeps the file < 1 MB
        else:
            # full 256x256 net: x is regenerated from the seed by the test; keep a strided sample of eps
            out["celeba_out_s8"] = r[:, :, ::8, ::8].contiguous().numpy()
            out["celeba_out_sum"] = np.array([r.double().sum().item(), r.double().abs().sum().item()])
        print(f"unet {name}: ok, out std {r.std().item():.4f}")
    np.savez_compressed(os.path.join(GOLD, "unet_simple.npz"), **out)


def ref_openai(cfg, seed):
    from guided_diffusion.script_util import create_model
    torch.manual_seed(seed)
    m = create_model(image_size=cfg.image_size, num_channels=cfg.model_channels, num_res_blocks=cfg.num_res_blocks,
                     channel_mult=",".join(str(c) for c in cfg.channel_mult), learn_sigma=(cfg.out_channels == 6),
                     class_cond=cfg.num_classes is not None,
                     attention_resolutions=",".join(str(r) for r in cfg.attention_resolutions), num_heads=4,
                     num_head_channels=cfg.num_head_channels, num_heads_upsample=-1, use_scale_shift_norm=True, dropout=0.0,
                     resblock_updown=True, use_fp16=False, use_new_attention_order=False)
    return m.eval()


def openai_fixtures():
    """imagenet_256.yml UNetModel in fp32 mode, zero-initialised tensors re-drawn (see oracle.unet_openai.init_state_dict)."""
    out = {}
    for name, cfg, B in (("tiny", UO.OpenAIUNetConfig.tiny(), 2), ("imagenet", UO.OpenAIUNetConfig.imagenet_256(), 1)):
        m = ref_openai(cfg, 1234)
        rsd = m.state_dict()
        sd = UO.init_state_dict(cfg, 1234)
        assert set(sd) == set(rsd)
        redrawn = 0
        for k in sd:
            if not torch.equal(sd[k], rsd[k]):
                assert rsd[k].abs().sum() == 0, f"{k}: differs from the reference but is not a zero-initialised tensor"
                redrawn += 1
        m.load_state_dict(sd)
        g = torch.Generator().manual_seed(99)
        x = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=g)
        t = torch.tensor([417.0, 3.0][:B])
        with torch.no_grad():
            r = m(x, t)
            taps = {}
            o = UO.forward(sd, x, t, cfg, taps=taps)
        close(o, r, 0.0, f"openai unet {name}")
        out[f"{name}_t"] = t.numpy()
        if name == "tiny":
            out["tiny_x"], out["tiny_out"] = x.numpy(), r.numpy()
            for k in ("in.0", "in.1", "in.2", "in.3", "mid", "out.0", "out.2", "out.5"):
                out["tiny_tap_s2_" + k] = taps[k][:, :, ::2, ::2].contiguous().numpy()   # strided sample keeps the file < 1 MB
        else:
            out["imagenet_out_s8"] = r[:, :, ::8, ::8].contiguous().numpy()
            out["imagenet_out_sum"] = np.array([r.double().sum().item(), r.double().abs().sum().item()])
        print(f"openai unet {name}: ok ({redrawn} zero-init tensors re-drawn), out std {r.std().item():.4f}")
    np.savez_compressed(os.path.join(GOLD, "unet_openai.npz"), **out)


# --------------------------------------------------------------------------------------------------
def _ref_inpainting(R, channels, img_dim, mask_flat):
    """The reference constructor's kept-index loop is O(N*missing) (svd_operators.py:330); build the
    same object through a boolean complement (identical kept/missing index tensors)."""
    mr = torch.nonzero(mask_flat == 0).long().reshape(-1) * 3          # diffusion.py:467-470
    missing = torch.cat([mr, mr + 1, mr + 2], dim=0)
    n = channels * img_dim ** 2
    r = R.Inpainting.__new__(R.Inpainting)
    r.channels, r.img_dim, r.missing_indices = channels, img_dim, missing
    r._singulars = torch.ones(n - missing.shape[0])
    keep = torch.ones(n, dtype=torch.bool)
    keep[missing] = False
    r.kept_indices = torch.nonzero(keep).reshape(-1)
    if img_dim <= 32:                                                     # small enough for the real loop
        rr = R.Inpainting(channels, img_dim, missing, "cpu")
        assert torch.equal(rr.kept_indices, r.kept_indices)
    return r


def gauss_kernel():
    # diffusion.py:504-509
    sigma = 10
    pdf = lambda z: torch.exp(torch.Tensor([-0.5 * (z / sigma) ** 2]))   # noqa: E731
    k = torch.Tensor([pdf(-2), pdf(-1), pdf(0), pdf(1), pdf(2)])
    return k / k.sum()


def build_ops(dim, rng):
    """(name, reference object, oracle object, artefact dict) for the six north-star operators at image size dim."""
    from functions import svd_operators as R
    ops = []
    r = R.SuperResolution(3, dim, 4, "cpu")
    ops.append(("sr4", r, O.SuperResolution(3, dim, 4, r.U_small, r.singulars_small, r.V_small),
                dict(U_small=r.U_small, singulars_small=r.singulars_small, V_small=r.V_small)))
    r = R.Colorization(dim, "cpu")
    ops.append(("color", r, O.Colorization(dim, r.U_small, r.singulars_small, r.V_small),
                dict(U_small=r.U_small, singulars_small=r.singulars_small, V_small=r.V_small)))
    if dim == 256:
        mask = np.load(os.path.join(REF, "exp/inp_masks/mask.npy"))
    else:
        mask = (torch.rand(dim, dim, generator=rng) > 0.3).long().numpy()
    r = _ref_inpainting(R, 3, dim, torch.from_numpy(mask).reshape(-1))
    ops.append(("inpaint", r, O.Inpainting(3, dim, mask), dict(mask=torch.from_numpy(mask))))
    perm = torch.randperm(dim ** 2, generator=rng)
    r = R.WalshHadamardCS(3, dim, 4, perm, "cpu")
    ops.append(("wh", r, O.WalshHadamardCS(3, dim, 4, perm), dict(perm=perm)))
    r = R.Deblurring(gauss_kernel(), 3, dim, "cpu")
    ops.append(("deblur", r, O.Deblurring(3, dim, r.U_small, r.V_small, r._singulars, r._singulars_orig, r._perm),
                dict(U_small=r.U_small, V_small=r.V_small, singulars=r._singulars, singulars_orig=r._singulars_orig,
                     perm=r._perm)))
    k = O.SRConv.bicubic_kernel(4)
    r = R.SRConv(k, 3, dim, "cpu", stride=4)
    ops.append(("bicubic", r, O.SRConv(3, dim, 4, r.U_small, r.singulars_small, r.V_small),
                dict(U_small=r.U_small, singulars_small=r.singulars_small, V_small=r.V_small)))
    ops.append(("denoise", R.Denoising(3, dim, "cpu"), O.Denoising(3, dim), dict()))
    grng = torch.random.get_rng_state()
    r = R.CS(3, dim, 0.25, "cpu")                     # its random basis is replaced by a machine-independent orthonormal one
    torch.random.set_rng_state(grng)
    r.V_small = O.hadamard_basis()
    r.Vt_small = r.V_small.transpose(0, 1)
    ops.append(("cs", r, O.CS(3, dim, 0.25, r.V_small), dict()))
    k1, k2 = aniso_kernels()
    r = R.Deblurring2D(k1, k2, 3, dim, "cpu")
    ops.append(("deblur2d", r, O.Deblurring2D(3, dim, r.U_small1, r.V_small1, r.U_small2, r.V_small2, r._singulars, r._perm),
                dict(U_small1=r.U_small1, V_small1=r.V_small1, U_small2=r.U_small2, V_small2=r.V_small2, singulars=r._singulars,
                     perm=r._perm)))
    return ops


def aniso_kernels():
    # diffusion.py:510-521 (deblur_aniso)
    def pdf(sigma):
        return lambda z: torch.exp(torch.Tensor([-0.5 * (z / sigma) ** 2]))
    k2 = torch.Tensor([pdf(20)(i) for i in range(-4, 5)])
    k1 = torch.Tensor([pdf(1)(i) for i in range(-4, 5)])
    return k1 / k1.sum(), k2 / k2.sum()


LAMBDA_CASES = [(0.9, 0.1, 0.3), (0.99, 0.1, 0.02), (1.0, 0.1, 0.0), (0.5, 0.0, 0.4)]   # (a, sigma_y, sigma_t)


def operator_fixtures():
    out = {}
    for dim, B in ((32, 2), (256, 1)):
        rng = torch.Generator().manual_seed(4321)
        x = torch.rand(B, 3, dim, dim, generator=rng) * 2 - 1
        v = torch.randn(B, 3 * dim * dim, generator=rng)
        e = torch.randn(B, 3 * dim * dim, generator=rng)
        tag = f"d{dim}"
        if dim == 32:
            out[f"{tag}_x"], out[f"{tag}_v"], out[f"{tag}_e"] = x.numpy(), v.numpy(), e.numpy()
        sub = (lambda z: z) if dim == 32 else (lambda z: z.reshape(B, -1)[:, ::61].contiguous())
        for name, r, o, art in build_ops(dim, rng):
            if dim == 32 or name in ("wh",):
                for k, a in art.items():
                    out[f"{tag}_{name}_art_{k}"] = a.numpy()
            y = r.A(x)
            close(o.A(x.reshape(B, -1)), y, 2e-6, f"{name} A")
            yq = y * 0.9 + 0.05
            pin = r.A_pinv(yq.clone())
            close(o.A_pinv(yq.clone()), pin, 2e-6, f"{name} A_pinv")
            proj = x - r.A_pinv(r.A(x.reshape(B, -1)) - yq.reshape(B, -1)).reshape(x.shape)
            close(o.project(x, yq), proj, 4e-6, f"{name} project")
            out[f"{tag}_{name}_A"] = sub(y).numpy()
            out[f"{tag}_{name}_Apinv"] = sub(pin).numpy()
            out[f"{tag}_{name}_proj"] = sub(proj).numpy()
            if name not in ("bicubic", "deblur2d", "cs"):
                for ci, (a, sy, st) in enumerate(LAMBDA_CASES):
                    at, stt = torch.tensor(a), torch.tensor(st)
                    L = r.Lambda(v.clone(), at, sy, stt, 0.85)
                    Ln = r.Lambda_noise(v.clone(), at, sy, stt, 0.85, e.clone())
                    close(o.Lambda(v.clone(), at, sy, stt, 0.85), L, 4e-6, f"{name} Lambda{ci}")
                    close(o.Lambda_noise(v.clone(), at, sy, stt, 0.85, e.clone()), Ln, 4e-6, f"{name} Lnoise{ci}")
                    out[f"{tag}_{name}_L{ci}"] = sub(L).numpy()
                    out[f"{tag}_{name}_Ln{ci}"] = sub(Ln).numpy()
            print(f"operator {name}@{dim}: ok")
    save_split(os.path.join(GOLD, "operators"), out)


# --------------------------------------------------------------------------------------------------
def sampler_fixtures():
    from functions.svd_ddnm import ddnm_diffusion, ddnm_plus_diffusion, get_schedule_jump
    for T, l, r in ((20, 1, 1), (100, 1, 1), (100, 3, 3), (100, 2, 2), (250, 1, 1), (10, 3, 2)):
        assert get_schedule_jump(T, l, r) == SCH.jump_schedule(T, l, r)
    cfg = U.SimpleUNetConfig.tiny()
    m = ref_model(cfg, 1234)
    sd = U.init_state_dict(cfg, 1234)
    betas = SCH.linear_betas()
    dim, B = cfg.resolution, 2
    out = {"betas": betas.numpy()}
    rng = torch.Generator().manual_seed(777)
    x_orig = torch.rand(B, 3, dim, dim, generator=rng) * 2 - 1
    x_T = torch.randn(B, 3, dim, dim, generator=rng)
    out["x_orig"], out["x_T"] = x_orig.numpy(), x_T.numpy()
    # same RNG protocol as operator_fixtures (x, v, e drawn first) so mask / perm equal the stored artefacts
    orng = torch.Generator().manual_seed(4321)
    torch.rand(B, 3, dim, dim, generator=orng), torch.randn(B, 3 * dim * dim, generator=orng), torch.randn(B, 3 * dim * dim, generator=orng)
    opsets = {n: (r_, o_) for n, r_, o_, _ in build_ops(dim, orng)}
    cases = [("sr4", 10, 1, 1, 0.0), ("sr4", 10, 3, 2, 0.0), ("sr4", 10, 1, 1, 0.1), ("color", 10, 1, 1, 0.0),
             ("inpaint", 10, 2, 2, 0.1), ("wh", 10, 1, 1, 0.0), ("deblur", 10, 1, 1, 0.1), ("bicubic", 10, 1, 1, 0.0)]
    for name, T, tl, tr, sy in cases:
        rop, oop = opsets[name]
        conf = ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=T, travel_length=tl, travel_repeat=tr))
        npairs = len(SCH.time_pairs(1000, T, tl, tr))
        nrng = torch.Generator().manual_seed(555)
        tape = [torch.randn(B, 3, dim, dim, generator=nrng) for _ in range(npairs)]
        y = rop.A(x_orig)
        if sy > 0:
            y = y + sy * torch.randn(y.shape, generator=nrng)
        with torch.no_grad(), cpu_shim(tape):
            if sy == 0.0:
                xs, x0s = ddnm_diffusion(x_T, m, betas, 0.85, rop, y, config=conf)
            else:
                xs, x0s = ddnm_plus_diffusion(x_T, m, betas, 0.85, rop, y, sy, config=conf)
        with torch.no_grad():
            ox, ox0 = S.ddnm_sample(x_T, lambda a, b: U.forward(sd, a, b, cfg), betas, 0.85, oop, y, tape,
                                    t_sampling=T, travel_length=tl, travel_repeat=tr, sigma_y=sy)
        d = close(ox, xs[0], 5e-4, f"sampler {name}")
        close(ox0, x0s[0], 5e-4, f"sampler {name} x0")
        key = f"{name}_T{T}_l{tl}_r{tr}_s{sy}"
        out[key + "_y"], out[key + "_x0"], out[key + "_x0pred"] = y.numpy(), xs[0].numpy(), x0s[0].numpy()
        print(f"sampler {key}: ok (oracle-ref {d:.2e}), npairs {npairs}")
    out["noise_seed"] = np.array([555])
    np.savez_compressed(os.path.join(GOLD, "sampler_tiny.npz"), **out)


# --------------------------------------------------------------------------------------------------
SIMPLIFIED_CASES = [("sr_averagepooling", 4, 0.1, 3, 1, 1), ("colorization", 1, 0.0, 3, 1, 1), ("inpainting", 1, 0.05, 3, 1, 1),
                    ("denoising", 1, 0.2, 3, 1, 1), ("mask_color_sr", 2, 0.05, 4, 2, 2)]   # deg, scale, sigma_y(arg), T, l, r
SIMPLIFIED_CASES_R2 = [("sr_averagepooling", 16, 0.2, 3, 1, 1)]   # evaluation.sh's 16x SR with noise; stored in simplified_r2.npz


def simplified_fixtures(cases=None, fname="simplified.npz", store_inputs=True):
    """Run the reference runner's own Diffusion.simplified_ddnm_plus (diffusion.py:211-415) on one synthetic image with the
    dataset / PNG writer stubbed out, capture the image it would save, and pin oracle.simplified to it."""
    import guided_diffusion.diffusion as D
    from oracle import simplified as SP
    cfg = U.SimpleUNetConfig.celeba_hq()
    m = ref_model(cfg, 1234)
    sd = U.init_state_dict(cfg, 1234)
    betas = SCH.linear_betas()
    g = torch.Generator().manual_seed(2024)
    x01 = torch.rand(1, 3, 256, 256, generator=g)                      # the "dataset image" in [0, 1]
    mask = torch.from_numpy(np.load(os.path.join(REF, "exp/inp_masks/mask.npy")))
    out = {"x01": x01.numpy(), "mask_bits": np.packbits(mask.numpy().astype(np.uint8).reshape(-1))} if store_inputs else {}
    cases = SIMPLIFIED_CASES if cases is None else cases
    cwd = os.getcwd()
    os.chdir(REF)                                                        # the runner loads exp/inp_masks/mask.npy relatively
    try:
        for deg, scale, sy, T, tl, tr in cases:
            npairs = len(SCH.time_pairs(1000, T, tl, tr))
            nrng = torch.Generator().manual_seed(556)
            tape = [torch.randn(1, 3, 256, 256, generator=nrng) for _ in range(npairs)]
            saved = {}
            fake = ns(args=ns(deg=deg, deg_scale=float(scale), sigma_y=sy, eta=0.85, subset_start=-1, subset_end=-1, seed=1234,
                              image_folder="/tmp/ddnm_golden_unused"),
                      config=ns(data=ns(num_workers=0, channels=3, image_size=256, uniform_dequantization=False,
                                        gaussian_dequantization=False, rescaled=True, logit_transform=False),
                                sampling=ns(batch_size=1), diffusion=ns(num_diffusion_timesteps=1000),
                                time_travel=ns(T_sampling=T, travel_length=tl, travel_repeat=tr)),
                      betas=betas, device=torch.device("cpu"))
            ds = torch.utils.data.TensorDataset(x01, torch.zeros(1, dtype=torch.long))
            orig = (D.get_dataset, D.tvu.save_image, D.os.makedirs)
            D.get_dataset = lambda a, c: (ds, ds)
            D.tvu.save_image = lambda t, path, **k: saved.__setitem__(os.path.basename(path), t.detach().clone())
            D.os.makedirs = lambda *a, **k: None
            try:
                torch.manual_seed(4242)                                  # x_T = first torch.randn after this seed (:310-316)
                with torch.no_grad(), cpu_shim(tape):
                    D.Diffusion.simplified_ddnm_plus(fake, m, None)
            finally:
                D.get_dataset, D.tvu.save_image, D.os.makedirs = orig
            ref_img = [v for k, v in saved.items() if k.endswith("_0.png")][-1].reshape(1, 3, 256, 256)
            # oracle
            torch.manual_seed(4242)
            x_T = torch.randn(1, 3, 256, 256)
            A, Ap = SP.degradation(deg, scale, mask.float(), 256)
            x_orig = 2 * x01 - 1.0
            y = A(x_orig)
            with torch.no_grad():
                ox, _ = SP.simplified_sample(x_T, lambda a, b: U.forward(sd, a, b, cfg), betas, 0.85, A, Ap, y, 2 * sy, tape,
                                             t_sampling=T, travel_length=tl, travel_repeat=tr)
            oimg = torch.clamp((ox + 1.0) / 2.0, 0.0, 1.0)
            d = close(oimg, ref_img, 2e-4, f"simplified {deg}")
            key = f"{deg}_s{scale}_sy{sy}_T{T}_l{tl}_r{tr}"
            out[key + "_img_s4"] = ref_img[:, :, ::4, ::4].contiguous().numpy()
            print(f"simplified {key}: ok (oracle-ref {d:.2e})")
    finally:
        os.chdir(cwd)
    np.savez_compressed(os.path.join(GOLD, fname), **out)


def runner_fixtures():
    """datasets/__init__.py data_transform / inverse_data_transform, tvu.save_image bytes (decoded back with PIL) and the PSNR
    line of diffusion.py:599-601, all executed from the reference / torchvision."""
    import io
    import torchvision.utils as tvu
    from PIL import Image
    from datasets import data_transform, inverse_data_transform
    from oracle import runner_io as RIO
    out = {}
    rng = torch.Generator().manual_seed(2718)
    X = torch.rand(2, 3, 16, 16, generator=rng)
    xm = torch.randn(2, 3, 16, 16, generator=rng) * 0.8          # "restored" images in model space, partly out of range
    out["X"], out["xm"] = X.numpy(), xm.numpy()
    cases = dict(rescaled=(True, False, False, False), logit=(False, True, False, False), deq=(True, False, True, True),
                 plain=(False, False, False, False))
    for name, (resc, logit, udq, gdq) in cases.items():
        cfg = ns(data=ns(rescaled=resc, logit_transform=logit, uniform_dequantization=udq, gaussian_dequantization=gdq))
        torch.manual_seed(99)
        un = torch.rand_like(X) if udq else None
        gn = torch.randn_like(X) if gdq else None
        torch.manual_seed(99)
        T = data_transform(cfg, X)
        close(RIO.data_transform(X, resc, logit, un, gn), T, 1e-6, f"data_transform {name}")
        out[f"{name}_T"] = T.numpy()
        if udq:
            out[f"{name}_un"], out[f"{name}_gn"] = un.numpy(), gn.numpy()
        inv = inverse_data_transform(cfg, xm)
        close(RIO.inverse_data_transform(xm, resc, logit), inv, 1e-6, f"inverse {name}")
        out[f"{name}_inv"] = inv.numpy()
        orig = inverse_data_transform(cfg, T)
        u8, ps = [], []
        for j in range(xm.shape[0]):
            buf = io.BytesIO()
            tvu.save_image(inv[j], buf, format="png")                      # diffusion.py:596-598
            buf.seek(0)
            img = np.array(Image.open(buf).convert("RGB"))
            assert np.array_equal(img, RIO.to_uint8_hwc(inv[j]).numpy()), "uint8 quantisation"
            u8.append(img)
            mse = torch.mean((inv[j] - orig[j]) ** 2)                      # :600
            psnr = 10 * torch.log10(1 / mse)                               # :601
            close(RIO.psnr(inv[j], orig[j]), psnr, 1e-6, "psnr")
            ps.append(float(psnr))
        out[f"{name}_u8"] = np.stack(u8)
        out[f"{name}_psnr"] = np.array(ps, dtype=np.float32)
    np.savez_compressed(os.path.join(GOLD, "runner_io.npz"), **out)
    print("runner I/O: ok")


def guided_fixtures():
    """Class-conditional denoiser (imagenet_256_cc.yml: class_cond, unet.py:478-479,651-653) and the classifier-guided branches of
    ddnm_diffusion / ddnm_plus_diffusion (svd_ddnm.py:48-52, 109-113) executed from the reference, with a toy differentiable
    classifier standing in for the ImageNet one (oracle/guidance.py)."""
    from functions.svd_ddnm import ddnm_diffusion, ddnm_plus_diffusion
    import functions.svd_ddnm as ref_mod
    from oracle.guidance import make_toy_cond_fn
    assert ref_mod.class_num == S.CLASS_NUM
    cfg = UO.OpenAIUNetConfig.tiny_class_cond()
    create_model_cfg = cfg
    import guided_diffusion.script_util as su
    assert su.NUM_CLASSES == cfg.num_classes
    m = ref_openai(create_model_cfg, 1234)
    rsd = m.state_dict()
    sd = UO.init_state_dict(cfg, 1234)
    assert set(sd) == set(rsd)
    for k in sd:
        if not torch.equal(sd[k], rsd[k]):
            assert rsd[k].abs().sum() == 0, f"{k}: differs from the reference but is not a zero-initialised tensor"
    m.load_state_dict(sd)
    out = {}
    g = torch.Generator().manual_seed(31)
    B, dim = 2, cfg.image_size
    x = torch.randn(B, 3, dim, dim, generator=g)
    t = torch.tensor([417.0, 3.0])
    labels = torch.tensor([951, 7])
    with torch.no_grad():
        r = m(x, t, labels)
        o = UO.forward(sd, x, t, cfg, y=labels)
    close(o, r, 0.0, "class-conditional unet")
    out["unet_x"], out["unet_t"], out["unet_labels"], out["unet_out"] = x.numpy(), t.numpy(), labels.numpy(), r.numpy()
    cond_fn = make_toy_cond_fn(dim, cfg.num_classes, scale=2.0)
    gcheck = cond_fn(x, t, labels)
    out["cond_grad"] = gcheck.numpy()
    betas = SCH.linear_betas()
    x_orig = torch.rand(B, 3, dim, dim, generator=g) * 2 - 1
    x_T = torch.randn(B, 3, dim, dim, generator=g)
    out["x_T"] = x_T.numpy()
    orng = torch.Generator().manual_seed(4321)
    torch.rand(B, 3, dim, dim, generator=orng), torch.randn(B, 3 * dim * dim, generator=orng), torch.randn(B, 3 * dim * dim, generator=orng)
    opsets = {n: (r_, o_) for n, r_, o_, _ in build_ops(dim, orng)}
    for name, T, sy in (("sr4", 6, 0.0), ("inpaint", 6, 0.1)):
        rop, oop = opsets[name]
        conf = ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=T, travel_length=1, travel_repeat=1))
        npairs = len(SCH.time_pairs(1000, T, 1, 1))
        nrng = torch.Generator().manual_seed(556)
        tape = [torch.randn(B, 3, dim, dim, generator=nrng) for _ in range(npairs)]
        y = rop.A(x_orig)
        if sy > 0:
            y = y + sy * torch.randn(y.shape, generator=nrng)
        with torch.no_grad(), cpu_shim(tape):
            if sy == 0.0:
                xs, x0s = ddnm_diffusion(x_T, m, betas, 0.85, rop, y, cls_fn=cond_fn, classes=torch.tensor([1, 2]), config=conf)
            else:
                xs, x0s = ddnm_plus_diffusion(x_T, m, betas, 0.85, rop, y, sy, cls_fn=cond_fn, classes=torch.tensor([1, 2]), config=conf)
        with torch.no_grad():
            ox, ox0 = S.ddnm_sample(x_T, lambda a, b, c: UO.forward(sd, a, b, cfg, y=c), betas, 0.85, oop, y, tape, t_sampling=T,
                                    travel_length=1, travel_repeat=1, sigma_y=sy, cls_fn=cond_fn)
        d = close(ox, xs[0], 5e-4, f"guided sampler {name}")
        close(ox0, x0s[0], 5e-4, f"guided sampler {name} x0")
        key = f"{name}_T{T}_s{sy}"
        out[key + "_y"], out[key + "_x0"], out[key + "_x0pred"] = y.numpy(), xs[0].numpy(), x0s[0].numpy()
        print(f"guided sampler {key}: ok (oracle-ref {d:.2e})")
    out["noise_seed"] = np.array([556])
    np.savez_compressed(os.path.join(GOLD, "guided_tiny.npz"), **out)


# --------------------------------------------------------------------------------------------------
from oracle.fullsize import FULLSIZE_CASES, fullsize_inputs, uni_kernel      # noqa: E402


def fullsize_ops(wh_perm=None):
    """Reference + oracle operators at 256x256 the way the runner builds them (diffusion.py:452-523)."""
    from functions import svd_operators as R
    ops = {}
    r = R.SuperResolution(3, 256, 4, "cpu")
    ops["sr4"] = (r, O.SuperResolution(3, 256, 4, r.U_small, r.singulars_small, r.V_small))
    r = R.Colorization(256, "cpu")
    ops["color"] = (r, O.Colorization(256, r.U_small, r.singulars_small, r.V_small))
    mask = np.load(os.path.join(REF, "exp/inp_masks/mask.npy"))
    r = _ref_inpainting(R, 3, 256, torch.from_numpy(mask).reshape(-1))
    ops["inpaint"] = (r, O.Inpainting(3, 256, mask))
    perm = torch.randperm(256 ** 2, generator=torch.Generator().manual_seed(4242)) if wh_perm is None else wh_perm
    r = R.WalshHadamardCS(3, 256, 4, perm, "cpu")
    ops["wh"] = (r, O.WalshHadamardCS(3, 256, 4, perm))
    for name, k in (("deblur", gauss_kernel()), ("deblur_uni", uni_kernel())):
        r = R.Deblurring(k, 3, 256, "cpu")
        ops[name] = (r, O.Deblurring(3, 256, r.U_small, r.V_small, r._singulars, r._singulars_orig, r._perm))
    return ops, mask, perm


def fullsize_fixtures():
    """BASELINE configs at their real size (256x256, the real celeba / imagenet networks with seeded random weights, the real
    exp/inp_masks/mask.npy) through the UNMODIFIED reference samplers, plus the deblur_uni operator (diffusion.py:500-503) that
    operators.npz lacks.  Stored: strided samples + sums of the reference results, the WH permutation, the mask bits and, for the
    two Deblurring operators, the LAPACK-dependent artefacts (U_small, V_small, singulars, perm) so that another machine's
    torch.svd cannot change the operator under test."""
    from functions.svd_ddnm import ddnm_diffusion, ddnm_plus_diffusion
    from functions import svd_operators as R
    out = {}
    ops, mask, perm = fullsize_ops()
    out["mask_bits"] = np.packbits(mask.astype(np.uint8).reshape(-1))
    out["wh_perm"] = perm.numpy().astype(np.int32)
    for name in ("deblur", "deblur_uni"):
        r = ops[name][0]
        for k, v in dict(U_small=r.U_small, V_small=r.V_small, singulars=r._singulars, singulars_orig=r._singulars_orig,
                         perm=r._perm).items():
            out[f"{name}_art_{k}"] = v.numpy() if k != "perm" else v.numpy().astype(np.int32)
    # ---- deblur_uni operator fixtures, dim 32 (full vectors + artefacts) and 256 (strided), as operator_fixtures does
    for dim, B in ((32, 2), (256, 1)):
        rng = torch.Generator().manual_seed(4321)
        x = torch.rand(B, 3, dim, dim, generator=rng) * 2 - 1
        v = torch.randn(B, 3 * dim * dim, generator=rng)
        e = torch.randn(B, 3 * dim * dim, generator=rng)
        tag = f"d{dim}_deblur_uni"
        if dim == 32:
            r = R.Deblurring(uni_kernel(), 3, dim, "cpu")
            o = O.Deblurring(3, dim, r.U_small, r.V_small, r._singulars, r._singulars_orig, r._perm)
            for k, a in dict(U_small=r.U_small, V_small=r.V_small, singulars=r._singulars, singulars_orig=r._singulars_orig,
                             perm=r._perm).items():
                out[f"{tag}_art_{k}"] = a.numpy()
        else:
            r, o = ops["deblur_uni"]
        sub = (lambda z: z) if dim == 32 else (lambda z: z.reshape(B, -1)[:, ::61].contiguous())
        y = r.A(x)
        close(o.A(x.reshape(B, -1)), y, 2e-6, "deblur_uni A")
        yq = y * 0.9 + 0.05
        pin = r.A_pinv(yq.clone())
        close(o.A_pinv(yq.clone()), pin, 2e-6, "deblur_uni A_pinv")
        proj = x - r.A_pinv(r.A(x.reshape(B, -1)) - yq.reshape(B, -1)).reshape(x.shape)
        close(o.project(x, yq), proj, 4e-6, "deblur_uni project")
        out[f"{tag}_A"], out[f"{tag}_Apinv"], out[f"{tag}_proj"] = sub(y).numpy(), sub(pin).numpy(), sub(proj).numpy()
        for ci, (a, sy, st) in enumerate(LAMBDA_CASES):
            at, stt = torch.tensor(a), torch.tensor(st)
            L = r.Lambda(v.clone(), at, sy, stt, 0.85)
            Ln = r.Lambda_noise(v.clone(), at, sy, stt, 0.85, e.clone())
            close(o.Lambda(v.clone(), at, sy, stt, 0.85), L, 4e-6, f"deblur_uni Lambda{ci}")
            close(o.Lambda_noise(v.clone(), at, sy, stt, 0.85, e.clone()), Ln, 4e-6, f"deblur_uni Lnoise{ci}")
            out[f"{tag}_L{ci}"], out[f"{tag}_Ln{ci}"] = sub(L).numpy(), sub(Ln).numpy()
        print(f"operator deblur_uni@{dim}: ok")
    # ---- real-size sampler runs through the reference
    betas = SCH.linear_betas()
    nets = {}

    def net(kind):
        if kind not in nets:
            if kind == "celeba":
                cfg = U.SimpleUNetConfig.celeba_hq()
                m, sd = ref_model(cfg, 1234), U.init_state_dict(cfg, 1234)
                fwd = lambda a, b: U.forward(sd, a, b, cfg)          # noqa: E731
            else:
                cfg = UO.OpenAIUNetConfig.imagenet_256()
                m, sd = ref_openai(cfg, 1234), UO.init_state_dict(cfg, 1234)
                m.load_state_dict(sd)
                fwd = lambda a, b: UO.forward(sd, a, b, cfg)         # noqa: E731
            nets[kind] = (m, fwd)
        return nets[kind]
    for key, kind, opname, T, tl, tr, sy in FULLSIZE_CASES:
        m, fwd = net(kind)
        rop, oop = ops[opname]
        conf = ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=T, travel_length=tl, travel_repeat=tr))
        npairs = len(SCH.time_pairs(1000, T, tl, tr))
        x_orig, x_T, tape, ynoise = fullsize_inputs(key, npairs)
        y = rop.A(x_orig)
        if sy > 0:
            y = y + sy * ynoise[:, : y.shape[1]]
        with torch.no_grad(), cpu_shim(tape):
            if sy == 0.0:
                xs, x0s = ddnm_diffusion(x_T, m, betas, 0.85, rop, y, config=conf)
            else:
                xs, x0s = ddnm_plus_diffusion(x_T, m, betas, 0.85, rop, y, sy, config=conf)
        with torch.no_grad():
            ox, ox0 = S.ddnm_sample(x_T, fwd, betas, 0.85, oop, y, tape, t_sampling=T, travel_length=tl, travel_repeat=tr, sigma_y=sy)
        d = close(ox, xs[0], 2e-3, f"fullsize {key}")
        close(ox0, x0s[0], 2e-3 * max(1.0, x0s[0].abs().max().item()), f"fullsize {key} x0")
        r0, r1 = xs[0], x0s[0]
        out[key + "_x0_s4"] = r0[:, :, ::4, ::4].contiguous().numpy()
        out[key + "_x0pred_s4"] = r1[:, :, ::4, ::4].contiguous().numpy()
        out[key + "_sums"] = np.array([r0.double().sum().item(), r0.double().abs().sum().item(), r1.double().sum().item(),
                                       r1.double().abs().sum().item()])
        out[key + "_resid"] = np.array([(rop.A(r0).reshape(1, -1) - y.reshape(1, -1)).abs().max().item()])
        print(f"fullsize {key}: ok (oracle-ref {d:.2e}), npairs {npairs}, |A x0 - y| {out[key + '_resid'][0]:.2e}")
    save_split(os.path.join(GOLD, "fullsize"), out)



def sr16_fixtures():
    """16x average-pooling super-resolution with measurement noise — evaluation.sh's `--deg sr_averagepooling --deg_scale 16
    --sigma_y 0.2 --add_noise` — through the reference: the SVD operator (K = 256 entries per patch, LAPACK-dependent 256 x 256
    basis stored), a DDNM+ sampling with the tiny network, and the runner's simplified loop on the celeba-size network."""
    from functions import svd_operators as R
    from functions.svd_ddnm import ddnm_plus_diffusion
    out = {}
    dim, B = 32, 2
    r = R.SuperResolution(3, dim, 16, "cpu")
    o = O.SuperResolution(3, dim, 16, r.U_small, r.singulars_small, r.V_small)
    out["art_U_small"], out["art_singulars_small"], out["art_V_small"] = r.U_small.numpy(), r.singulars_small.numpy(), r.V_small.numpy()
    rng = torch.Generator().manual_seed(4321)
    x = torch.rand(B, 3, dim, dim, generator=rng) * 2 - 1
    v = torch.randn(B, 3 * dim * dim, generator=rng)
    e = torch.randn(B, 3 * dim * dim, generator=rng)
    y = r.A(x)
    close(o.A(x.reshape(B, -1)), y, 2e-6, "sr16 A")
    yq = y * 0.9 + 0.05
    pin = r.A_pinv(yq.clone())
    close(o.A_pinv(yq.clone()), pin, 2e-6, "sr16 A_pinv")
    proj = x - r.A_pinv(r.A(x.reshape(B, -1)) - yq.reshape(B, -1)).reshape(x.shape)
    close(o.project(x, yq), proj, 4e-6, "sr16 project")
    out["op_A"], out["op_Apinv"], out["op_proj"] = y.numpy(), pin.numpy(), proj.numpy()
    for ci, (a, sy, st) in enumerate(LAMBDA_CASES):
        at, stt = torch.tensor(a), torch.tensor(st)
        L = r.Lambda(v.clone(), at, sy, stt, 0.85)
        Ln = r.Lambda_noise(v.clone(), at, sy, stt, 0.85, e.clone())
        close(o.Lambda(v.clone(), at, sy, stt, 0.85), L, 4e-6, f"sr16 Lambda{ci}")
        close(o.Lambda_noise(v.clone(), at, sy, stt, 0.85, e.clone()), Ln, 4e-6, f"sr16 Lnoise{ci}")
        out[f"op_L{ci}"], out[f"op_Ln{ci}"] = L.numpy(), Ln.numpy()
    print("operator sr16@32: ok")
    # DDNM+ sampling, tiny network, sigma_y = 0.2 (0.4 internal)
    cfg = U.SimpleUNetConfig.tiny()
    m, sd = ref_model(cfg, 1234), U.init_state_dict(cfg, 1234)
    betas = SCH.linear_betas()
    g = torch.Generator().manual_seed(1616)
    x_orig = torch.rand(B, 3, dim, dim, generator=g) * 2 - 1
    x_T = torch.randn(B, 3, dim, dim, generator=g)
    T, sy = 6, 0.4
    tape = [torch.randn(B, 3, dim, dim, generator=g) for _ in range(T)]
    yn = r.A(x_orig)
    yn = yn + sy * torch.randn(yn.shape, generator=g)
    conf = ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=T, travel_length=1, travel_repeat=1))
    with torch.no_grad(), cpu_shim(tape):
        xs, x0s = ddnm_plus_diffusion(x_T, m, betas, 0.85, r, yn, sy, config=conf)
    with torch.no_grad():
        ox, ox0 = S.ddnm_sample(x_T, lambda a, b: U.forward(sd, a, b, cfg), betas, 0.85, o, yn, tape, t_sampling=T, sigma_y=sy)
    d = close(ox, xs[0], 2e-3, "sr16 sampler")   # the K = 256 basis products re-associate; the random-init net amplifies it
    out["samp_x_orig"], out["samp_x_T"], out["samp_y"] = x_orig.numpy(), x_T.numpy(), yn.numpy()
    out["samp_x0"], out["samp_x0pred"], out["samp_seed"] = xs[0].numpy(), x0s[0].numpy(), np.array([1616])
    print(f"sampler sr16 DDNM+: ok (oracle-ref {d:.2e})")
    np.savez_compressed(os.path.join(GOLD, "sr16.npz"), **out)


def hq_fixtures():
    """hq_demo's arbitrary-size restoration (mask-shift trick) through ITS OWN code: create_model_and_diffusion + SpacedDiffusion.
    p_sample_loop (hq_demo/guided_diffusion/gaussian_diffusion.py:318-390, :578-750) on a 256 x 384 canvas (two windows, the second
    one irregular: W % 128 == 0 here so also a 320-wide case), a small class-conditional UNet (64 base channels, 256 x 256 input,
    learn_sigma), 4x average-pooling SR with and without measurement noise, a short jump schedule with time travel.  Must run in
    a process that has not imported the main reference's `guided_diffusion` package (same package name): `gen_golden hq` alone."""
    assert "guided_diffusion" not in sys.modules, "run `python -m oracle.gen_golden hq` on its own"
    HQ = os.path.join(REF, "hq_demo")
    sys.path.insert(0, HQ)
    import guided_diffusion.gaussian_diffusion as GD
    from guided_diffusion.script_util import create_model_and_diffusion, model_and_diffusion_defaults, select_args
    import conf_mgt
    from oracle import hq as HQO
    assert os.path.abspath(GD.__file__).startswith(HQ)
    # the loop writes progress PNGs under results/ (:49-52, :341-343) and hands its result to save_image(finalresult[0], .../final)
    # (:750-752); p_sample_loop's own return value is unusable (it iterates over the returned dict's keys), so capture that call
    saved = {}
    GD.save_image = lambda img, save_dir, idx: saved.__setitem__(os.path.basename(save_dir), img.detach().clone())
    GD.os.makedirs = lambda *a, **k: None
    out = {}
    jump = dict(t_T=6, n_sample=1, jump_length=2, jump_n_sample=2)
    conf = conf_mgt.conf_base.Default_Conf()
    conf.update(dict(attention_resolutions="32,16,8", class_cond=True, diffusion_steps=1000, learn_sigma=True, noise_schedule="linear",
                     num_channels=64, num_head_channels=64, num_heads=4, num_res_blocks=1, resblock_updown=True, use_fp16=False,
                     use_scale_shift_norm=True, timestep_respacing="6", use_kl=False, predict_xstart=False, rescale_timesteps=False,
                     rescale_learned_sigmas=False, num_heads_upsample=-1, channel_mult="", dropout=0.0, use_checkpoint=False,
                     use_new_attention_order=False, image_size=256, name="inet256", schedule_jump_params=jump))
    torch.manual_seed(1234)
    model, diffusion = create_model_and_diffusion(**select_args(conf, model_and_diffusion_defaults().keys()), conf=conf)
    model.eval()
    cfg = UO.OpenAIUNetConfig(image_size=256, model_channels=64, num_res_blocks=1, channel_mult=(1, 1, 2, 2, 4, 4),
                              attention_resolutions=(32, 16, 8), num_head_channels=64, out_channels=6, num_classes=1000)
    sd = UO.init_state_dict(cfg, 1234)
    rsd = model.state_dict()
    assert set(sd) == set(rsd), sorted(set(sd) ^ set(rsd))[:8]
    for k in sd:
        if not torch.equal(sd[k], rsd[k]):
            assert rsd[k].abs().sum() == 0, f"{k}: differs from the reference but is not a zero-initialised tensor"
    model.load_state_dict(sd)
    K = HQO.SpacedConstants(1000, 6)
    assert K.timestep_map == diffusion.timestep_map
    for name in ("betas", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_variance", "posterior_mean_coef1",
                 "posterior_mean_coef2"):
        assert np.array_equal(getattr(K, name), getattr(diffusion, name)), name
    from guided_diffusion.scheduler import get_schedule_jump as ref_jump
    for jp in (jump, dict(t_T=100, n_sample=1, jump_length=10, jump_n_sample=3), dict(t_T=20, n_sample=1, jump_length=5, jump_n_sample=2)):
        assert ref_jump(**jp) == HQO.get_schedule_jump(**jp)
    classes = torch.tensor([950])

    def model_fn(x, t, y=None, gt=None, **kwargs):            # main.py:84-86
        return model(x, t, y, gt=gt)
    for key, (h, w), sy in (("w384", (64, 96), 0.0), ("w320_noisy", (64, 80), 0.1), ("h320", (80, 64), 0.0)):
        g = torch.Generator().manual_seed(700 + w + h)
        y_img = torch.rand(1, 3, h, w, generator=g) * 2 - 1     # the low-resolution input image ("gt" in main.py:103-110)
        ndraw = HQO.count_draws(4 * h, 4 * w, jump)
        tape = [torch.randn(1, 3, 256, 256, generator=g) for _ in range(ndraw)]
        kw = dict(gt=y_img.clone(), scale=4, deg="sr_averagepooling", resize_y=True, sigma_y=sy, save_path="unused", y=classes)
        rt = list(tape[1:])
        saved.clear()
        with torch.no_grad(), cpu_shim(rt) as shim:
            diffusion.p_sample_loop(model_fn, (1, 3, 256, 256), noise=tape[0], clip_denoised=True, model_kwargs=kw, cond_fn=None,
                                    device="cpu", progress=False, return_all=True, conf=conf)
        assert len(shim.tape) == 0, f"reference consumed a different number of draws ({len(shim.tape)} left)"
        ref = saved["final"][None]
        with torch.no_grad():
            o = HQO.restore(lambda a, b, c: UO.forward(sd, a, b.float(), cfg, y=c), y_img, classes, tape, deg="sr_averagepooling",
                            scale=4, sigma_y=sy, resize_y=True, respacing=6, jump=jump)
        d = close(o, ref, 2e-3, f"hq {key}")
        out[key + "_y"], out[key + "_out_s2"] = y_img.numpy(), ref[:, :, ::2, ::2].contiguous().numpy()
        out[key + "_sums"] = np.array([ref.double().sum().item(), ref.double().abs().sum().item()])
        out[key + "_seed"] = np.array([700 + w + h])
        print(f"hq {key}: canvas {tuple(ref.shape)}, {ndraw} draws, ok (oracle-ref {d:.2e})")
    np.savez_compressed(os.path.join(GOLD, "hq.npz"), **out)


def general_fixtures():
    """GeneralA (svd_operators.py:173-208): a dense 48 x 192 degradation with two singular values pushed under the
    1e-3 threshold so the zeroing branch (:185) is exercised."""
    import contextlib
    import io
    from functions import svd_operators as R
    rng = torch.Generator().manual_seed(97)
    A = torch.randn(48, 192, generator=rng) / 192 ** 0.5
    U0, S0, V0 = torch.svd(A, some=True)
    S0[-2:] = torch.tensor([5e-4, 1e-5])
    A = (U0 * S0) @ V0.t()
    with contextlib.redirect_stdout(io.StringIO()):
        r = R.GeneralA(A)
    o = O.GeneralA(r._U, r._singulars, r._V)
    assert int((r._singulars == 0).sum()) == 2
    x = torch.rand(3, 192, generator=rng) * 2 - 1
    y = r.A(x)
    close(o.A(x), y, 2e-6, "general A")
    yq = y * 0.9 + 0.05
    pin = r.A_pinv(yq.clone())
    close(o.A_pinv(yq.clone()), pin, 2e-6, "general A_pinv")
    proj = x - r.A_pinv(r.A(x) - yq)
    close(o.project(x, yq), proj, 4e-6, "general project")
    np.savez_compressed(os.path.join(GOLD, "general_a.npz"), A=A.numpy(), U=r._U.numpy(), S=r._singulars.numpy(), V=r._V.numpy(),
                        x=x.numpy(), yq=yq.numpy(), y=y.numpy(), pinv=pin.numpy(), proj=proj.numpy())
    print("operator general: ok")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    which = sys.argv[1:] or ["unet", "openai", "ops", "sampler", "simplified", "general", "runner", "guided", "fullsize", "sr16"]
    if "hq" in which:
        hq_fixtures()
    if "general" in which:
        general_fixtures()
    if "guided" in which:
        guided_fixtures()
    if "runner" in which:
        runner_fixtures()
    if "unet" in which:
        unet_fixtures()
    if "openai" in which:
        openai_fixtures()
    if "ops" in which:
        operator_fixtures()
    if "sampler" in which:
        sampler_fixtures()
    if "simplified" in which:
        simplified_fixtures()
    if "fullsize" in which:
        fullsize_fixtures()
    if "sr16" in which:
        sr16_fixtures()
        simplified_fixtures(SIMPLIFIED_CASES_R2, "simplified_r2.npz", store_inputs=False)   # x01 / mask: same as simplified.npz
    print("golden fixtures written to", GOLD)
