"""Drop-in for ``functions/svd_ddnm.py``: ``ddnm_diffusion`` (:19-78) and ``ddnm_plus_diffusion`` (:80-164) with the
reference's signatures and return convention (``([x_0.cpu()], [x0_pred.cpu()])``).

The whole loop runs inside libddnm_b200.so on the current CUDA stream without host round trips.  The Gaussian draws
are taken from torch's generator in the reference's order (one ``randn_like`` per time pair, :65/:74), a bounded chunk of
pairs at a time on a side stream while the previous chunk is being denoised (``NOISE_CHUNK_BYTES``), so a run is
seed-for-seed comparable with the reference on the same device and its noise memory does not grow with the schedule.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .guidance import ClassifierCondFn
from .model import _EngineModel
from .operators import CS, Deblurring2D, GeneralA, SRConv, _Operator
from .schedule import alpha_bar_table, time_pairs

class_num = 951

# Upper bound for ONE of the two noise buffers of the chunked loop (the other is being refilled on a side stream): the reference
# draws one randn_like per pair and keeps none, so its noise memory is O(1); here it is 2 x NOISE_CHUNK_BYTES at most, whatever
# T_sampling / travel_repeat are.
NOISE_CHUNK_BYTES = 256 << 20


def _chunked(n_pairs, x, run_range, rows=None):
    """Drive ``run_range(k0, k1, noise_chunk)`` over the schedule with the Gaussian draws produced chunk by chunk on a side stream
    (double-buffered), in the reference's generator order: pair k gets the k-th ``randn_like(x)`` after the caller's last draw.
    ``rows`` > x.shape[0]: the chunk buffers carry that many rows (a batch padded to a larger engine); only the real rows are drawn,
    with exactly the generator consumption of ``randn_like(x)``, the padding rows stay zero."""
    n = x.shape[0]
    rows = n if rows is None else rows
    shape = (rows,) + tuple(x.shape[1:])
    per_pair = rows * x[0].numel() * 4
    K = max(1, min(n_pairs, NOISE_CHUNK_BYTES // per_pair))
    main = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    mk = torch.zeros if rows != n else torch.empty
    bufs = [mk((K,) + shape, device=x.device, dtype=torch.float32) for _ in range(2 if n_pairs > K else 1)]
    consumed = [None, None]
    side.wait_stream(main)                                  # the buffers' allocation / earlier use of their memory
    chunks = [(k0, min(n_pairs, k0 + K)) for k0 in range(0, n_pairs, K)]

    def fill(c):
        k0, k1 = chunks[c]
        b = bufs[c % len(bufs)]
        with torch.cuda.stream(side):
            if consumed[c % 2] is not None:
                side.wait_event(consumed[c % 2])
            for k in range(k1 - k0):
                if rows == n:
                    b[k].normal_()                          # == torch.randn_like(x): same generator consumption, no extra copy
                else:
                    b[k, :n] = torch.randn_like(x)
            ev = torch.cuda.Event()
            ev.record(side)
        return ev
    ready = fill(0)
    for c, (k0, k1) in enumerate(chunks):
        nxt = fill(c + 1) if c + 1 < len(chunks) else None  # next chunk's draws overlap this chunk's denoising steps
        main.wait_event(ready)
        run_range(k0, k1, bufs[c % len(bufs)])
        ev = torch.cuda.Event()
        ev.record(main)
        consumed[c % 2] = ev
        ready = nxt
    for b in bufs:
        b.record_stream(side)                               # allocated on the caller's stream, written on the side stream


def sample_device(x, model, b, eta, A_funcs, y, sigma_y, plus, config, noise=None, cls_fn=None):
    """The loop with device-resident inputs and outputs (no host copies): returns (x_0, x0_pred) CUDA tensors."""
    return _run(x, model, b, eta, A_funcs, y, sigma_y, plus, cls_fn, None, config, noise, to_host=False)


def _run(x, model, b, eta, A_funcs, y, sigma_y, plus, cls_fn, classes, config, noise=None, to_host=True):
    if not isinstance(model, _EngineModel):
        model = getattr(model, "module", model)          # tolerate nn.DataParallel-style wrappers
    if not isinstance(model, _EngineModel) or not isinstance(A_funcs, _Operator):
        raise TypeError("ddnm_b200.sampler needs a ddnm_b200.model denoiser and a ddnm_b200.operators operator")
    if plus and isinstance(A_funcs, (SRConv, Deblurring2D, CS, GeneralA)):
        # these operators define no Lambda / Lambda_noise: the reference fails at its first step with the base class's
        # NotImplementedError (svd_operators.py:93-97)
        raise NotImplementedError()
    with torch.no_grad():
        if not x.is_cuda:
            x = x.to("cuda", non_blocking=True)            # the reference moves xs[-1] to 'cuda' itself (svd_ddnm.py:45)
        n = x.size(0)
        pairs = time_pairs(config.diffusion.num_diffusion_timesteps, config.time_travel.T_sampling,
                           config.time_travel.travel_length, config.time_travel.travel_repeat)
        abar = np.ascontiguousarray(alpha_bar_table(b).numpy())
        ti = np.ascontiguousarray(np.array([p[0] for p in pairs], dtype=np.int32))
        tj = np.ascontiguousarray(np.array([p[1] for p in pairs], dtype=np.int32))
        x = x.float().contiguous()
        if noise is not None:                               # a caller-supplied tape (tests, seed-for-seed comparisons)
            assert noise.shape == (len(pairs),) + tuple(x.shape)
            noise = noise.to(x.device).float().contiguous()
        yv = y.reshape(n, -1).to(x.device, non_blocking=True).float().contiguous()
        assert yv.shape[1] == A_funcs.y_dim, f"y has {yv.shape[1]} entries per image, operator expects {A_funcs.y_dim}"
        s = _lib.Schedule()
        s.n_pairs, s.t_i, s.t_j, s.abar = len(pairs), ti.ctypes.data, tj.ctypes.data, abar.ctypes.data
        s.num_timesteps, s.eta, s.sigma_y = int(config.diffusion.num_diffusion_timesteps), float(eta), float(sigma_y)
        s.plus = 1 if plus else 0
        # a ragged last batch rides on an existing bigger engine, padded (classifier guidance keeps the exact size: cls_fn sees n rows)
        eng, eb = (model.engine(n), n) if cls_fn is not None else model.engine_for(n)
        out = model.pad_rows(x, eb).clone()                 # the iterate, updated in place range by range
        x0p = torch.empty_like(out)
        yv = model.pad_rows(yv, eb)
        if noise is not None and eb != n:
            noise = torch.cat([noise, noise[:, -1:].expand(noise.shape[0], eb - n, *noise.shape[2:])], dim=1).contiguous()
        have_x0 = C.c_int(0)
        user = None
        if cls_fn is None:
            labels = grad = fn = None
            failure = []
        elif isinstance(cls_fn, ClassifierCondFn):
            labels, grad, fn, user = _native_guidance(x, model, n, cls_fn)
            failure = []
        else:
            labels, grad, fn, failure = _guidance(x, model, n, cls_fn)

        def run_range(k0, k1, chunk):
            rc = _lib.lib().ddnm_sample_range(eng, A_funcs._h, C.byref(s), k0, k1, _lib.ptr(out), _lib.ptr(x0p), C.byref(have_x0),
                                             _lib.ptr(yv), _lib.ptr(chunk), eb, _lib.ptr(labels), _lib.ptr(grad),
                                             None if fn is None else C.cast(fn, C.c_void_p), user, _lib.cur_stream())
            if failure:
                raise failure[0]
            _lib.check(rc)
        if noise is not None:
            run_range(0, len(pairs), noise)
        else:
            _chunked(len(pairs), x, run_range, rows=eb)
        if eb != n:
            out, x0p = out[:n], x0p[:n]
        if not to_host:
            return out, x0p
        return [out.to("cpu")], [x0p.to("cpu")]


CLASS_NUM = 951   # functions/svd_ddnm.py:7


def _guidance(x, model, n, cls_fn):
    """Classifier guidance (svd_ddnm.py:48-52, :109-113).  As in the reference, the caller's ``classes`` are replaced by
    ``class_num`` for every row, the denoiser is called as ``model(xt, t, classes)``, only channels 0..2 of its output are
    kept, and ``cls_fn`` is evaluated at ``x`` — the function's INPUT, not the current iterate.  ``cls_fn`` (the classifier's
    autograd gradient, diffusion.py:181-189) is the caller's PyTorch callable; everything else runs in libddnm_b200.so.
    Returns (labels, grad buffer, C callback, list that collects an exception raised inside the callback)."""
    assert model.num_classes is not None, "must specify y if and only if the model is class-conditional"   # unet.py:644-646
    classes = torch.ones(n, dtype=torch.long, device=x.device) * CLASS_NUM
    labels = classes.to(torch.int32)
    grad = torch.empty_like(x)
    failure = []

    def cb(_user, _k, t, _stream):
        try:
            tt = torch.ones(n, device=x.device) * t
            with torch.enable_grad():
                g = cls_fn(x, tt, classes)
            grad.copy_(g.reshape(grad.shape))
            return 0
        except BaseException as e:   # noqa: BLE001 — re-raised after the C call returns
            failure.append(e)
            return 1
    return labels, grad, _lib.GuidanceFn(cb), failure


def _native_guidance(x, model, n, cond):
    """As _guidance, with the gradient computed by the library's classifier (ddnm_classifier_guidance_fn) inside the loop: no
    host callback.  Returns (labels, grad buffer, C function, guidance context)."""
    assert model.num_classes is not None, "must specify y if and only if the model is class-conditional"   # unet.py:644-646
    labels = torch.full((n,), CLASS_NUM, dtype=torch.int32, device=x.device)
    grad = torch.empty_like(x)
    ctx = _lib.ClassifierGuidance()
    ctx.classifier = cond.classifier.engine(n)
    ctx.x, ctx.labels, ctx.scale, ctx.grad_buf = x.data_ptr(), labels.data_ptr(), cond.scale, grad.data_ptr()
    ctx.batch, ctx.labels_checked = n, 0
    # x, labels and grad stay referenced by _run's frame for the whole loop, ctx by the returned pointer
    return labels, grad, _lib.lib().ddnm_classifier_guidance_fn, C.cast(C.pointer(ctx), C.c_void_p)


def ddnm_diffusion(x, model, b, eta, A_funcs, y, cls_fn=None, classes=None, config=None, noise=None):
    return _run(x, model, b, eta, A_funcs, y, 0.0, False, cls_fn, classes, config, noise)


def ddnm_plus_diffusion(x, model, b, eta, A_funcs, y, sigma_y, cls_fn=None, classes=None, config=None, noise=None):
    return _run(x, model, b, eta, A_funcs, y, sigma_y, True, cls_fn, classes, config, noise)


# ------------------------------------------------------------------------------------------------------------------
# The runner's "simplified" DDNM+ (guided_diffusion/diffusion.py:211-415): the reference inlines this loop in
# Diffusion.simplified_ddnm_plus; here it is a function with the same ingredients.
# ------------------------------------------------------------------------------------------------------------------
class SimplifiedDegradation:
    """A / Ap of diffusion.py:244-290 for ``args.deg`` in {colorization, denoising, sr_averagepooling, inpainting,
    mask_color_sr, diy}; ``mask`` is the (H, W) 0/1 array of exp/inp_masks/mask.npy."""

    def __init__(self, deg, deg_scale=1, mask=None, image_size=256, device="cuda"):
        table = {"colorization": (0, 1, 1), "denoising": (0, 0, 1), "sr_averagepooling": (0, 0, None), "inpainting": (1, 0, 1),
                 "mask_color_sr": (1, 1, None), "diy": (1, 1, None)}
        if deg not in table:
            raise NotImplementedError("degradation type not supported")
        use_mask, use_gray, sc = table[deg]
        self.scale = int(round(deg_scale)) if sc is None else sc
        self.image_size = image_size
        self._mask = None
        if use_mask:
            assert mask is not None, "this degradation needs the inpainting mask"
            self._mask = torch.as_tensor(mask).to(device=device, dtype=torch.float32).reshape(image_size, image_size).contiguous()
        d = _lib.SimpleDeg()
        d.use_mask, d.use_gray, d.scale, d.img_dim, d.channels = use_mask, use_gray, self.scale, image_size, 3
        d.mask = None if self._mask is None else self._mask.data_ptr()
        self._d = d

    def A(self, z):
        z = z.float().contiguous()
        s = self.image_size // self.scale
        y = torch.empty(z.shape[0], 3, s, s, device=z.device, dtype=torch.float32)
        _lib.check(_lib.lib().ddnm_simplified_A(C.byref(self._d), _lib.ptr(z), z.shape[0], _lib.ptr(y), _lib.cur_stream()))
        return y

    def Ap(self, y):
        y = y.float().contiguous()
        x = torch.empty(y.shape[0], 3, self.image_size, self.image_size, device=y.device, dtype=torch.float32)
        _lib.check(_lib.lib().ddnm_simplified_Ap(C.byref(self._d), _lib.ptr(y), y.shape[0], _lib.ptr(x), _lib.cur_stream()))
        return x


def simplified_ddnm_plus(x, model, b, eta, degradation, y, sigma_y, config=None, noise=None):
    """x: x_T (B,3,H,W); y = degradation.A(x_orig); sigma_y already doubled (diffusion.py:292).  Returns
    ``([x_0.cpu()], [x0_pred.cpu()])`` like the SVD samplers."""
    if not isinstance(model, _EngineModel):
        model = getattr(model, "module", model)
    if not isinstance(model, _EngineModel) or not isinstance(degradation, SimplifiedDegradation):
        raise TypeError("simplified_ddnm_plus needs a ddnm_b200.model denoiser and a SimplifiedDegradation")
    with torch.no_grad():
        if not x.is_cuda:
            x = x.to("cuda", non_blocking=True)
        n = x.size(0)
        pairs = time_pairs(config.diffusion.num_diffusion_timesteps, config.time_travel.T_sampling,
                           config.time_travel.travel_length, config.time_travel.travel_repeat)
        abar = np.ascontiguousarray(alpha_bar_table(b).numpy())
        ti = np.ascontiguousarray(np.array([p[0] for p in pairs], dtype=np.int32))
        tj = np.ascontiguousarray(np.array([p[1] for p in pairs], dtype=np.int32))
        x = x.float().contiguous()
        if noise is not None:
            noise = noise.to(x.device).float().contiguous()
        yv = y.to(x.device, non_blocking=True).float().contiguous()
        s = _lib.Schedule()
        s.n_pairs, s.t_i, s.t_j, s.abar = len(pairs), ti.ctypes.data, tj.ctypes.data, abar.ctypes.data
        s.num_timesteps, s.eta, s.sigma_y, s.plus = int(config.diffusion.num_diffusion_timesteps), float(eta), float(sigma_y), 1
        out, x0p = x.clone(), torch.empty_like(x)
        eng = model.engine(n)
        have_x0 = C.c_int(0)

        def run_range(k0, k1, chunk):
            _lib.check(_lib.lib().ddnm_sample_simplified_range(eng, C.byref(degradation._d), C.byref(s), k0, k1, _lib.ptr(out),
                                                              _lib.ptr(x0p), C.byref(have_x0), _lib.ptr(yv), _lib.ptr(chunk), n,
                                                              _lib.cur_stream()))
        if noise is not None:
            run_range(0, len(pairs), noise)
        else:
            _chunked(len(pairs), x, run_range)
        return [out.to("cpu")], [x0p.to("cpu")]
