"""Drop-ins for the reference denoisers: ``guided_diffusion.models.Model`` (models.py:192-341, celeba_hq.yml) and
``guided_diffusion.unet.UNetModel`` via ``create_model`` (unet.py:396-664, script_util.py:130-185, imagenet_256.yml).

    model = Model(config)  |  model = create_model(**vars(config.model))      # the reference's own constructors
    model.load_state_dict(state_dict)     # same keys/layout as the reference checkpoint
    et = model(xt, t)                     # same call as functions/svd_ddnm.py:47

The forward pass runs entirely inside libddnm_b200.so (CUDA graph of hand-written sm_90a kernels); torch is
only used for tensor storage and the current stream.  Inference only (the reference samples under no_grad).
"""
import ctypes as C
import math

import torch

from . import _lib


class _EngineModel:
    """torch.nn.Module-like surface the reference runner uses (diffusion.py:117-164) over a libddnm_b200 handle."""
    out_ch = 3
    resolution = 256

    def _init_common(self):
        self._sd = None
        self._engines = {}      # batch -> handle
        self.use_cuda_graph = True
        # "fp32": fp32-grade tensor-core products (3 fp16 MMAs per MAC) — the parity mode and the default.
        # "fp16": one fp16 product per MAC, fp32 accumulation — fast mode, NOT within the fp32 parity tolerance.
        self.precision = "fp32"
        _lib.lib()              # fail early if the CUDA library is absent

    def load_state_dict(self, sd, strict=True):
        self._sd = {k.replace("module.", "", 1) if k.startswith("module.") else k: v.detach().float().contiguous()
                    for k, v in sd.items()}
        self._destroy()
        return self

    def to(self, *a, **k):
        return self

    def eval(self):
        return self

    def cuda(self):
        return self

    def parameters(self):
        return iter(self._sd.values()) if self._sd else iter(())

    def _create(self, batch):
        raise NotImplementedError

    def _freq(self):
        raise NotImplementedError

    def engine(self, batch):
        if batch in self._engines:
            return self._engines[batch]
        if self._sd is None:
            raise _lib.DDNMError("model has no weights: call load_state_dict first")
        L = _lib.lib()
        h = self._create(batch)
        params = dict(self._sd)
        params["__freq"] = self._freq()
        for name, t in params.items():
            t = t.contiguous()
            _lib.check(L.ddnm_unet_set_param(h, name.encode(), _lib.ptr(t), t.numel()))
        if self.precision not in ("fp32", "fp16"):
            raise ValueError("precision must be 'fp32' (parity) or 'fp16' (fast)")
        _lib.check(L.ddnm_unet_set_precision(h, 3 if self.precision == "fp32" else 1))
        _lib.check(L.ddnm_unet_finalize(h))
        _lib.check(L.ddnm_unet_set_graph(h, 1 if self.use_cuda_graph else 0))
        self._engines[batch] = h
        return h

    def engine_for(self, batch):
        """(handle, engine batch) able to run `batch` rows: the engine built for exactly that batch if it exists, else the smallest
        existing engine with a LARGER batch (a dataset's ragged last batch is padded to it instead of building a second engine with
        its own copy of every weight and its own multi-GiB workspace), else a new engine of that size."""
        if batch in self._engines:
            return self._engines[batch], batch
        bigger = sorted(b for b in self._engines if b > batch)
        if bigger:
            return self._engines[bigger[0]], bigger[0]
        return self.engine(batch), batch

    @staticmethod
    def pad_rows(t, rows):
        """t with its leading dimension padded to `rows` by repeating the last row (rows of a batch are independent trajectories)."""
        if t is None or t.shape[0] == rows:
            return t
        return torch.cat([t, t[-1:].expand(rows - t.shape[0], *t.shape[1:])], dim=0).contiguous()

    def __call__(self, x, t, y=None):
        return self.forward(x, t, y)

    num_classes = None       # class-conditional UNetModel only (unet.py:464)

    def forward(self, x, t, y=None):
        # unet.py:644-646
        assert (y is not None) == (self.num_classes is not None), "must specify y if and only if the model is class-conditional"
        assert x.is_cuda and x.dtype == torch.float32, "ddnm_b200 denoisers run on CUDA fp32 tensors"
        assert x.shape[2] == x.shape[3] == self.resolution     # models.py:302
        n = x.shape[0]
        t = t.to(device=x.device, dtype=torch.float32)
        if y is not None:
            assert y.shape == (n,)                              # unet.py:652
        h, eb = self.engine_for(n)
        x, t = self.pad_rows(x.contiguous(), eb), self.pad_rows(t.contiguous(), eb)
        out = torch.empty(eb, self.out_ch, self.resolution, self.resolution, device=x.device, dtype=torch.float32)
        if y is None:
            _lib.check(_lib.lib().ddnm_unet_forward(h, _lib.ptr(x), _lib.ptr(t), _lib.ptr(out), _lib.cur_stream()))
        else:
            labels = self.pad_rows(y.to(device=x.device, dtype=torch.int32).contiguous(), eb)
            _lib.check(_lib.lib().ddnm_unet_forward_cond(h, _lib.ptr(x), _lib.ptr(t), _lib.ptr(labels), _lib.ptr(out), _lib.cur_stream()))
        return out[:n] if eb != n else out

    # --- extras ---
    def read_tap(self, batch, name, shape):
        out = torch.empty(shape, device="cuda", dtype=torch.float32)
        _lib.check(_lib.lib().ddnm_unet_read_tap(self.engine(batch), name.encode(), _lib.ptr(out), out.numel(), _lib.cur_stream()))
        return out

    def info(self, batch):
        ws, nl, fl = C.c_longlong(), C.c_int(), C.c_double()
        _lib.check(_lib.lib().ddnm_unet_info(self.engine(batch), C.byref(ws), C.byref(nl), C.byref(fl)))
        return dict(workspace_bytes=ws.value, launches=nl.value, flops_per_forward=fl.value)

    def profile(self, x, t):
        import json
        out = torch.empty(x.shape[0], self.out_ch, self.resolution, self.resolution, device=x.device, dtype=torch.float32)
        buf = C.create_string_buffer(1 << 21)
        _lib.check(_lib.lib().ddnm_unet_profile(self.engine(x.shape[0]), _lib.ptr(x.contiguous()),
                                               _lib.ptr(t.float().contiguous()), _lib.ptr(out), _lib.cur_stream(), buf, len(buf)))
        return json.loads(buf.value.decode())

    def _destroy(self):
        if self._engines:
            L = _lib.lib()
            for h in self._engines.values():
                L.ddnm_unet_destroy(h)
        self._engines = {}

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass


class Model(_EngineModel):
    """guided_diffusion.models.Model (models.py:192-341): ``Model(config)``."""

    def __init__(self, config):
        m = config.model
        self.ch, self.out_ch = int(m.ch), int(m.out_ch)
        self.ch_mult = tuple(int(v) for v in m.ch_mult)
        self.num_res_blocks = int(m.num_res_blocks)
        self.attn_resolutions = tuple(int(v) for v in m.attn_resolutions)
        self.in_channels = int(m.in_channels)
        self.resolution = int(config.data.image_size)
        assert getattr(m, "resamp_with_conv", True), "only resamp_with_conv=True (the shipped configs) is built"
        self.config = config
        self._init_common()

    def _create(self, batch):
        c = _lib.SimpleCfg()
        c.ch, c.out_ch, c.n_levels = self.ch, self.out_ch, len(self.ch_mult)
        for i, v in enumerate(self.ch_mult):
            c.ch_mult[i] = v
        c.num_res_blocks = self.num_res_blocks
        c.n_attn_res = len(self.attn_resolutions)
        for i, v in enumerate(self.attn_resolutions):
            c.attn_res[i] = v
        c.in_channels, c.resolution, c.groups, c.eps = self.in_channels, self.resolution, 32, 1e-6
        h = C.c_void_p()
        _lib.check(_lib.lib().ddnm_unet_simple_create(C.byref(c), batch, C.byref(h)))
        return h

    def _freq(self):
        # frequency table with the reference's own arithmetic (models.py:15-18)
        half = self.ch // 2
        return torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))


class UNetModel(_EngineModel):
    """guided_diffusion.unet.UNetModel (unet.py:396-664) for the variant the shipped configs build
    (use_scale_shift_norm, resblock_updown, legacy attention order; optional class conditioning: ``model(x, t, y)``)."""

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None, use_checkpoint=False,
                 use_fp16=False, num_heads=1, num_head_channels=-1, num_heads_upsample=-1, use_scale_shift_norm=False,
                 resblock_updown=False, use_new_attention_order=False):
        self.num_classes = None if num_classes is None else int(num_classes)   # label_emb (unet.py:478-479), imagenet_256_cc.yml
        if not (use_scale_shift_norm and resblock_updown) or use_new_attention_order or num_head_channels <= 0 or dims != 2:
            raise NotImplementedError("ddnm_b200 builds the imagenet_256.yml UNetModel variant: use_scale_shift_norm, "
                                      "resblock_updown, legacy attention order, num_head_channels > 0")
        self.image_size = self.resolution = int(image_size)
        self.in_channels, self.model_channels, self.out_ch = int(in_channels), int(model_channels), int(out_channels)
        self.out_channels = self.out_ch
        self.num_res_blocks = int(num_res_blocks)
        self.attention_resolutions = tuple(int(v) for v in attention_resolutions)   # downsample rates, as in the reference
        # the reference computes int(mult * model_channels) (unet.py:484); the engine's config carries integer multipliers, so a
        # fractional one (create_model's image_size=512 default starts with 0.5) is refused instead of being truncated to 0
        if any(float(v) != int(v) for v in channel_mult):
            raise NotImplementedError(f"ddnm_b200 UNetModel: non-integer channel multipliers {tuple(channel_mult)} are not built")
        self.channel_mult = tuple(int(v) for v in channel_mult)
        self.num_head_channels = int(num_head_channels)
        self.use_fp16 = bool(use_fp16)
        self.dtype = torch.float32       # the engine always computes with fp32-grade arithmetic
        self._init_common()

    def convert_to_fp16(self):
        """No-op: the reference casts its torso to fp16 here (unet.py:619-625); this engine keeps fp32-grade products
        on the tensor cores (3x fp16 split), which is at least as accurate as the reference's fp32 mode."""
        return None

    def convert_to_fp32(self):
        return None

    def _create(self, batch):
        c = _lib.OpenAICfg()
        c.image_size, c.model_channels, c.num_res_blocks = self.image_size, self.model_channels, self.num_res_blocks
        c.n_levels = len(self.channel_mult)
        for i, v in enumerate(self.channel_mult):
            c.channel_mult[i] = v
        c.n_attn_ds = len(self.attention_resolutions)
        for i, v in enumerate(self.attention_resolutions):
            c.attn_ds[i] = v
        c.num_head_channels, c.out_channels, c.in_channels, c.groups, c.eps = self.num_head_channels, self.out_ch, self.in_channels, 32, 1e-5
        c.num_classes = self.num_classes or 0
        h = C.c_void_p()
        _lib.check(_lib.lib().ddnm_unet_openai_create(C.byref(c), batch, C.byref(h)))
        return h

    def _freq(self):
        # nn.py:113-115
        half = self.model_channels // 2
        return torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)


def create_model(image_size, num_channels, num_res_blocks, channel_mult="", learn_sigma=False, class_cond=False,
                 use_checkpoint=False, attention_resolutions="16", num_heads=1, num_head_channels=-1, num_heads_upsample=-1,
                 use_scale_shift_norm=False, dropout=0, resblock_updown=False, use_fp16=False, use_new_attention_order=False,
                 **kwargs):
    """guided_diffusion.script_util.create_model (:130-185), same keyword interface (``create_model(**vars(config.model))``)."""
    if channel_mult == "":
        if image_size == 512:
            channel_mult = (0.5, 1, 1, 2, 2, 4, 4)
        elif image_size == 256:
            channel_mult = (1, 1, 2, 2, 4, 4)
        elif image_size == 128:
            channel_mult = (1, 1, 2, 3, 4)
        elif image_size == 64:
            channel_mult = (1, 2, 3, 4)
        else:
            raise ValueError(f"unsupported image size: {image_size}")
    else:
        channel_mult = tuple(int(ch_mult) for ch_mult in channel_mult.split(","))
    attention_ds = [image_size // int(res) for res in attention_resolutions.split(",")]
    return UNetModel(image_size=image_size, in_channels=3, model_channels=num_channels,
                     out_channels=(3 if not learn_sigma else 6), num_res_blocks=num_res_blocks,
                     attention_resolutions=tuple(attention_ds), dropout=dropout, channel_mult=channel_mult,
                     num_classes=(1000 if class_cond else None), use_checkpoint=use_checkpoint, use_fp16=use_fp16,
                     num_heads=num_heads, num_head_channels=num_head_channels, num_heads_upsample=num_heads_upsample,
                     use_scale_shift_norm=use_scale_shift_norm, resblock_updown=resblock_updown,
                     use_new_attention_order=use_new_attention_order)


class EncoderUNetModel(_EngineModel):
    """guided_diffusion.unet.EncoderUNetModel (unet.py:684-895), the classifier of imagenet_256_cc.yml, for the variant
    create_classifier builds there (use_scale_shift_norm, resblock_updown, legacy attention order in the blocks, num_head_channels > 0,
    integer channel multipliers) with pool "attention" or "adaptive".  ``classifier(x, t)`` returns the logits; ``grad(x, t, y, scale)``
    is the classifier-guidance gradient of diffusion.py:183-189 computed by the library's own backward pass."""

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions, dropout=0,
                 channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, use_checkpoint=False, use_fp16=False, num_heads=1,
                 num_head_channels=-1, num_heads_upsample=-1, use_scale_shift_norm=False, resblock_updown=False,
                 use_new_attention_order=False, pool="adaptive"):
        if pool not in ("adaptive", "attention"):
            raise NotImplementedError(f"ddnm_b200 EncoderUNetModel: pool {pool!r} is not built (only 'attention' and 'adaptive')")
        if not (use_scale_shift_norm and resblock_updown) or use_new_attention_order or num_head_channels <= 0 or dims != 2:
            raise NotImplementedError("ddnm_b200 builds the imagenet_256_cc.yml EncoderUNetModel variant: use_scale_shift_norm, "
                                      "resblock_updown, legacy attention order, num_head_channels > 0")
        if any(float(v) != int(v) for v in channel_mult):
            raise NotImplementedError(f"ddnm_b200 EncoderUNetModel: non-integer channel multipliers {tuple(channel_mult)} are not built")
        self.image_size = self.resolution = int(image_size)
        self.in_channels, self.model_channels, self.out_channels = int(in_channels), int(model_channels), int(out_channels)
        self.out_ch = self.out_channels
        self.num_res_blocks = int(num_res_blocks)
        self.attention_resolutions = tuple(int(v) for v in attention_resolutions)
        self.channel_mult = tuple(int(v) for v in channel_mult)
        self.num_head_channels = int(num_head_channels)
        self.pool = pool
        self.use_fp16 = bool(use_fp16)
        self.dtype = torch.float32
        self._init_common()

    def convert_to_fp16(self):
        """No-op: the reference casts its torso to fp16 here (unet.py:859-864); this engine keeps fp32-grade products
        on the tensor cores (3x fp16 split), which is at least as accurate as the reference's fp32 mode."""
        return None

    def convert_to_fp32(self):
        return None

    def _create(self, batch):
        c = _lib.ClassifierCfg()
        c.image_size, c.model_channels, c.num_res_blocks = self.image_size, self.model_channels, self.num_res_blocks
        c.n_levels = len(self.channel_mult)
        if not 1 <= c.n_levels <= 8 or len(self.attention_resolutions) > 4:
            raise NotImplementedError("ddnm_b200 EncoderUNetModel: at most 8 levels and 4 attention resolutions")
        for i, v in enumerate(self.channel_mult):
            c.channel_mult[i] = v
        c.n_attn_ds = len(self.attention_resolutions)
        for i, v in enumerate(self.attention_resolutions):
            c.attn_ds[i] = v
        c.num_head_channels, c.out_channels, c.in_channels, c.groups, c.eps = (self.num_head_channels, self.out_channels,
                                                                               self.in_channels, 32, 1e-5)
        c.pool = 1 if self.pool == "attention" else 0
        h = C.c_void_p()
        _lib.check(_lib.lib().ddnm_classifier_create(C.byref(c), batch, C.byref(h)))
        return h

    def _freq(self):
        half = self.model_channels // 2   # nn.py:113-115
        return torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)

    def _inputs(self, x, t):
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32):
            raise _lib.DDNMError("ddnm_b200 classifier runs on CUDA fp32 tensors")
        if x.dim() != 4 or x.shape[1] != self.in_channels or x.shape[2] != self.image_size or x.shape[3] != self.image_size:
            raise _lib.DDNMError(f"classifier input must be [B, {self.in_channels}, {self.image_size}, {self.image_size}], got {tuple(x.shape)}")
        n = x.shape[0]
        t = torch.as_tensor(t, device=x.device).to(torch.float32).reshape(-1).expand(n).contiguous()
        return x.contiguous(), t, n

    def forward(self, x, timesteps):
        x, t, n = self._inputs(x, timesteps)
        logits = torch.empty(n, self.out_channels, device=x.device, dtype=torch.float32)
        _lib.check(_lib.lib().ddnm_classifier_forward(self.engine(n), _lib.ptr(x), _lib.ptr(t), _lib.ptr(logits), _lib.cur_stream()))
        return logits

    def __call__(self, x, timesteps):
        return self.forward(x, timesteps)

    def profile(self, x, t):
        """per-op timing of one eager forward + backward (labels 0, scale 1 unless a grad() call set others)"""
        import json
        x, t, n = self._inputs(x, t)
        logits = torch.empty(n, self.out_channels, device=x.device, dtype=torch.float32)
        buf = C.create_string_buffer(1 << 21)
        _lib.check(_lib.lib().ddnm_unet_profile(self.engine(n), _lib.ptr(x), _lib.ptr(t), _lib.ptr(logits), _lib.cur_stream(), buf, len(buf)))
        return json.loads(buf.value.decode())

    def grad(self, x, timesteps, y, scale=1.0, return_logits=False):
        """scale * d/dx sum_b log_softmax(self(x, t))[b, y_b] (the reference's cond_fn, diffusion.py:183-189)."""
        x, t, n = self._inputs(x, timesteps)
        labels = torch.as_tensor(y, device=x.device).reshape(-1).to(torch.int32).contiguous()
        if labels.numel() != n:
            raise _lib.DDNMError(f"{labels.numel()} labels for a batch of {n}")
        g = torch.empty_like(x)
        logits = torch.empty(n, self.out_channels, device=x.device, dtype=torch.float32) if return_logits else None
        _lib.check(_lib.lib().ddnm_classifier_grad(self.engine(n), _lib.ptr(x), _lib.ptr(t), _lib.ptr(labels), float(scale), _lib.ptr(g),
                                                   _lib.ptr(logits), _lib.cur_stream()))
        return (g, logits) if return_logits else g


def create_classifier(image_size, classifier_use_fp16, classifier_width, classifier_depth, classifier_attention_resolutions,
                      classifier_use_scale_shift_norm, classifier_resblock_updown, classifier_pool):
    """guided_diffusion.script_util.create_classifier (:229-267), same signature."""
    if image_size == 512:
        channel_mult = (0.5, 1, 1, 2, 2, 4, 4)
    elif image_size == 256:
        channel_mult = (1, 1, 2, 2, 4, 4)
    elif image_size == 128:
        channel_mult = (1, 1, 2, 3, 4)
    elif image_size == 64:
        channel_mult = (1, 2, 3, 4)
    else:
        raise ValueError(f"unsupported image size: {image_size}")
    attention_ds = [image_size // int(res) for res in classifier_attention_resolutions.split(",")]
    return EncoderUNetModel(image_size=image_size, in_channels=3, model_channels=classifier_width, out_channels=1000,
                            num_res_blocks=classifier_depth, attention_resolutions=tuple(attention_ds), channel_mult=channel_mult,
                            use_fp16=classifier_use_fp16, num_head_channels=64, use_scale_shift_norm=classifier_use_scale_shift_norm,
                            resblock_updown=classifier_resblock_updown, pool=classifier_pool)
