"""Multi-GPU: independent images shard over ranks, zero traffic inside the sampling loop, ONE all-gather of the
restored images at the end (BASELINE.json north_star; replaces the reference's per-forward nn.DataParallel
scatter / replicate / gather, guided_diffusion/diffusion.py:140,164)."""
import torch
import torch.distributed as dist


def shard_rows(n_rows, rank, world):
    """Contiguous row range [lo, hi) of rank ``rank``; ranges differ by at most one row and cover [0, n_rows)."""
    base, extra = divmod(n_rows, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def sharded_sample(sample_fn, x, y, noise=None, group=None):
    """Run ``sample_fn(x_rows, y_rows, noise_rows) -> (x0_rows, x0_pred_rows)`` on this rank's rows and all-gather.

    x: (B, ...), y: (B, M), noise: (n_pairs, B, ...) or None — the GLOBAL batch, identical on every rank (so a sharded
    run reproduces the unsharded one row for row).  Returns the full (B, ...) results on every rank.
    """
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    B = x.shape[0]
    lo, hi = shard_rows(B, rank, world)
    nz = None if noise is None else noise[:, lo:hi]
    x0, x0p = sample_fn(x[lo:hi], y[lo:hi], nz)
    return _gather_rows(x0, x0p, B, lo, hi, world, group)


def sharded_sample_seeded(sample_fn, x, y, seed, group=None):
    """As ``sharded_sample`` with library-drawn noise: runs ``sample_fn(x_rows, y_rows, seed, row_offset=lo)`` on this rank's rows
    [lo, hi) and all-gathers.  A seeded draw depends on the GLOBAL row index only, so no rank needs a noise tape.  With the
    model (and classifier) in ``batch_invariant`` mode the result equals the unsharded ``sample_fn(x, y, seed, row_offset=0)``
    bit for bit, at any world size; otherwise it agrees to fp32 reassociation."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    B = x.shape[0]
    lo, hi = shard_rows(B, rank, world)
    x0, x0p = sample_fn(x[lo:hi], y[lo:hi], seed, row_offset=lo)
    return _gather_rows(x0, x0p, B, lo, hi, world, group)


def _gather_rows(x0, x0p, B, lo, hi, world, group):
    """All ranks' (x0, x0_pred) row blocks -> the full batch on every rank."""
    if world == 1:
        return x0, x0p
    counts = [shard_rows(B, r, world) for r in range(world)]
    width = max(h - l for l, h in counts)
    # one collective: both results ride in a single padded buffer
    buf = torch.zeros((2, width) + tuple(x0.shape[1:]), dtype=x0.dtype, device=x0.device)
    buf[0, : hi - lo] = x0
    buf[1, : hi - lo] = x0p
    out = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(out, buf, group=group)
    full0 = torch.cat([out[r][0, : h - l] for r, (l, h) in enumerate(counts)], dim=0)
    full1 = torch.cat([out[r][1, : h - l] for r, (l, h) in enumerate(counts)], dim=0)
    return full0, full1
