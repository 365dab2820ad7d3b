"""Data-parallel inference over the GPUs of one box: one process per GPU, clips sharded on dim 0, weights
replicated by one broadcast, a single all-gather of the logits per step.

This is the H100 counterpart of the reference's only multi-GPU construct, ``torch.nn.DataParallel(model)``
(examples/imagenet_eval.py:136, nonlocalnet.py:604): scatter the batch, run replicas, gather outputs.  Clips are
independent (eval-mode BN, per-sample attention), so the data path needs no collective until the
``[B/world, num_classes]`` fp32 logits are gathered -- a few KB per rank, latency-bound, issued on NCCL over
NVLink/NVSwitch (gloo in the CPU tests).
"""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Initialise torch.distributed from RANK / WORLD_SIZE / MASTER_* (torchrun).  Returns (rank, world, local)."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_bounds(n_items, world, rank):
    """Contiguous, balanced split of ``n_items`` clips: the first ``n_items % world`` ranks get one extra."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(x, world=None, rank=None):
    """This rank's slice of a batch (what DataParallel's scatter does on dim 0)."""
    if world is None:
        world = dist.get_world_size() if dist.is_initialized() else 1
    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    lo, hi = shard_bounds(x.shape[0], world, rank)
    return x[lo:hi]


def broadcast_parameters(module, src=0):
    """Replicate weights and buffers from ``src`` (DataParallel's replicate step, done once instead of per call)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    for t in list(module.parameters()) + list(module.buffers()):
        dist.broadcast(t.data, src=src)


def gather_logits(local_logits, total):
    """All-gather per-rank logits of a ``shard_bounds`` split back into batch order: [total, classes]."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local_logits
    world = dist.get_world_size()
    base, extra = divmod(total, world)
    if extra == 0:                            # equal shards: one flat all-gather straight into batch order
        out = torch.empty((total, local_logits.shape[1]), dtype=local_logits.dtype, device=local_logits.device)
        dist.all_gather_into_tensor(out, local_logits.contiguous())
        return out
    pad_rows = base + 1
    padded = local_logits
    if local_logits.shape[0] < pad_rows:      # equal-size buffers for all_gather
        padded = torch.cat([local_logits, local_logits.new_zeros(pad_rows - local_logits.shape[0],
                                                                 local_logits.shape[1])])
    bufs = [torch.empty_like(padded) for _ in range(world)]
    dist.all_gather(bufs, padded.contiguous())
    parts = []
    for r, b in enumerate(bufs):
        lo, hi = shard_bounds(total, world, r)
        parts.append(b[:hi - lo])
    return torch.cat(parts)


class DataParallelForward:
    """``model`` replicated on every rank; ``__call__(full_batch)`` returns the full logits on every rank."""

    def __init__(self, model, forward_fn=None):
        self.model = model
        self.forward_fn = forward_fn if forward_fn is not None else model
        broadcast_parameters(model)

    def __call__(self, full_batch):
        world = dist.get_world_size() if dist.is_initialized() else 1
        if full_batch.shape[0] < world:
            raise ValueError("batch of %d clips cannot be sharded over %d ranks" % (full_batch.shape[0], world))
        return gather_logits(self.forward_fn(shard_batch(full_batch)), full_batch.shape[0])
