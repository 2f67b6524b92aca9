"""Instance-parallel sharding of the denoise path across GPUs (SURVEY 8e).

The reference shards its test set over DDP ranks with batch size 1 (train.py:106-115,
pl_meta_model.py:194-198): instances never interact, so the GPU path is one process per GPU,
each owning a contiguous block of instances, NO collective inside the 50-step loop, and one
all_gather of the final heatmaps at the end (north_star).  Works with the nccl backend on GPUs and
with gloo on CPU tensors (tests/test_distributed_cpu.py).
"""
import torch
import torch.distributed as dist


def shard_range(n_items, rank, world):
  """Contiguous, balanced block [lo, hi) of rank `rank`: first n % world ranks get one extra item."""
  if world < 1 or not (0 <= rank < world):
    raise ValueError(f"bad rank/world {rank}/{world}")
  base, extra = divmod(int(n_items), int(world))
  lo = rank * base + min(rank, extra)
  return lo, lo + base + (1 if rank < extra else 0)


def gather_heatmaps(local, sizes=None, group=None):
  """All-gather per-rank heatmap tensors (1-D, possibly different lengths) into a list ordered by rank.

  local: 1-D float tensor of this rank.  sizes: optional list of every rank's length (skips the size
  exchange).  Ragged lengths are padded to the max for the collective and trimmed afterwards."""
  world = dist.get_world_size(group)
  if world == 1:
    return [local]
  if sizes is None:
    n = torch.tensor([local.numel()], device=local.device, dtype=torch.int64)
    all_n = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(all_n, n, group=group)
    sizes = [int(x.item()) for x in all_n]
  m = max(sizes)
  buf = local if local.numel() == m else torch.cat([local, local.new_zeros(m - local.numel())])
  out = [torch.empty(m, device=local.device, dtype=local.dtype) for _ in range(world)]
  dist.all_gather(out, buf.contiguous(), group=group)
  return [o[:s] for o, s in zip(out, sizes)]


def denoise_sharded(instances, run_batch, rank=None, world=None, batch=16, group=None, device=None,
                    dtype=torch.float32):
  """Round of instance-parallel inference.

  instances: list of problem descriptions (anything `run_batch` understands), identical on all ranks.
  run_batch(list_of_instances) -> 1-D float tensor: concatenated heatmaps of that block-diagonal batch.
  Every rank processes its contiguous shard in batches of `batch`; returns, on every rank, the list of
  per-rank concatenated heatmaps (rank order == instance order).
  device / dtype: where an EMPTY shard (more ranks than instances) lives; every rank must join the collectives with a
  tensor of the backend's device (CUDA for nccl) and of the same dtype as the other ranks' heatmaps.  Default device:
  the current CUDA device under nccl, the CPU otherwise."""
  rank = dist.get_rank(group) if rank is None else rank
  world = dist.get_world_size(group) if world is None else world
  lo, hi = shard_range(len(instances), rank, world)
  outs = [run_batch(instances[i:min(i + batch, hi)]) for i in range(lo, hi, batch)]
  if outs:
    local = torch.cat(outs)
  else:
    if device is None:
      nccl = dist.is_initialized() and dist.get_backend(group) == "nccl"
      device = torch.device("cuda", torch.cuda.current_device()) if nccl else torch.device("cpu")
    local = torch.zeros(0, device=device, dtype=dtype)
  return gather_heatmaps(local, group=group)
