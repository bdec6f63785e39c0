"""Process-group helpers -- mirror of reference utils/distributed.py (NCCL via torch.distributed; `gloo` is accepted
so the multi-rank logic is testable on CPU).  The data path shards samples across ranks; the only exchange per
step is DDP's bucketed gradient all-reduce plus a 3-scalar loss reduce (SURVEY.md 2.4)."""
import os

import torch
import torch.distributed as dist


def setup_distributed(backend="nccl"):
    """torchrun environment -> process group.  Returns True when running distributed."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return False
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if backend == "nccl":
        torch.cuda.set_device(local_rank)
    if not dist.is_initialized():
        if backend == "nccl":   # bind the communicator to this rank's device up front (no device guessing at the first barrier)
            dist.init_process_group(backend=backend, init_method="env://", device_id=torch.device("cuda", local_rank))
        else:
            dist.init_process_group(backend=backend, init_method="env://")
    synchronize()
    return True


def is_distributed():
    return dist.is_available() and dist.is_initialized()


def get_rank():
    return dist.get_rank() if is_distributed() else 0


def primary():
    return get_rank() == 0


def get_world_size():
    return dist.get_world_size() if is_distributed() else 1


def synchronize():
    if is_distributed() and dist.get_world_size() > 1:
        dist.barrier()


def all_gather(tensor, cat=True):
    """Gather equally-shaped tensors from every rank (reference distributed.py:87-100)."""
    if get_world_size() == 1:
        return tensor if cat else [tensor]
    out = [torch.empty_like(tensor) for _ in range(get_world_size())]
    dist.all_gather(out, tensor.contiguous())
    return torch.cat(out, 0) if cat else out


def all_gatherv(tensor):
    """Gather tensors whose first dimensions differ across ranks, concatenated in rank order (reference
    distributed.py:103-122): the sizes are gathered first, every rank pads to the largest, the padding is dropped."""
    if get_world_size() == 1:
        return tensor
    counts = all_gather(torch.tensor([tensor.size(0)], device=tensor.device)).tolist()
    padded = torch.zeros((max(counts),) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
    padded[:tensor.size(0)] = tensor
    return torch.cat([part[:c] for part, c in zip(all_gather(padded, cat=False), counts)], 0)


def rank0_to_all(tensor):
    """Rank 0's value of `tensor` on every rank (reference distributed.py:134-137)."""
    return all_gather(tensor)[0]


def all_reduce_mean(tensor):
    if get_world_size() == 1:
        return tensor
    t = tensor.clone()
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t / get_world_size()


def reduce_loss_dict(loss_dict):
    """Mean of each scalar loss on rank 0 (reference distributed.py:140-162): ONE reduce of the stacked scalars."""
    world = get_world_size()
    if world < 2:
        return loss_dict
    with torch.no_grad():
        keys = sorted(loss_dict.keys())
        stacked = torch.stack([loss_dict[k].detach().reshape(()) for k in keys], 0)
        dist.reduce(stacked, dst=0)
        if dist.get_rank() == 0:
            stacked = stacked / world
        return {k: v for k, v in zip(keys, stacked)}
