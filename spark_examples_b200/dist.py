"""Multi-GPU plumbing (one process per GPU, torch.distributed): the path shards over variants -- Spark partition p is
owned by rank p % world -- and the only exchange is the all-reduce of the partial Grams, the `reduceByKey(_ + _)` of
VariantsPca.scala:190."""
from __future__ import annotations

from typing import List, Tuple


def rank_world() -> Tuple[int, int]:
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(), dist.get_world_size()
    except ImportError:
        pass
    return 0, 1


def partition_owner(partition_id: int, world: int) -> int:
    return partition_id % world


def my_partitions(num_partitions: int, rank: int, world: int) -> List[int]:
    return [p for p in range(num_partitions) if partition_owner(p, world) == rank]


def allreduce_gram(gram_tensor):
    """Sum the n x n int32 partial Grams of all ranks in place (NCCL on GPU tensors, gloo on CPU tensors)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(gram_tensor, op=dist.ReduceOp.SUM)
    return gram_tensor


def allreduce_count(value: int, device=None) -> int:
    """Sum of one integer over all ranks (variants per rank, for the int32 bound of the summed Gram)."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return int(value)
    t = torch.tensor([int(value)], dtype=torch.int64, device=device if device is not None else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return int(t.item())


def gather_to_rank0(obj) -> list:
    """`obj` of every rank in rank order on rank 0 (other ranks get None); a single process gets [obj]."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return [obj]
    out = [None] * dist.get_world_size() if dist.get_rank() == 0 else None
    dist.gather_object(obj, out, dst=0)
    return out


def allreduce_f64(arr, device=None):
    """Element-wise sum of a float64 numpy array over all ranks (projection partial sums); returns numpy."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return arr
    t = torch.from_numpy(arr).to(device if device is not None else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t.cpu().numpy()
