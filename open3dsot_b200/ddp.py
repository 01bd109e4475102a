"""Data-parallel training plumbing: one process per GPU, one flat gradient bucket, one NCCL all-reduce per step.

The reference trains with Lightning's DDP plugin (main.py:82-85: `pl.Trainer(gpus=-1, accelerator='ddp')`), i.e.
torch DDP with bucketed all-reduce, per-rank BatchNorm statistics (no sync_batchnorm) and a per-GPU batch size.
The gradient payload is <= 9 MB (SURVEY.md §2.2), so a single flat bucket over NVLink/NVSwitch is latency-bound;
`FlatParams` makes every `p.grad` a view into one contiguous buffer, so the collective needs no packing copy and
the optimizer can run as one kernel over the flat buffers.
"""
import torch
import torch.distributed as dist


class FlatParams:
    """Re-homes a module's parameters and gradients into two flat fp32 buffers (views keep the module usable)."""

    def __init__(self, module: torch.nn.Module):
        self.params = [p for p in module.parameters() if p.requires_grad]
        total = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat = torch.empty(total, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(total, dtype=torch.float32, device=dev)
        off = 0
        for p in self.params:
            n = p.numel()
            self.flat[off:off + n].copy_(p.data.reshape(-1))
            p.data = self.flat[off:off + n].view_as(p)
            p.grad = self.grad[off:off + n].view_as(p)
            off += n
        self.numel = total

    def zero_grad(self):
        self.grad.zero_()


def init_distributed(backend=None):
    """Initialise torch.distributed from the torchrun environment (RANK / WORLD_SIZE / MASTER_*)."""
    import os
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world == 1:
        return 0, 1, 0
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if backend is None:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
    if backend == "nccl":
        torch.cuda.set_device(local)
    if not dist.is_initialized():
        dist.init_process_group(backend=backend)
    return rank, world, local


def pin_to_gpu_numa_node(local_rank):
    """Bind this process (and the threads it starts from now on) to the CPUs next to its GPU.  With eight ranks on a
    two-socket host, a rank whose Python thread runs on the far socket issues its copies and launches across the socket
    link; the skew lands in every collective.  Best effort: NVML's ideal-CPU mask, silently skipped when unavailable."""
    import os
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        index = int(vis.split(",")[local_rank]) if vis and vis.split(",")[local_rank].isdigit() else local_rank
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        ncpu = os.cpu_count() or 1
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (ncpu + 63) // 64)
        cpus = {64 * w + b for w, m in enumerate(words) for b in range(64) if (m >> b) & 1}
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            return len(cpus)
    except Exception:
        return 0
    return 0


def is_distributed():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def broadcast_parameters(flat: FlatParams, module: torch.nn.Module):
    """Rank 0's parameters and buffers become everyone's (DDP does the same at construction)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    dist.broadcast(flat.flat, src=0)
    broadcast_buffers(module)


def broadcast_buffers(module: torch.nn.Module):
    """Rank 0's buffers (BatchNorm running statistics) become everyone's; no-op on a single rank.  The collective writes
    bump no tensor version, so the weights generation advances for the static-weight caches."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    from . import runtime
    for b in module.buffers():
        dist.broadcast(b, src=0)
    runtime.advance_weights_generation()


def allreduce_gradients(flat: FlatParams, async_op=False):
    """Mean of the flat gradient bucket over all ranks (sum then divide, as DDP does)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return None
    flat.grad.div_(dist.get_world_size())
    return dist.all_reduce(flat.grad, op=dist.ReduceOp.SUM, async_op=async_op)
