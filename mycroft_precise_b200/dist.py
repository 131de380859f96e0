"""Multi-GPU plumbing: independent audio streams are block-sharded over ranks (one process per
GPU, torch.distributed); the only exchange on the path is the all-reduce of the detection count
(SURVEY 8e).  Works with the ``nccl`` backend on GPUs and ``gloo`` on CPU (tests).
"""
import os


def shard_range(n_streams: int, rank: int, world: int):
    """Contiguous block sharding: stream s lives on rank s // ceil(n/world).  A stream's state can move to another handle or
    rank with StreamBatch.export_streams / import_streams; carrying the snapshot between ranks is the caller's."""
    per = -(-n_streams // world)
    lo = min(rank * per, n_streams)
    hi = min(lo + per, n_streams)
    return lo, hi


def owner_of(stream: int, n_streams: int, world: int) -> int:
    per = -(-n_streams // world)
    return stream // per


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's env (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*).
    Returns (rank, local_rank, world).  Single process when WORLD_SIZE is unset or 1."""
    import torch
    import torch.distributed as dist
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = 'nccl' if torch.cuda.is_available() else 'gloo'
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        kw = {}
        if backend == 'nccl':
            torch.cuda.set_device(local)
            kw['device_id'] = torch.device('cuda', local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kw)
    return rank, local, world


def gpu_numa_cpus(local_rank: int):
    """CPUs of the NUMA node the GPU's PCIe root hangs off (sysfs), or None when the platform does not say."""
    import torch
    try:
        pr = torch.cuda.get_device_properties(local_rank)
        dev = '%04x:%02x:%02x.0' % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
        node = int(open('/sys/bus/pci/devices/%s/numa_node' % dev).read().strip())
        if node < 0:
            return None
        cpus = set()
        for part in open('/sys/devices/system/node/node%d/cpulist' % node).read().strip().split(','):
            if '-' in part:
                a, b = part.split('-')
                cpus.update(range(int(a), int(b) + 1))
            elif part:
                cpus.add(int(part))
        return cpus or None
    except Exception:
        return None


def bind_to_gpu_numa_node(local_rank: int):
    """Pin this process to the CPUs next to its GPU BEFORE it allocates pinned host buffers: first-touch then places the staging
    memory on the GPU's NUMA node, and the host-fed tick (pb_update_host) does not cross the socket interconnect.  Returns the
    CPU set used (restricted to what the process was allowed before) or None when nothing was changed."""
    cpus = gpu_numa_cpus(local_rank)
    if not cpus or not hasattr(os, 'sched_setaffinity'):
        return None
    allowed = os.sched_getaffinity(0) & cpus
    if not allowed:
        return None
    os.sched_setaffinity(0, allowed)
    return sorted(allowed)


class DetectionCounter:
    """Per-rank detection counts -> global sum.  ``local`` is a 1-element (or [k]) integer tensor that the device kernels
    accumulate into.

    ``all_reduce`` enqueues one SUM all-reduce on the current stream (8..24 bytes, latency-bound: ~25 us of every tick).
    ``all_reduce_overlapped`` takes it off the tick's critical path (SURVEY 8e: "overlap with the next tick's K1"): only a
    snapshot copy of the counter stays on the compute stream; the all-reduce of the snapshot runs on a side stream under the
    next tick's MFCC kernel.  ``wait()`` joins the side stream (call it before reading ``total`` / before stopping a timer)."""

    def __init__(self, local):
        self.local = local
        self.total = local.clone()
        self._snap = [local.clone(), local.clone()]
        self._k = 0
        self._side = None
        self._done = None

    def all_reduce(self, async_op=False):
        import torch.distributed as dist
        self.total.copy_(self.local)
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            return dist.all_reduce(self.total, op=dist.ReduceOp.SUM, async_op=async_op)
        return None

    def all_reduce_overlapped(self):
        import torch
        import torch.distributed as dist
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        if not self.local.is_cuda:                       # CPU / gloo: nothing to overlap with
            return self.all_reduce()
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.local.device)
        snap = self._snap[self._k & 1]
        self._k += 1
        main = torch.cuda.current_stream(self.local.device)
        if self._done is not None:
            main.wait_event(self._done)                  # the snapshot buffer written two ticks ago has been reduced
        snap.copy_(self.local)                           # the only work left on the compute stream
        ev = torch.cuda.Event()
        ev.record(main)
        with torch.cuda.stream(self._side):
            self._side.wait_event(ev)
            if multi:
                dist.all_reduce(snap, op=dist.ReduceOp.SUM)
            self.total.copy_(snap)
            self._done = torch.cuda.Event()
            self._done.record(self._side)
        return None

    def wait(self):
        """Make the current stream wait for every overlapped all-reduce issued so far."""
        import torch
        if self._done is not None:
            torch.cuda.current_stream(self.local.device).wait_event(self._done)
