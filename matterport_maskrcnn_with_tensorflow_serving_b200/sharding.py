"""Multi-GPU plumbing: images are independent units, so a batch shards by image with no
collective on the data path; the only exchange is the final gather of per-image mask
canvases to rank 0 (BASELINE.json north_star; the reference itself is single-image,
single-process: serve.py:48).

Two gathers, both into ONE receive buffer on rank 0 that is allocated once and holds the whole
batch in image order (rank 0's own shard is written there by its kernels, never copied):

  RootGather (NCCL)   the north_star's gather: point-to-point send / recv (NCCL has no gather
                      primitive), issued per chunk of images so that the send of chunk k
                      overlaps the expand kernels of chunk k+1; works with `gloo` on CPU
                      tensors, which is how tests/ cover world_size 2 without a GPU.
  PeerGather (fused)  rank 0 exports its receive buffer (CUDA IPC, csrc/peer.cu); the other
                      ranks map it and hand the mapped address to the expand kernels as their
                      output pointer: the kernels' bulk (TMA) stores travel over NVLink /
                      NVSwitch while the kernel is still computing -- compute and gather are
                      one kernel, no NCCL call and no host round trip; completion is a
                      system-scope flag per rank that rank 0's stream waits on.

Both move either layout: the reference's byte canvases [H,W,N] or the bit-packed extension
(8x fewer bytes through rank 0's NVLink ingress, which is what bounds the gather).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _native as N


def partition_images(costs, world_size):
    """Contiguous partition of images over ranks balancing `costs` (e.g. H*W*N bytes).

    Returns a list of (start, stop) per rank, covering range(len(costs)) in order.
    Contiguity keeps the gathered result in the original image order.  Greedy prefix
    split at multiples of total/world_size.
    """
    costs = np.asarray(costs, dtype=np.float64)
    n = len(costs)
    world_size = int(world_size)
    if world_size < 1:
        raise ValueError("world_size must be >= 1")
    if n == 0:
        return [(0, 0)] * world_size
    prefix = np.concatenate([[0.0], np.cumsum(costs)])
    total = prefix[-1]
    bounds = [0]
    for r in range(1, world_size):
        target = total * r / world_size
        # first index whose prefix reaches the target, but leave enough images for the rest
        i = int(np.searchsorted(prefix, target, side="left"))
        if i > 0 and abs(prefix[i - 1] - target) <= abs(prefix[min(i, n)] - target):
            i -= 1
        i = max(i, bounds[-1])
        i = min(i, n)
        bounds.append(i)
    bounds.append(n)
    return [(bounds[r], bounds[r + 1]) for r in range(world_size)]


def equal_partition(n_images, world_size):
    """Contiguous blocks of ceil/floor(n/world) images (equal-cost images)."""
    return partition_images(np.ones(n_images), world_size)


def chunk_bounds(n_images, n_chunks):
    """Split range(n_images) into at most n_chunks contiguous, nearly equal, non-empty runs."""
    n_chunks = max(1, min(int(n_chunks), int(n_images))) if n_images > 0 else 1
    edges = [round(i * n_images / n_chunks) for i in range(n_chunks + 1)]
    return [(edges[i], edges[i + 1]) for i in range(n_chunks) if edges[i + 1] > edges[i]]


def gather_bytes_to_root(local, sizes, dst=0, group=None):
    """Gather ragged uint8 tensors to rank `dst` in one blocking step (fresh receive buffers).
    Kept for callers without a persistent plan; `RootGather` is the pipelined form.

    local: 1-D uint8 tensor of this rank's bytes (device or CPU).
    sizes: list of byte counts per rank (known to all ranks; derived from the partition).
    Returns on dst a list of tensors (one per rank, rank order); None elsewhere."""
    import torch.distributed as dist

    rank = dist.get_rank(group)
    world = dist.get_world_size(group)
    if len(sizes) != world:
        raise ValueError("sizes must have one entry per rank")
    if local.numel() != int(sizes[rank]):
        raise ValueError(f"rank {rank}: local has {local.numel()} bytes, sizes says {sizes[rank]}")
    if rank == dst:
        out = []
        ops = []
        for r in range(world):
            if r == dst:
                out.append(local)
            else:
                buf = torch.empty((int(sizes[r]),), dtype=torch.uint8, device=local.device)
                out.append(buf)
                if sizes[r] > 0:
                    ops.append(dist.P2POp(dist.irecv, buf, r, group))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
        return out
    if sizes[rank] > 0:
        for req in dist.batch_isend_irecv([dist.P2POp(dist.isend, local, dst, group)]):
            req.wait()
    return None


class RootGather:
    """Pipelined gather of per-rank byte ranges into one preallocated buffer on rank `dst`.

    sizes[r]: bytes rank r contributes (all ranks know all sizes: they follow from the
    partition).  On dst, `self.recv` is one uint8 tensor of sum(sizes) bytes and
    `self.slot(r)` is rank r's range in it -- dst's kernels write straight into `slot(dst)`.
    Elsewhere `self.recv` is None and the rank sends from its own buffer.

        g = RootGather(sizes, device)
        for (lo, hi) in byte ranges of this rank's chunks, in order:
            ... enqueue the kernels that produce local[lo:hi] on the current stream ...
            g.post(local, lo, hi)      # send (or, on dst, receive every peer's matching chunk)
        g.wait()                       # the current stream now waits for every transfer

    Every rank must post the same NUMBER of chunks (`chunk_ranges` gives matching splits of
    unequal shards).  With NCCL each post is ordered after the work already queued on the
    current stream and runs on NCCL's own stream, so later kernels overlap it."""

    def __init__(self, sizes, device, dst=0, group=None):
        import torch.distributed as dist

        self.dist = dist
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        if len(sizes) != self.world:
            raise ValueError("sizes must have one entry per rank")
        self.sizes = [int(s) for s in sizes]
        self.offsets = np.concatenate([[0], np.cumsum(self.sizes)]).astype(np.int64)
        self.dst = int(dst)
        self.recv = None
        if self.rank == self.dst:
            self.recv = torch.empty((int(self.offsets[-1]),), dtype=torch.uint8, device=device)
        self._reqs = []
        self._chunk = 0
        self._n_chunks = None
        self._ranges = None

    def slot(self, r):
        return self.recv[int(self.offsets[r]):int(self.offsets[r + 1])]

    @staticmethod
    def chunk_ranges(size, n_chunks, align=16):
        """n_chunks consecutive byte ranges covering [0, size), boundaries multiples of `align`
        (ranges may be empty when size is small): the same n_chunks on every rank."""
        edges = [min(size, (size * i // n_chunks) // align * align) for i in range(n_chunks)] + [size]
        return [(edges[i], edges[i + 1]) for i in range(n_chunks)]

    def begin(self, n_chunks, ranges_by_rank=None):
        """Start a gather of n_chunks chunks per rank.  ranges_by_rank[r] = the byte ranges
        rank r will send, in order (default: `chunk_ranges(sizes[r], n_chunks)`); every rank
        must pass the same table."""
        self._reqs = []
        self._chunk = 0
        self._n_chunks = int(n_chunks)
        self._ranges = ranges_by_rank

    def post(self, local=None, lo=0, hi=0):
        """Non-dst ranks: send local[lo:hi] as chunk number `self._chunk`.  dst: receive the
        matching chunk of every peer (its ranges follow from `chunk_ranges(sizes[r], n)`)."""
        dist = self.dist
        k, n = self._chunk, self._n_chunks
        self._chunk += 1
        ops = []
        if self.rank == self.dst:
            for r in range(self.world):
                if r == self.dst:
                    continue
                plo, phi = (self._ranges[r] if self._ranges is not None
                            else self.chunk_ranges(self.sizes[r], n))[k]
                if phi > plo:
                    ops.append(dist.P2POp(dist.irecv, self.slot(r)[plo:phi], r, self.group))
        elif hi > lo:
            ops.append(dist.P2POp(dist.isend, local[lo:hi], self.dst, self.group))
        if ops:
            self._reqs.extend(dist.batch_isend_irecv(ops))

    def wait(self):
        for req in self._reqs:
            req.wait()
        self._reqs = []


class PeerGather:
    """Fused compute + gather: rank `dst` owns one receive buffer, every rank's expand kernels
    write their output straight into it (their own range of it) over NVLink.

        pg = PeerGather(sizes, device)            # collective: exchanges the IPC handle
        ptr = pg.out_ptr()                        # where THIS rank's bytes go (device address)
        engine.enqueue_expand(stream, canvas_ptr=ptr)      # or enqueue_expand_packed(...)
        pg.signal(stream)                         # after this rank's kernels
        pg.wait(stream)                           # dst: stream proceeds when every rank signalled
        pg.recv                                   # dst: uint8 tensor over the whole buffer

    `close()` unmaps / frees; the buffer is allocated with cudaMalloc by libmrx (not by torch's
    caching allocator) so that the IPC handle covers exactly it."""

    HEADER = 4096     # flags live in front of the data (one uint32 per rank)

    def __init__(self, sizes, device, dst=0, group=None):
        import torch.distributed as dist

        self.lib = N.load()
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.dst = int(dst)
        self.sizes = [int(s) for s in sizes]
        # every rank's range starts 256-byte aligned
        starts, pos = [], self.HEADER
        for s in self.sizes:
            starts.append(pos)
            pos += (s + 255) // 256 * 256
        self.starts = starts
        self.total = pos
        self.epoch = 0
        self._base = C.c_void_p(0)
        self._owner = self.rank == self.dst
        # every step below is collective: a failure on ONE rank (no peer access, IPC refused by
        # the container) must fail the construction on EVERY rank, or the others would hang
        handle, err = [None], None
        try:
            if self._owner:
                N.check(self.lib.mrx_peer_alloc(self.total, C.byref(self._base)),
                        "mrx_peer_alloc")
                buf = C.create_string_buffer(N.MRX_PEER_HANDLE_BYTES)
                N.check(self.lib.mrx_peer_export(self._base, buf), "mrx_peer_export")
                handle = [bytes(buf.raw)]
        except Exception as e:      # noqa: BLE001
            err = e
        dist.broadcast_object_list(handle, src=self.dst, group=group)
        try:
            if not self._owner and handle[0] is not None:
                N.check(self.lib.mrx_peer_open(handle[0], C.byref(self._base)), "mrx_peer_open")
        except Exception as e:      # noqa: BLE001
            err = e
        ok = torch.tensor([0 if (err is not None or not self._base.value) else 1],
                          dtype=torch.int32, device=device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
        self.base = int(self._base.value or 0)
        self.recv = None
        self._all = None
        if int(ok.item()) == 0:
            self._release_local()
            raise RuntimeError(f"peer memory unavailable on at least one rank ({err})")
        if self._owner:
            self._all = torch.as_tensor(N.DeviceBytes(self.base, self.total), device=device)
            self._all[:self.HEADER].zero_()
            self.recv = self._all[self.HEADER:]
            torch.cuda.synchronize()
        dist.barrier(group)

    def _release_local(self):
        if self._base.value:
            self.recv = None
            self._all = None
            if self._owner:
                self.lib.mrx_peer_free(self._base)
            else:
                self.lib.mrx_peer_close(self._base)
            self._base = C.c_void_p(0)

    def out_ptr(self, r=None):
        return self.base + self.starts[self.rank if r is None else r]

    def slot(self, r):
        lo = self.starts[r] - self.HEADER
        return self.recv[lo:lo + self.sizes[r]]

    def next_epoch(self):
        self.epoch += 1
        return self.epoch

    def signal(self, stream=None):
        """After everything queued on `stream`: tell dst that this rank's bytes have landed."""
        with N.on_stream(stream):
            N.check(self.lib.mrx_peer_signal(self.base + 4 * self.rank, self.epoch,
                                             N.stream_ptr()), "mrx_peer_signal")

    def wait(self, stream=None):
        """dst only: `stream` proceeds once every rank has signalled the current epoch."""
        if not self._owner:
            return
        with N.on_stream(stream):
            N.check(self.lib.mrx_peer_wait(self.base, self.world, self.epoch, N.stream_ptr()),
                    "mrx_peer_wait")

    def close(self):
        torch.cuda.synchronize()
        self.dist_barrier()
        if not self._owner:          # mappings go first, the allocation last
            self._release_local()
        self.dist_barrier()
        if self._owner:
            self._release_local()

    def dist_barrier(self):
        import torch.distributed as dist

        dist.barrier(self.group)


def bind_to_gpu_numa_node(local_rank):
    """Pin this process to the CPUs of the NUMA node its GPU hangs off (torchrun does not):
    pinned host buffers allocated afterwards are node-local and the H2D / D2H copies do not
    cross the socket interconnect.  Returns a dict describing what was done (for the bench
    line); never raises -- without sysfs / NVML it reports why and leaves the affinity alone."""
    info = {"bound": False}
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(int(local_rank))
        bus = pynvml.nvmlDeviceGetPciInfo(h).busId
        bus = bus.decode() if isinstance(bus, bytes) else bus
        bus = bus.lower()
        if len(bus.split(":")[0]) == 8:          # NVML prints an 8-digit domain, sysfs a 4-digit one
            bus = bus[4:]
        with open(f"/sys/bus/pci/devices/{bus}/numa_node") as f:
            node = int(f.read().strip())
        info["pci"] = bus
        info["numa_node"] = node
        if node < 0:
            info["why"] = "sysfs reports no NUMA node for the GPU"
            return info
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = _parse_cpulist(f.read().strip())
        allowed = os.sched_getaffinity(0)
        cpus = sorted(set(cpus) & set(allowed))
        if not cpus:
            info["why"] = "no allowed CPU on the GPU's node"
            return info
        os.sched_setaffinity(0, cpus)
        info["bound"] = True
        info["cpus"] = len(cpus)
    except Exception as e:      # noqa: BLE001  (diagnostic helper: report, do not fail the job)
        info["why"] = f"{type(e).__name__}: {e}"
    return info


def _parse_cpulist(text):
    cpus = []
    for part in text.split(","):
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            cpus.extend(range(int(a), int(b) + 1))
        else:
            cpus.append(int(part))
    return cpus
