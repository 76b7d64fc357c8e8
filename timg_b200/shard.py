"""Multi-GPU plumbing for the frame-sharded path (SURVEY.md 8e): frames are independent units,
each rank encodes a contiguous chunk on its own GPU, and the only exchange is the gather of the
encoded byte buffers to rank 0 (NCCL on GPUs; the same code runs over gloo on CPU for tests).

The reference has no counterpart (single process; frames go one Send() at a time to one tty,
src/renderer.cc:55-58); what is mirrored is its ordering contract: rank 0 ends up with the frames'
bytes concatenated in display order, as BufferedWriteSequencer's FIFO would write them
(src/buffered-write-sequencer.cc:70-89).
"""
import torch
import torch.distributed as dist


def shard_range(n_frames, rank, world):
    """Contiguous chunk [lo, hi) of frames for `rank`: sizes differ by at most one."""
    base, extra = divmod(n_frames, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def animation_chunk(n_frames, rank, world):
    """Delta-encoded animations (block modes): frame k depends on frame k-1's SCALED PIXELS only (the backing
    store equals the previous frame, src/unicode-block-canvas.cc:244,310), so a rank that owns [lo, hi) loads one
    extra halo frame lo-1 and encodes with Batch.animation = 2 (frame 0 of the batch is then a reference only).
    Returns (first frame to load, frames to load, animation flag)."""
    lo, hi = shard_range(n_frames, rank, world)
    if hi <= lo:
        return lo, 0, 1
    return (lo, hi - lo, 1) if lo == 0 else (lo - 1, hi - lo + 1, 2)


class _Gather:
    """An in-flight gather_encoded_async: wait() finishes it (on NCCL that makes the *current CUDA
    stream* wait, not the host) and returns what gather_encoded returns."""

    def __init__(self, works, result, fix, keep=()):
        self._works, self._result, self._fix, self._keep = works, result, fix, keep   # keep: buffers in flight

    def wait(self):
        for w in self._works:
            w.wait()
        for fs, base in self._fix:
            if base:
                fs += base
        self._works, self._fix, self._keep = [], [], ()
        return self._result


def gather_encoded_async(payload, offsets, dst=0, group=None):
    """Start gathering this rank's encoded frames to `dst`; returns a handle whose wait() yields, on
    `dst`, (all_bytes uint8 tensor, all_offsets int64 [N+1]) with every rank's frames in rank order,
    and (None, None) elsewhere.  `payload` (uint8, frames back to back) and `offsets` (int64 [n+1], same
    device) must stay untouched until wait() -- callers that keep encoding meanwhile double-buffer them,
    which is how a stream of pages / video windows hides the exchange behind the next batch's kernels.

    One size exchange (all_gather of [frame count, byte total], the only host sync), then
    point-to-point sends of exactly the encoded bytes and offsets straight into their final place on
    `dst` (no padding, no concat)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dev = payload.device
    n_local = offsets.numel() - 1
    meta = torch.stack([torch.tensor(n_local, dtype=torch.int64, device=dev), offsets[n_local].to(torch.int64)])
    metas = [torch.empty(2, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(metas, meta, group=group)
    m = torch.stack(metas).cpu().tolist()                      # the only host sync
    counts = [int(v[0]) for v in m]
    totals = [int(v[1]) for v in m]
    if rank != dst:
        ops = []
        offs_out = offsets[1: n_local + 1].to(torch.int64).contiguous()
        if totals[rank]:
            ops.append(dist.P2POp(dist.isend, payload[: totals[rank]], dst, group))
        if counts[rank]:
            ops.append(dist.P2POp(dist.isend, offs_out, dst, group))
        return _Gather(dist.batch_isend_irecv(ops) if ops else [], (None, None), [], (payload, offs_out))
    all_bytes = torch.empty(sum(totals), dtype=torch.uint8, device=dev)
    all_offs = torch.zeros(sum(counts) + 1, dtype=torch.int64, device=dev)
    ops, bbase, fbase, fix = [], 0, 0, []
    for r in range(world):
        bs, fs = all_bytes[bbase: bbase + totals[r]], all_offs[1 + fbase: 1 + fbase + counts[r]]
        if r == rank:
            bs.copy_(payload[: totals[r]])
            fs.copy_(offsets[1: n_local + 1])
        else:
            if totals[r]:
                ops.append(dist.P2POp(dist.irecv, bs, r, group))
            if counts[r]:
                ops.append(dist.P2POp(dist.irecv, fs, r, group))
        fix.append((fs, bbase))
        bbase += totals[r]
        fbase += counts[r]
    return _Gather(dist.batch_isend_irecv(ops) if ops else [], (all_bytes, all_offs), fix)


def gather_encoded(payload, offsets, dst=0, group=None):
    """gather_encoded_async(...).wait(): see there."""
    return gather_encoded_async(payload, offsets, dst, group).wait()


class AbiGather:
    """The C-ABI gather (b200timg_gather, timg_b200/csrc/gather.cu) driven from Python: NCCL communicator created
    inside the library, fixed slots, no host synchronisation per gather.  torch.distributed is used once, to hand
    rank 0's ncclUniqueId to the other ranks."""

    class _Ticket:
        def __init__(self, owner, ticket, dst, dst_offsets):
            self.owner, self.ticket, self.dst, self.dst_offsets = owner, ticket, dst, dst_offsets

        def wait(self, block_host=False):
            """Order the compute stream (or, with block_host, the host) after this gather.  On the root returns
            (bytes of all ranks in fixed slots, absolute offsets [world * (n + 1)]), else (None, None)."""
            self.owner._chk(self.owner.L.b200timg_gather_wait(self.owner.ctx.h, self.ticket, int(block_host)))
            return self.dst, self.dst_offsets

    def __init__(self, ctx, n_frames, slot_bytes, root=0, group=None, buffers=2):
        import ctypes as C
        import timg_b200
        self.L, self.ctx, self.n, self.slot, self.root = timg_b200.lib(), ctx, n_frames, int(slot_bytes), root
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        ident = C.create_string_buffer(128)
        if self.rank == root:
            self._chk(self.L.b200timg_gather_unique_id(ident))
        box = [ident.raw]
        dist.broadcast_object_list(box, src=root, group=group)
        self._chk(self.L.b200timg_gather_init(ctx.h, box[0], self.rank, self.world))
        dev = torch.device("cuda", ctx.device)
        self.k, self.dsts, self.dst_offs = 0, [], []
        if self.rank == root:
            self.dsts = [torch.empty(self.world * self.slot, dtype=torch.uint8, device=dev) for _ in range(buffers)]
            self.dst_offs = [torch.zeros(self.world * (n_frames + 1), dtype=torch.int64, device=dev) for _ in range(buffers)]
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.dst = self.dst_offsets = None

    def _chk(self, rc):
        if rc < 0:
            raise RuntimeError(self.L.b200timg_last_error(self.ctx.h).decode())

    def start(self, payload, offsets):
        """payload: uint8 cuda tensor with >= slot_bytes capacity; offsets: int64/uint64 [n+1] on the same device."""
        i = self.k % max(1, len(self.dsts)) if self.dsts else 0
        self.k += 1
        if self.rank == self.root:
            self.dst, self.dst_offsets = self.dsts[i], self.dst_offs[i]
            rc = self.L.b200timg_gather(self.ctx.h, payload.data_ptr(), offsets.data_ptr(), self.n, self.slot,
                                        self.dst.data_ptr(), self.dst_offsets.data_ptr(), self.status.data_ptr(), self.root)
        else:
            rc = self.L.b200timg_gather(self.ctx.h, payload.data_ptr(), offsets.data_ptr(), self.n, self.slot, None, None, None,
                                        self.root)
        self._chk(rc)
        return AbiGather._Ticket(self, rc, self.dst, self.dst_offsets)
