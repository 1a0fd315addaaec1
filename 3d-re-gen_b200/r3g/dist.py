"""Multi-GPU plumbing: one process per GPU, objects sharded round-robin, finished meshes gathered to rank 0.

The reference's only parallelism on this path is data-parallel over objects (src/2d_to_3d_models/run.py:176-194:
task i -> GPU i % num_devices through a process pool, results meet on disk).  Here rank r takes objects
{i : i % world == r} of the sorted list and rank 0 -- which runs the downstream scene assembly
(src/scene_reconstruction/run.py:62-76 reads <out>/3D/<name>/<name>.glb) -- receives every mesh over
NCCL (NVLink / NVSwitch).  Every mesh travels as one fixed-capacity `pack_mesh` message, [nv, nf, 0, 0, verts...,
faces...] as int32 words, with the capacity agreed across ranks, so rank 0 posts its receives without a size exchange:

  * MeshBatchGatherer: each rank packs its meshes into a [steps, capacity] staging buffer and sends it to rank 0 in
    one message at the end; rank 0 lands the used words through a two-slot pinned ring.  The stage-3 twin and
    bench.py at N > 1 use it.
  * MeshStreamGatherer: one message per rank and object on a side stream, under the next object's compute; rank 0
    lands it through a pinned ring on a consumer thread.  bench.py's e2e arm uses it at N = 1.

There is no compute kernel to fuse this with: the payload is a few MB per object, after the last kernel.
"""
import torch
import torch.distributed as dist


def shard_indices(n_items, rank=None, world=None):
    """Indices of the items this rank processes (round-robin, like task i -> GPU i % num_devices)."""
    if world is None:
        world = dist.get_world_size() if dist.is_initialized() else 1
    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    return list(range(rank, n_items, world))


def _world_rank():
    return (dist.get_world_size(), dist.get_rank()) if dist.is_initialized() else (1, 0)


def _agree_max(world, device, *values):
    """The element-wise maximum of `values` over all ranks, in one all_reduce.  Every rank must post the SAME message
    size (an NCCL send / recv pair with different counts is undefined) while callers size from their own meshes."""
    if world == 1:
        return [int(x) for x in values]
    t = torch.tensor([int(x) for x in values], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.tolist()


def _mesh_views(msg, nv, nf):
    """(verts float32 [nv, 3], faces int32 [nf, 3]): views into a pack_mesh message."""
    return msg[4:4 + 3 * nv].view(torch.float32).view(nv, 3), msg[4 + 3 * nv:4 + 3 * nv + 3 * nf].view(nf, 3)


def pack_mesh(buf, verts, faces, cap_v, cap_f):
    """[nv, nf, 0, 0, verts..., faces...] as int32 words into `buf` (device copy, asynchronous on the current stream)."""
    nv = 0 if verts is None else int(verts.shape[0])
    nf = 0 if faces is None else int(faces.shape[0])
    if nv > cap_v or nf > cap_f:
        raise ValueError(f"mesh ({nv} vertices, {nf} faces) exceeds the gather capacity ({cap_v}, {cap_f})")
    buf[:4] = torch.tensor([nv, nf, 0, 0], dtype=torch.int32).to(buf.device, non_blocking=True)
    if nv:
        buf[4:4 + 3 * nv].copy_(verts.reshape(-1).contiguous().view(torch.int32), non_blocking=True)
    if nf:
        buf[4 + 3 * nv:4 + 3 * nv + 3 * nf].copy_(faces.reshape(-1).to(torch.int32), non_blocking=True)
    return nv, nf


class MeshBatchGatherer:
    """Device-resident gather for a batch of objects per rank with NO collective while the objects compute: every
    finished mesh is packed into this rank's staging buffer [steps, cap] (no allocator traffic), and `finish()` moves
    the whole buffer to rank 0 in one NCCL message per peer.  `steps` and the capacities are agreed as the maxima over
    the ranks, so each rank may submit its own number of meshes (up to the `steps` it passed).  A send / recv kernel
    that is resident while a persistent, statically scheduled GEMM runs can hold one of its SMs until the peer arrives --
    measured at N = 8 as ~0.15 s per object when the per-object exchange of MeshStreamGatherer overlapped the next
    object -- so the device-resident arm of bench.py keeps its NVLink traffic out of the compute phase."""

    def __init__(self, cap_vertices, cap_faces, steps, device, to_host=False):
        self.world, self.rank = _world_rank()
        self.cap_v, self.cap_f, self.steps = _agree_max(self.world, device, cap_vertices, cap_faces, steps)
        self.cap = 4 + 3 * self.cap_v + 3 * self.cap_f
        self.stage = torch.empty(self.steps, self.cap, dtype=torch.int32, device=device)
        self.stage[:, :4] = 0               # a row that is never submitted reads as an absent object
        self.k = 0
        # everything finish() needs exists before the first object: rank 0's receive buffers, the pinned ring, and the
        # NCCL point-to-point connections (a first send / recv to a peer sets the channel up; done here on 4 words)
        self.recv = ([torch.empty_like(self.stage) for _ in range(self.world - 1)] if self.rank == 0 else [])
        self.ring = ([torch.empty(self.cap, dtype=torch.int32, pin_memory=self.stage.is_cuda) for _ in range(2)]
                     if to_host and self.rank == 0 else None)
        self._exchange(4)

    def _exchange(self, words=None):
        """Every peer's staging buffer (or its first `words` words of the first mesh) -> rank 0's receive buffers."""
        if self.world == 1 or self.steps == 0:
            return
        cut = (lambda b: b.view(-1)[:words]) if words else (lambda b: b)
        if self.rank == 0:
            ops = [dist.P2POp(dist.irecv, cut(self.recv[r - 1]), r) for r in range(1, self.world)]
        else:
            ops = [dist.P2POp(dist.isend, cut(self.stage), 0)]
        for w in dist.batch_isend_irecv(ops):
            w.wait()

    def submit(self, verts, faces):
        pack_mesh(self.stage[self.k], verts, faces, self.cap_v, self.cap_f)
        self.k += 1

    def finish(self, to_host=False, sink=None):
        """Moves every rank's staging buffer to rank 0 (one NCCL message per peer).  Returns, on rank 0, the per-rank
        buffers [world][steps, cap] on the device; elsewhere [].  to_host: rank 0 then copies the USED words of every
        mesh through a two-slot pinned ring (copy engine, large transfers) and calls sink(step, rank, verts, faces) with
        views into the slot as each one lands; rows whose header reads nv == nf == 0 are skipped."""
        self._exchange()
        if self.rank != 0:
            return []
        bufs = [self.stage] + self.recv
        if not to_host:
            return bufs
        cuda = self.stage.is_cuda
        hdr = torch.stack([b[:, :2] for b in bufs]).cpu()             # [world, steps, 2]: nv, nf of every mesh
        ring = self.ring or [torch.empty(self.cap, dtype=torch.int32, pin_memory=cuda) for _ in range(2)]
        done = [None, None]
        pending = []

        def deliver(item):
            slot, r, k, nv, nf = item
            if done[slot] is not None:
                done[slot].synchronize()
            if sink is not None:
                sink(k, r, *_mesh_views(ring[slot], nv, nf))
        i = 0
        for r in range(len(bufs)):
            for k in range(self.steps):
                nv, nf = int(hdr[r, k, 0]), int(hdr[r, k, 1])
                if nv == 0 and nf == 0:         # absent object, or a row its rank did not fill
                    continue
                slot = i % 2
                if len(pending) == 2:           # the slot about to be overwritten must have been delivered
                    deliver(pending.pop(0))
                n = 4 + 3 * nv + 3 * nf
                ring[slot][:n].copy_(bufs[r][k, :n], non_blocking=True)
                if cuda:
                    done[slot] = torch.cuda.Event()
                    done[slot].record()
                pending.append((slot, r, k, nv, nf))
                i += 1
        while pending:
            deliver(pending.pop(0))
        return bufs


class MeshStreamGatherer:
    """Per-object gather to rank 0, overlapped with the next object's compute (SURVEY.md section 8e: "run it on a side
    stream so rank 0 can start writing .glbs while others finish").

    Every rank calls `submit(verts, faces)` once per step (None, None when it has no object in that step) right after
    its object has been enqueued; all ranks make the same number of calls.  A step is one fixed-capacity message per
    peer -- [nv, nf, verts..., faces...] as int32 words -- so rank 0 can post its receives without knowing the sizes
    and without a host round trip; the messages move over NCCL on a SIDE stream (NVLink / NVSwitch; a few hundred MB
    per step) while the compute stream runs the next object.  On rank 0 the sizes are read one step later (by then the
    step's header copy has long landed: no stall), the payloads go device -> PINNED ring -> a consumer thread that
    hands the arrays to `sink(step, rank, verts, faces)` (views into the ring slot; default: copies kept for `finish()`).  Nothing on this path is
    a pageable synchronous `.cpu()` (round 1's limiter: 4.8 GB/s into rank 0).

    Also runs on gloo with CPU tensors (tests/test_dist_gloo.py), where streams do not exist and every wait is a host
    wait."""

    def __init__(self, cap_vertices, cap_faces, device=None, to_host=True, depth=2, sink=None):
        import queue
        import threading
        self.world, self.rank = _world_rank()
        self.cuda = torch.cuda.is_available() and (device is None or torch.device(device).type == "cuda") and (
            not dist.is_initialized() or dist.get_backend() == "nccl")
        self.device = torch.device(device) if device is not None else (
            torch.device("cuda", torch.cuda.current_device()) if self.cuda else torch.device("cpu"))
        self.cap_v, self.cap_f = _agree_max(self.world, self.device, cap_vertices, cap_faces)
        self.cap = 4 + 3 * self.cap_v + 3 * self.cap_f
        self.depth, self.to_host, self.step = depth, to_host, 0
        self.side = torch.cuda.Stream(self.device) if self.cuda else None
        i32 = dict(dtype=torch.int32, device=self.device)
        self.send = [torch.empty(self.cap, **i32) for _ in range(depth)]
        self.results, self.sink = {}, sink
        self.pending = []            # rank 0: steps whose headers have been requested but whose payloads are not read yet
        self._slot_done = [None] * depth   # event after which a send slot may be repacked (transfer / host copy done)
        if self.rank == 0:
            self.recv = [[torch.empty(self.cap, **i32) for _ in range(self.world - 1)] for _ in range(depth)]
            pin = self.cuda
            self.hdr = [torch.empty(self.world, 4, dtype=torch.int32, pin_memory=pin) for _ in range(depth)]
            self.land = [[torch.empty(self.cap, dtype=torch.int32, pin_memory=pin) for _ in range(self.world)]
                         for _ in range(depth)] if to_host else None
            self.slot_free = [threading.Event() for _ in range(depth)]
            for e in self.slot_free:
                e.set()
            self.q = queue.Queue()
            self.err = None
            self.thread = threading.Thread(target=self._consume, daemon=True)
            self.thread.start()

    # ------------------------------------------------------------------------------------------------ helpers
    def _stream(self):
        import contextlib
        return torch.cuda.stream(self.side) if self.cuda else contextlib.nullcontext()

    def _consume(self):
        try:
            while True:
                item = self.q.get()
                if item is None:
                    return
                step, slot, event, sizes = item
                if event is not None:
                    event.synchronize()
                for r, (nv, nf) in enumerate(sizes):
                    if nv == 0 and nf == 0:
                        continue
                    src = self.land[slot][r] if self.to_host else (self.send[slot] if r == 0 else self.recv[slot][r - 1])
                    v, f = _mesh_views(src, nv, nf)     # views into the ring slot: a sink that keeps them must copy
                    if self.sink is not None:
                        self.sink(step, r, v, f)
                    else:
                        self.results[(step, r)] = (v.clone(), f.clone())
                self.slot_free[slot].set()
        except Exception as e:      # surfaced by finish()
            self.err = e
            for ev in self.slot_free:
                ev.set()

    def _read_payloads(self, step, slot, hdr_event):
        """rank 0, one step later: sizes are on the host now; copy exactly the used words into the pinned ring."""
        if hdr_event is not None:
            hdr_event.synchronize()
        sizes = [(int(self.hdr[slot][r, 0]), int(self.hdr[slot][r, 1])) for r in range(self.world)]
        event = None
        if self.to_host and self.cuda:
            with self._stream():
                for r, (nv, nf) in enumerate(sizes):
                    n = 4 + 3 * nv + 3 * nf
                    src = self.send[slot] if r == 0 else self.recv[slot][r - 1]
                    self.land[slot][r][:n].copy_(src[:n], non_blocking=True)
                event = torch.cuda.Event()
                event.record(self.side)
                self._slot_done[slot] = event
        elif self.to_host:
            for r, (nv, nf) in enumerate(sizes):
                n = 4 + 3 * nv + 3 * nf
                self.land[slot][r][:n].copy_((self.send[slot] if r == 0 else self.recv[slot][r - 1])[:n])
        elif self.cuda:          # device-resident consumer: it must still see the transfers of this step completed
            event = torch.cuda.Event()
            event.record(self.side)
            self._slot_done[slot] = event
        self.q.put((step, slot, event, sizes))

    # ------------------------------------------------------------------------------------------------ API
    def submit(self, verts, faces):
        step, slot = self.step, self.step % self.depth
        self.step += 1
        if self.rank == 0:
            # the previous step's sizes are on the host by now (its messages left the peers a whole object ago):
            # queue its payload copies BEFORE this step's receives, so a late peer cannot hold them up
            while self.pending:
                self._read_payloads(*self.pending.pop(0))
            # the slot's previous occupant (step - depth) must have left the pinned ring
            self.slot_free[slot].wait()
            self.slot_free[slot].clear()
        # the mesh is copied into the ring slot on the CALLER's stream (a 150 MB device copy, ~50 us): its tensors are free
        # again at once -- tying them to the side stream (record_stream) kept their ~200 MB blocks out of the caching
        # allocator until the host copy had finished, and the next object's marching cubes paid a cudaMalloc (~100 ms)
        if self.cuda:
            if self._slot_done[slot] is not None:       # the slot's previous transfer / host copy must have left it
                torch.cuda.current_stream(self.device).wait_event(self._slot_done[slot])
        pack_mesh(self.send[slot], verts, faces, self.cap_v, self.cap_f)
        if self.cuda:
            self.side.wait_stream(torch.cuda.current_stream(self.device))
        with self._stream():
            if self.world > 1:
                if self.rank == 0:
                    works = dist.batch_isend_irecv([dist.P2POp(dist.irecv, self.recv[slot][r - 1], r)
                                                    for r in range(1, self.world)])
                else:
                    works = dist.batch_isend_irecv([dist.P2POp(dist.isend, self.send[slot], 0)])
                for w in works:
                    w.wait()          # NCCL: orders the side stream after the transfer; gloo: host wait
            if self.rank == 0:
                self.hdr[slot][0].copy_(self.send[slot][:4], non_blocking=True)
                for r in range(1, self.world):
                    self.hdr[slot][r].copy_(self.recv[slot][r - 1][:4], non_blocking=True)
                ev = None
                if self.cuda:
                    ev = torch.cuda.Event()
                    ev.record(self.side)
                self.pending.append((step, slot, ev))     # its payloads are read at the next submit() / finish()
            elif self.cuda:
                self._slot_done[slot] = torch.cuda.Event()
                self._slot_done[slot].record(self.side)   # the send has left this slot

    def finish(self):
        """Drain.  Returns, on rank 0, [(verts, faces)] ordered by (rank, step); [] elsewhere."""
        if self.rank != 0:
            if self.cuda:
                self.side.synchronize()
            return []
        while self.pending:
            self._read_payloads(*self.pending.pop(0))
        self.q.put(None)
        self.thread.join()
        if self.err is not None:
            raise self.err
        if self.cuda:
            self.side.synchronize()
        return [self.results[k] for k in sorted(self.results, key=lambda k: (k[1], k[0]))]
