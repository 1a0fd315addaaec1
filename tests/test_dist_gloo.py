"""CPU, world_size 2 over gloo: the N > 1 path's host logic (object sharding + fixed-capacity mesh gather)."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _mesh(i):
    """Mesh i: i+1 vertices and 2i+1 faces with recognisable content."""
    g = torch.Generator().manual_seed(i)
    return torch.rand(i + 1, 3, generator=g), torch.randint(0, i + 1, (2 * i + 1, 3), generator=g, dtype=torch.int32)


def _np(meshes):
    # plain numpy through the queue: torch tensors travel as shared-memory file descriptors that the parent has to
    # fetch from the worker, which may already have exited (ConnectionResetError in a slow parent)
    return [(v.numpy().copy(), f.numpy().copy()) for v, f in meshes]


def _assert_meshes(got, ids):
    """got: [(verts, faces)] numpy arrays; they must be meshes `ids`, in that order, bit for bit."""
    assert len(got) == len(ids)
    for (v, f), i in zip(got, ids):
        ev, ef = _mesh(i)
        assert v.dtype == np.float32 and f.dtype == np.int32 and v.shape == ev.shape and f.shape == ef.shape
        assert v.tobytes() == ev.numpy().tobytes() and f.tobytes() == ef.numpy().tobytes()


def _shard_and_gather(rank, world):
    """Seven objects sharded round-robin; both gatherers with ragged capacities and a None object on rank 1."""
    from r3g.dist import MeshBatchGatherer, MeshStreamGatherer, shard_indices
    mine = shard_indices(7)
    meshes = [_mesh(i) for i in mine]
    # streaming gather: one fixed-capacity message per rank and step, ring of depth 2
    sg = MeshStreamGatherer(cap_vertices=8 + 8 * rank, cap_faces=32 - 8 * rank, device="cpu")   # ranks agree on the max
    for step in range(4):
        sg.submit(*(meshes[step] if step < len(meshes) else (None, None)))
    streamed = sg.finish()
    # batch gather: staging buffer per rank, one message per peer at the end, pinned-ring landing
    bg = MeshBatchGatherer(cap_vertices=8 + 8 * rank, cap_faces=32 - 8 * rank, steps=4, device="cpu")
    for step in range(4):
        bg.submit(*(meshes[step] if step < len(meshes) else (None, None)))
    landed = []
    bufs = bg.finish(to_host=True, sink=lambda k, r, v, f: landed.append((r, k, v.clone(), f.clone())))
    return mine, _np(streamed), len(bufs), [(r, k) for r, k, _, _ in landed], _np((v, f) for _, _, v, f in landed)


def _batch(rank, world, objects, steps):
    """Rank r gathers meshes objects[r] with steps[r] and capacities sized from its own meshes, as the stage-3 twin
    does."""
    from r3g.dist import MeshBatchGatherer
    meshes = [_mesh(i) for i in objects[rank]]
    bg = MeshBatchGatherer(max((v.shape[0] for v, _ in meshes), default=0),
                           max((f.shape[0] for _, f in meshes), default=0), steps[rank], "cpu", to_host=True)
    for v, f in meshes:
        bg.submit(v, f)
    landed = []
    bufs = bg.finish(to_host=True, sink=lambda k, r, v, f: landed.append((r, k, v.clone(), f.clone())))
    return len(bufs), [(r, k) for r, k, _, _ in landed], _np((v, f) for _, _, v, f in landed)


def _worker(rank, world, port, q, job, args):
    sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    q.put((rank, job(rank, world, *args)))
    dist.barrier()
    dist.destroy_process_group()


def _run_world2(job, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, job, args)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=120) for _ in range(2))
    except Exception:
        res = None
    for p in procs:
        p.join(timeout=120)
        if p.is_alive():
            p.terminate()
            p.join()
    return [res[0], res[1]] if res is not None and all(p.exitcode == 0 for p in procs) else None


def _world2(job, *args):
    # the TCP rendezvous on a just-released port can be reset on a loaded box: one retry on a fresh port
    res = _run_world2(job, *args) or _run_world2(job, *args)
    assert res is not None, "world-size-2 gloo run failed twice"
    return res


def test_shard_and_fixed_capacity_gather_world2():
    r0, r1 = _world2(_shard_and_gather)
    assert r0[0] == [0, 2, 4, 6] and r1[0] == [1, 3, 5]
    order = [0, 2, 4, 6, 1, 3, 5]  # (rank, local index)
    _, streamed, n_bufs, where, landed = r0
    _assert_meshes(streamed, order)
    assert n_bufs == 2 and where == [(0, 0), (0, 1), (0, 2), (0, 3), (1, 0), (1, 1), (1, 2)]
    _assert_meshes(landed, order)
    assert r1[1:] == ([], 0, [], [])


# (objects[r], steps[r]): the meshes rank r gathers and the steps it passes; uneven counts are what shard_indices
# gives when the objects do not divide evenly over the ranks
BATCH_CASES = {
    "same_steps_rank1_sends_more": ([[0, 2], [1, 3, 5, 7, 9]], [5, 5]),
    "different_steps": ([[0, 2], [1, 3, 5, 7, 9]], [2, 5]),
    "rank1_sends_nothing": ([[0, 2, 4, 6], []], [4, 0]),
    "nothing_at_all": ([[], []], [0, 0]),
}


@pytest.mark.parametrize("case", sorted(BATCH_CASES))
def test_batch_gather_uneven_world2(case):
    """Every mesh of every rank reaches rank 0 bit for bit, in (rank, local index) order, whatever each rank submits."""
    objects, steps = BATCH_CASES[case]
    r0, r1 = _world2(_batch, objects, steps)
    n_bufs, where, landed = r0
    assert n_bufs == 2 and where == [(r, k) for r in range(2) for k in range(len(objects[r]))]
    _assert_meshes(landed, objects[0] + objects[1])
    assert r1 == (0, [], [])


def test_stream_gatherer_single_process():
    sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
    from r3g.dist import MeshStreamGatherer
    seen = []
    sg = MeshStreamGatherer(8, 8, device="cpu", sink=lambda step, r, v, f: seen.append((step, r, v.shape[0], f.shape[0])))
    for i in range(5):
        sg.submit(torch.rand(i + 1, 3), torch.zeros(i, 3, dtype=torch.int32))
    assert sg.finish() == [] and seen == [(i, 0, i + 1, i) for i in range(5)]
    with pytest.raises(ValueError):
        MeshStreamGatherer(2, 2, device="cpu").submit(torch.rand(3, 3), torch.zeros(1, 3, dtype=torch.int32))


def test_batch_gatherer_single_process():
    """Without a process group the batch gatherer is a world of one: rank 0's own buffer, its meshes landed in order."""
    sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
    from r3g.dist import MeshBatchGatherer, shard_indices
    assert shard_indices(5, 1, 3) == [1, 4]
    bg = MeshBatchGatherer(4, 8, 3, "cpu")
    for m in (_mesh(3), (None, None), _mesh(1)):
        bg.submit(*m)
    landed = []
    bufs = bg.finish(to_host=True, sink=lambda k, r, v, f: landed.append((r, k, v.clone(), f.clone())))
    assert len(bufs) == 1 and bufs[0] is bg.stage
    assert [(r, k) for r, k, _, _ in landed] == [(0, 0), (0, 2)]
    _assert_meshes(_np((v, f) for _, _, v, f in landed), [3, 1])


def test_shard_indices_partition_property():
    """Every object index is owned by exactly one rank, in increasing order per rank, for any (n, world)."""
    sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
    from hypothesis import given, settings, strategies as st
    from r3g.dist import shard_indices

    @settings(max_examples=200, deadline=None)
    @given(st.integers(0, 200), st.integers(1, 16))
    def check(n, world):
        seen = []
        for r in range(world):
            mine = shard_indices(n, r, world)
            assert mine == sorted(mine) and all(i % world == r for i in mine)
            seen += mine
        assert sorted(seen) == list(range(n))
    check()
