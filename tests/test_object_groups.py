"""CPU: object groups (r3g/dist.py) -- the plan every rank derives, and the exchange / broadcast / slice-gather helpers
on gloo at world size 2 and 4."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))


def test_plan_assigns_every_object_once():
    from hypothesis import given, settings, strategies as st
    from r3g.dist import plan_object_groups, shard_indices

    @settings(max_examples=300, deadline=None)
    @given(st.integers(0, 100), st.integers(1, 16))
    def check(K, W):
        plan = plan_object_groups(K, W)
        assert plan == plan_object_groups(K, W)                     # a pure function of (K, W): every rank agrees
        assert [i for i, _ in plan.assignments] == list(range(K))    # each object exactly once, in order
        tail = K % W
        for i, ranks in plan.assignments:
            assert list(ranks) == sorted(ranks) and all(0 <= r < W for r in ranks)
            if i < K - tail:                                         # full waves: shard_indices' assignment
                assert ranks == (i % W,) and i in shard_indices(K, i % W, W)
            else:
                assert len(ranks) == W // tail
        tail_groups = [set(r) for i, r in plan.assignments if i >= K - tail]
        assert sum(len(g) for g in tail_groups) == len(set().union(*tail_groups))    # the tail wave's groups are disjoint
        # what each rank runs: its full-wave objects, then the tail group it belongs to, if any
        for r in range(W):
            mine = plan.for_rank(r)
            assert [i for i, _ in mine if i < K - tail] == [i for i in shard_indices(K, r, W) if i < K - tail]
            assert len([1 for i, _ in mine if i >= K - tail]) <= 1
    check()


def test_plan_examples():
    from r3g.dist import plan_object_groups
    assert plan_object_groups(3, 2).assignments == ((0, (0,)), (1, (1,)), (2, (0, 1)))
    assert plan_object_groups(1, 8).assignments == ((0, tuple(range(8))),)
    assert plan_object_groups(9, 8).assignments[-1] == (8, tuple(range(8)))
    assert plan_object_groups(6, 4).groups() == [(0, 1), (2, 3)]
    assert plan_object_groups(7, 4).groups() == []            # 3 tail objects on 4 ranks: groups of one
    assert plan_object_groups(5, 1).groups() == []
    with pytest.raises(ValueError):
        plan_object_groups(3, 0)


def test_chunk_ranges_balanced_and_contiguous():
    from r3g.dist import chunk_ranges
    for n in range(0, 40):
        for G in range(1, 9):
            rs = chunk_ranges(n, G)
            assert rs[0][0] == 0 and rs[-1][1] == n and all(a[1] == b[0] for a, b in zip(rs, rs[1:]))
            sizes = [c1 - c0 for c0, c1 in rs]
            assert max(sizes) - min(sizes) <= 1


def test_chunk_span_is_the_single_gpu_chunking():
    from r3g.vae import CrossAttentionDecoder
    geo = CrossAttentionDecoder(1024, 16, device="cpu")
    assert geo.grid_chunks(256) == (65536, 260)
    assert geo.chunk_span(256) == (0, 257 ** 3) and geo.chunk_span(256, (259, 260)) == (259 * 65536, 257 ** 3)
    assert geo.chunk_span(100, (3, 3)) == (3 * 65536, 3 * 65536)
    assert geo.grid_chunks(20) == (21 ** 3, 1)
    with pytest.raises(ValueError):
        geo.chunk_span(256, (0, 261))


def test_graph_cache_retain_keeps_the_selected_keys():
    from r3g.graphs import GraphCache
    gc = GraphCache(keep_all=True)
    gc.entries = {(256, "b", None): 1, (256, "b", (0, 130)): 2, (128, "b", None): 3}
    gc.retain(lambda k: k[:2] == (256, "b"))
    assert gc.entries == {(256, "b", None): 1, (256, "b", (0, 130)): 2} and gc.captures == 0


# ------------------------------------------------------------------------------------------------ gloo, world 2 / 4
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _helpers(rank, world, K, n_chunks, cq, ragged):
    """Every tail group of plan_object_groups(K, world) runs the three helpers and the input check once."""
    from r3g.dist import (broadcast_from_leader, check_same_inputs, chunk_ranges, create_object_groups,
                          exchange_cfg_pair, gather_flat_slices, group_layout, plan_object_groups)
    plan = plan_object_groups(K, world)
    groups = create_object_groups(plan)
    out = {}
    for i, ranks in plan.for_rank(rank):
        if len(ranks) == 1:
            continue
        g = groups[ranks]
        m, rr = group_layout(g)
        assert rr == ranks
        G = len(rr)
        res = dict(member=m)
        if m < 2:
            v = torch.full((3, 4), float(10 * i + m))
            pair = torch.full((2, 3, 4), -1.0)
            exchange_cfg_pair(v, pair, g)
            res["pair"] = [pair[0].unique().tolist(), pair[1].unique().tolist()]
        x = torch.arange(6.0) + 100 * i if m < 2 else torch.zeros(6)
        broadcast_from_leader(x, g, skip_pair=True)
        res["bcast_pair"] = x.tolist()
        y = torch.arange(5.0) + i if m == 0 else torch.zeros(5)
        broadcast_from_leader(y, g)
        res["bcast"] = y.tolist()
        total = n_chunks * cq - ragged
        spans = [(min(c0 * cq, total), min(c1 * cq, total)) for c0, c1 in chunk_ranges(n_chunks, G)]
        res["spans"] = spans
        flat = torch.full((total,), -1.0)
        s0, s1 = spans[m]
        flat[s0:s1] = torch.arange(s0, s1, dtype=torch.float32) + 1000 * i
        gather_flat_slices(flat, spans, g)
        res["flat"] = flat.tolist() if m == 0 else None
        check_same_inputs(g, torch.ones(7, dtype=torch.float16), torch.arange(9.0))
        try:
            check_same_inputs(g, torch.full((7,), float(m == G - 1), dtype=torch.float16))
            res["raised"] = False
        except RuntimeError:
            res["raised"] = True
        out[i] = res
    return out


def _worker(rank, world, port, q, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        q.put((rank, _helpers(rank, world, *args)))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _run(world, *args):
    ctx = mp.get_context("spawn")
    for _ in range(2):       # one retry on a fresh port: a just-released port can be reset on a loaded box
        q, port = ctx.Queue(), _free_port()
        procs = [ctx.Process(target=_worker, args=(r, world, port, q, args)) for r in range(world)]
        for p in procs:
            p.start()
        try:
            res = dict(q.get(timeout=120) for _ in range(world))
        except Exception:
            res = None
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join()
        if res is not None and all(p.exitcode == 0 for p in procs):
            return res
    raise AssertionError(f"gloo world of {world} failed twice")


# (world, K, chunks, queries per chunk, missing queries of the last chunk): K mod world tail objects on groups of
# world // (K mod world) ranks
CASES = {
    "w2_one_group_uneven_chunks": (2, 3, 5, 4, 3),
    "w4_one_group_empty_member": (4, 1, 3, 4, 1),
    "w4_two_groups": (4, 6, 7, 3, 2),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_group_helpers_on_gloo(case):
    world, K, n_chunks, cq, ragged = CASES[case]
    from r3g.dist import plan_object_groups
    res = _run(world, K, n_chunks, cq, ragged)
    total = n_chunks * cq - ragged
    for i, ranks in plan_object_groups(K, world).assignments:
        if len(ranks) == 1:
            continue
        got = {res[r][i]["member"]: res[r][i] for r in ranks}
        assert sorted(got) == list(range(len(ranks)))
        for m, g in got.items():
            if m < 2:         # (cond, uncond) on both members of the pair
                assert g["pair"] == [[10.0 * i], [10.0 * i + 1]]
            assert g["bcast_pair"] == (torch.arange(6.0) + 100 * i).tolist()
            assert g["bcast"] == (torch.arange(5.0) + i).tolist()
            assert g["raised"]                                  # the last member's input differed: all of them raise
        assert got[0]["flat"] == (torch.arange(total, dtype=torch.float32) + 1000 * i).tolist()
        if case == "w4_one_group_empty_member":
            assert got[0]["spans"][0] == (0, 0)                 # the leader decodes nothing and still receives
