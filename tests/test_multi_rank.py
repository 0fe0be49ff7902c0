"""world_size-2 gloo test of the N>1 host logic (sharding + count/payload all-gather + compaction).
Per-rank conversion is done by the oracle here (CPU box, no GPU); on the GPU box the same
plan_shards / all_gather_records code runs over NCCL in bench.py --gpus N."""
from __future__ import annotations

import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank: int, world: int, port: int, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist

    import oracle
    from mesh2splat_b200 import _abi, synth
    from mesh2splat_b200.shard import all_gather_records, estimate_cost, plan_shards

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        tri = synth.displaced_sphere(24, 12, seed=2)
        s = _abi.Scene(tri, [_abi.Primitive(0, len(tri), (1, 1, 1, 1), 0, -1, -1)], [synth.random_texture(32, 32, 1)])
        s.compute_bboxes()
        R, layout = 64, _abi.LAYOUT_PACKED56
        cost = estimate_cost(s.triangles, s.primitives[0].bbox_min, s.primitives[0].bbox_max, R)
        shards = plan_shards(s.triangle_count, world, cost)
        first, count = shards[rank]
        rec, keys, total = oracle.convert(s, R, layout, first_triangle=first, triangle_count=max(count, 0) or 0) \
            if count else (np.zeros(0, _abi.record_dtype(layout)), np.zeros(0, np.uint64), 0)
        local = torch.from_numpy(np.frombuffer(rec.tobytes(), np.uint8).copy())
        buf, counts = all_gather_records(local, len(rec), _abi.STRIDES[layout], dist, torch)
        whole, wkeys, wtotal = oracle.convert(s, R, layout)
        got = buf.numpy().view(_abi.record_dtype(layout))
        # rank-major concatenation of contiguous triangle ranges == the single-process output order
        ok = (sum(counts) == wtotal == len(got)) and got.tobytes() == whole.tobytes()
        q.put((rank, ok, counts, shards))
    finally:
        dist.destroy_process_group()


def test_two_rank_shard_and_gather_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ok, counts, shards in res:
        assert ok, f"rank {rank}: gathered buffer differs from the single-process result"
        assert len(counts) == 2 and all(c > 0 for c in counts)
        assert shards[0][0] == 0 and shards[0][0] + shards[0][1] == shards[1][0]


def test_plan_shards_properties():
    sys.path.insert(0, ROOT)
    from mesh2splat_b200.shard import plan_shards
    for T in (0, 1, 7, 1000, 70074):
        for w in (1, 2, 3, 8):
            sh = plan_shards(T, w)
            assert len(sh) == w and sh[0][0] == 0 and sum(c for _, c in sh) == T
            assert all(sh[i][0] + sh[i][1] == sh[i + 1][0] for i in range(w - 1))
            assert max(c for _, c in sh) - min(c for _, c in sh) <= 1
    cost = np.ones(100); cost[:10] = 10.0   # the first 10 triangles carry about half of the work
    sh = plan_shards(100, 2, cost)
    assert 8 <= sh[0][1] <= 12 and sh[0][1] + sh[1][1] == 100
    with pytest.raises(ValueError):
        plan_shards(10, 0)


def _assert_partition(sh, T, w):
    """The non-empty ranges are contiguous in rank order, come first and partition [0, T); every empty range is
    (T, 0), the only (first, count) m2s_params reads as no triangles (a count of 0 means "to the end")."""
    assert len(sh) == w and sum(c for _, c in sh) == T
    full = [r for r in sh if r[1] > 0]
    assert sh[len(full):] == [(T, 0)] * (w - len(full)), sh
    if full:
        assert full[0][0] == 0 and full[-1][0] + full[-1][1] == T
        assert all(full[i][0] + full[i][1] == full[i + 1][0] for i in range(len(full) - 1)), sh


def test_plan_shards_empty_ranges():
    """Fewer triangles than ranks, or one triangle heavier than a rank's share, leave ranks without triangles: they
    get (T, 0), after the ranks that have triangles, and the oracle converts no record for them."""
    sys.path.insert(0, ROOT)
    import oracle
    from mesh2splat_b200 import synth
    from mesh2splat_b200.shard import estimate_cost, plan_shards, plan_work
    for T in (0, 1, 2, 3, 7, 1000):
        for w in (1, 2, 3, 8):
            sh = plan_shards(T, w)
            _assert_partition(sh, T, w)
            assert sum(c == 0 for _, c in sh) == max(0, w - T)
    heavy = np.ones(5); heavy[2] = 1000.0   # one triangle outweighs every other
    for w in (2, 4, 8):
        sh = plan_shards(5, w, heavy)
        _assert_partition(sh, 5, w)
        assert (w > 2) == any(c == 0 for _, c in sh), sh
    assert plan_shards(3, 8) == [(0, 1), (1, 1), (2, 1)] + [(3, 0)] * 5
    assert plan_shards(2, 3) == [(0, 1), (1, 1), (2, 0)]
    # plan_work without a cost, or with one when there are fewer rows than ranks, hands out triangle ranges
    assert plan_work(2, 4, 512, None) == [(0, 1, 0, 0), (1, 1, 0, 0), (2, 0, 0, 0), (2, 0, 0, 0)]
    q = synth.unit_quad()
    plan = plan_work(q.triangle_count, 4, 2, estimate_cost(q.triangles, q.primitives[0].bbox_min, q.primitives[0].bbox_max, 2))
    assert plan == [(0, 1, 0, 0), (1, 1, 0, 0), (2, 0, 0, 0), (2, 0, 0, 0)]
    # the oracle reads the range as m2s_params does: an empty range converts 0 records, the others their triangles
    for R, ranges in ((2, [p[:2] for p in plan]), (64, plan_shards(2, 3)), (64, plan_shards(2, 8))):
        totals = [oracle.convert(q, R, first_triangle=a, triangle_count=n)[2] for a, n in ranges]
        assert all((t == 0) == (n == 0) for t, (_, n) in zip(totals, ranges)), (ranges, totals)
        assert sum(totals) == oracle.convert(q, R)[2] == R * R


def test_plan_work_switches_to_row_bands_for_huge_triangles():
    """A 2-triangle quad cannot be balanced by triangle ranges: plan_work hands every rank all triangles and a
    band of pixel rows; the bands partition the grid and the per-band oracle outputs add up to the whole."""
    sys.path.insert(0, ROOT)
    import oracle
    from mesh2splat_b200 import _abi, synth
    from mesh2splat_b200.shard import estimate_cost, plan_work
    s = synth.unit_quad()
    R = 100
    cost = estimate_cost(s.triangles, s.primitives[0].bbox_min, s.primitives[0].bbox_max, R)
    assert plan_work(s.triangle_count, 2, R, cost) == [(0, 1, 0, 0), (1, 1, 0, 0)]  # two equal triangles, two ranks: ranges do
    for world in (3, 8):
        plan = plan_work(s.triangle_count, world, R, cost)
        assert all(p[0] == 0 and p[1] == s.triangle_count for p in plan)
        assert plan[0][2] == 0 and plan[-1][3] == R and all(plan[i][3] == plan[i + 1][2] for i in range(world - 1))
        keys = []
        for first, count, r0, r1 in plan:
            rec, k, total = oracle.convert(s, R, _abi.LAYOUT_PACKED56, first_triangle=first, triangle_count=count,
                                           row_begin=r0, row_end=r1)
            rows = (k >> np.uint64(12)) & np.uint64(0xFFF)
            assert total == len(k) == (r1 - r0) * R and rows.min() >= r0 and rows.max() < r1
            keys.append(k)
        whole, wk, wtotal = oracle.convert(s, R, _abi.LAYOUT_PACKED56)
        assert np.array_equal(np.sort(np.concatenate(keys)), np.sort(wk))
    # a mesh of many similar triangles keeps contiguous triangle ranges (whole grid: rows 0, 0)
    tri = synth.displaced_sphere(24, 12, seed=2)
    sp = _abi.Scene(tri, [_abi.Primitive(0, len(tri), (1, 1, 1, 1), -1, -1, -1)], [])
    sp.compute_bboxes()
    c2 = estimate_cost(sp.triangles, sp.primitives[0].bbox_min, sp.primitives[0].bbox_max, 64)
    plan = plan_work(sp.triangle_count, 4, 64, c2)
    assert all(p[2] == 0 and p[3] == 0 for p in plan) and sum(p[1] for p in plan) == sp.triangle_count


def test_choose_strategy_on_the_measured_configs():
    # step times and record counts of configs 2 and 4 as single-GPU inputs of the cost model
    sys.path.insert(0, ROOT)
    from mesh2splat_b200.shard import choose_strategy
    for g in (2, 4, 8):
        assert choose_strategy(39.9, 643438, 56, g) == "replicate"      # config 2: the gather alone outlasts the conversion
        assert choose_strategy(122.7, 169183, 56, g) == "shard"         # config 4: 1 M triangles, 9.5 MB of records
    assert choose_strategy(122.7, 169183, 56, 1) == "replicate"
