"""Multi-GPU host logic: triangle sharding and concatenation of per-rank gaussian buffers.

The reference has one atomic counter as its only shared state (converterFS.glsl:34,46); every
triangle is independent given the per-primitive constants.  So the triangle list is cut into one
contiguous range per rank (m2s_params.first_triangle / triangle_count), every rank converts its
range on its own GPU, and the per-rank buffers are concatenated on every rank:

    counts   all_gather of one int64 per rank  -> exclusive scan = global offsets
    payload  all_gather of max-count-padded buffers, then compaction to offsets (rank-major order)

Works with any torch.distributed backend: NCCL on GPUs, gloo in the CPU tests.

PeerGather is the NVLink-native form of the same step: the final buffer of every rank lives in
symmetric (peer-mapped) memory and each rank's fragment kernel stores its records straight into all
of them over NVLink at its rank-major offset (m2s_convert_gather_enqueue) — no collective call, no
host round trip on the data path.
"""
from __future__ import annotations

import numpy as np


def plan_shards(triangle_count: int, world: int, cost: np.ndarray | None = None) -> list:
    """Contiguous (first, count) per rank.  With `cost` (per-triangle estimated work, e.g. bbox pixel
    area) the cuts balance cumulative cost; otherwise triangle counts.  The non-empty ranges go to the first ranks,
    in triangle order.  The ranks left without triangles (fewer triangles than ranks, or one heavy triangle) come
    last, each with (triangle_count, 0): m2s_params reads a count of 0 as "to the end", so that is the only range it
    converts as empty, and it keeps every range starting where the previous one ends."""
    if world < 1:
        raise ValueError("world must be >= 1")
    if cost is None or triangle_count == 0:
        cuts = [(triangle_count * r) // world for r in range(world + 1)]
    else:
        c = np.asarray(cost, np.float64)
        if len(c) != triangle_count:
            raise ValueError("cost must have one entry per triangle")
        cum = np.concatenate([[0.0], np.cumsum(np.maximum(c, 0.0) + 1e-9)])
        targets = cum[-1] * np.arange(world + 1) / world
        cuts = np.searchsorted(cum, targets, side="left").astype(np.int64)
        cuts[0], cuts[-1] = 0, triangle_count
        cuts = np.maximum.accumulate(np.clip(cuts, 0, triangle_count)).tolist()
    ranges = [(int(cuts[r]), int(cuts[r + 1] - cuts[r])) for r in range(world) if cuts[r + 1] > cuts[r]]
    return ranges + [(int(triangle_count), 0)] * (world - len(ranges))


def plan_work(triangle_count: int, world: int, resolution: int, cost: np.ndarray | None = None) -> list:
    """Per-rank work item (first_triangle, triangle_count, row_begin, row_end) for m2s_params.

    Normally contiguous triangle ranges balanced by `cost` (plan_shards).  When a few huge triangles dominate
    — no cut of the triangle list can balance it, e.g. a 2-triangle quad on 8 GPUs — every rank takes ALL
    triangles but only a band of pixel rows of the R x R grid (SURVEY 8e: "split very large triangles by
    pixel-row bands"); the per-triangle set-up is then replicated, which is cheap exactly when triangles are few."""
    ranges = plan_shards(triangle_count, world, cost)
    if world > 1 and cost is not None and triangle_count > 0:
        c = np.maximum(np.asarray(cost, np.float64), 0.0)
        cum = np.concatenate([[0.0], np.cumsum(c)])
        worst = max(cum[a + n] - cum[a] for a, n in ranges)
        if worst > 1.25 * cum[-1] / world and resolution >= world:  # triangle ranges cannot balance this scene
            rows = [(resolution * r) // world for r in range(world + 1)]
            return [(0, triangle_count, rows[r], rows[r + 1]) for r in range(world)]
    return [(a, n, 0, 0) for a, n in ranges]


def choose_strategy(t_single_us: float, n_records: int, stride: int, world: int, fixed_us: float = 35.0,
                    nvlink_gb_s: float = 450.0) -> str:
    """"shard" or "replicate" for a conversion whose result every rank must hold.

    Sharding costs t_single/world of compute, the fixed multi-GPU overhead (count exchange, done flags, rank skew:
    ~35 us, an estimate not measured on H100 nodes; NVLink 4 per direction from the H100 SXM data sheet) and at least (world-1)/world * n_records * stride bytes of NVLink ingress per GPU; replicating
    costs t_single and no traffic.  Output-heavy scenes (BASELINE config 2: 36 MB of records) replicate;
    triangle-heavy ones (config 4: 9.5 MB from a longer conversion) shard."""
    if world <= 1:
        return "replicate"
    ingress_us = (world - 1) / world * n_records * stride / (nvlink_gb_s * 1e3)
    return "shard" if t_single_us / world + fixed_us + ingress_us < t_single_us else "replicate"


def estimate_cost(triangles: np.ndarray, bbox_min, bbox_max, resolution: int) -> np.ndarray:
    """Per-triangle candidate-pixel estimate: area of the dominant-axis projection's bounding box on
    the R x R grid (+1 for the fixed per-triangle set-up)."""
    t = np.asarray(triangles, np.float32).reshape(-1, 3, 12)[:, :, :3]
    e1, e2 = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
    n = np.abs(np.cross(e1, e2))
    axis = np.where((n[:, 0] > n[:, 1]) & (n[:, 0] > n[:, 2]), 0, np.where(n[:, 1] > n[:, 2], 1, 2))
    ext = t.max(axis=1) - t.min(axis=1)
    rng = np.asarray(bbox_max, np.float32) - np.asarray(bbox_min, np.float32)
    ia = np.where(axis == 0, 1, 0)
    ib = np.where(axis == 2, 1, 2)
    idx = np.arange(len(t))
    r = np.maximum(rng[ia], rng[ib])
    r = np.where(r > 0, r, 1.0)
    w = ext[idx, ia] / r * resolution + 1.0
    h = ext[idx, ib] / r * resolution + 1.0
    return (w * h + 1.0).astype(np.float64)


def all_gather_records(local, n_local: int, stride: int, dist, torch, out=None):
    """Concatenate per-rank record buffers on every rank.

    local: 1-D uint8 tensor holding at least n_local*stride bytes (this rank's gaussians).
    Returns (buffer, counts): `buffer` holds sum(counts)*stride bytes, rank-major; counts is a list."""
    world = dist.get_world_size()
    dev = local.device
    cnt = torch.tensor([n_local], dtype=torch.int64, device=dev)
    counts = torch.zeros(world, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(counts, cnt)
    c = [int(x) for x in counts.cpu().tolist()]
    mx = max(c) if c else 0
    total = sum(c)
    if out is None:
        out = torch.empty(max(1, total) * stride, dtype=torch.uint8, device=dev)
    if mx == 0:
        return out[:0], c
    padded = torch.zeros(mx * stride, dtype=torch.uint8, device=dev)
    padded[: n_local * stride] = local[: n_local * stride]
    gathered = torch.empty(world * mx * stride, dtype=torch.uint8, device=dev)
    dist.all_gather_into_tensor(gathered, padded)
    off = 0
    for r in range(world):
        out[off * stride:(off + c[r]) * stride] = gathered[r * mx * stride: r * mx * stride + c[r] * stride]
        off += c[r]
    return out[: total * stride], c


class PeerGather:
    """Final buffers + exchange blocks in torch symmetric memory, wired to m2s_convert_gather_enqueue.

    Every rank constructs one (collectively), then calls convert() the same number of times."""

    def __init__(self, ctx, capacity: int, stride: int, dist, torch):
        import ctypes as C

        import torch.distributed._symmetric_memory as symm

        from . import _abi
        self.ctx, self.capacity, self.stride, self.torch = ctx, int(capacity), int(stride), torch
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        if self.world > _abi.MAX_PEERS:
            raise ValueError("PeerGather supports up to 8 ranks (one NVSwitch domain)")
        dev = torch.device("cuda", ctx.device)
        group = dist.group.WORLD
        self.final = symm.empty(max(1, self.capacity) * self.stride, dtype=torch.uint8, device=dev)
        self.xch = symm.empty(_abi.MAX_PEERS * 4, dtype=torch.int64, device=dev)
        self.xch.zero_()
        self.total = torch.zeros(1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize(dev)
        try:
            hf = symm.rendezvous(self.final, group)
            hx = symm.rendezvous(self.xch, group)
        except TypeError:  # older signature: group name
            hf = symm.rendezvous(self.final, group.group_name)
            hx = symm.rendezvous(self.xch, group.group_name)
        self._handles = (hf, hx)
        dist.barrier()  # every rank has zeroed its exchange block before anyone signals into it
        self.peers = _abi.m2s_peers()
        self.peers.world, self.peers.rank = self.world, self.rank
        for r in range(self.world):
            self.peers.out[r] = int(hf.buffer_ptrs[r])
            self.peers.xch[r] = int(hx.buffer_ptrs[r])
        self._C = C

    def convert_enqueue(self, dscene, params, stream: int = 0) -> None:
        from ._lib import check, lib
        C = self._C
        check(lib().m2s_convert_gather_enqueue(self.ctx.handle, dscene.handle, C.byref(params), C.byref(self.peers),
                                               self.capacity, self.total.data_ptr(), stream or None))

    def barrier(self) -> None:
        """Device-side barrier across the ranks on the current torch stream (symmetric-memory signal pads)."""
        self._handles[1].barrier()

    def records(self, layout: int):
        """(structured numpy view of the gathered records, count) — synchronises."""
        from . import _abi
        self.torch.cuda.synchronize(self.final.device)  # the kernels may have run on the context's own stream
        n = int(self.total.item())
        n = min(n, self.capacity)
        raw = self.final[: n * self.stride].cpu().numpy()
        return raw.view(_abi.record_dtype(layout)), n
