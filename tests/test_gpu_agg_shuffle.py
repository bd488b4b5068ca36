"""GPU: HashAgg behind the hash shuffle -- rwgpu_agg_push_device_counted (the row count read on the device, the chunk's
buffers being its capacity), the one-kernel flat exchange feeding it, and Nexmark q4's second exchange (the inner
HashAgg's delta regrouped by `category` across ranks).

Every comparison is a multiset: the device emits a barrier's rows in dirty-list order."""
from collections import Counter

import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import AggCall, HashAggExecutor, MockSource
from risingwave_b200.stream_chunk import Column, StreamChunk, net_multiset, pack_bits, unpack_bits

from helpers import load_golden
from test_gpu_shuffle import _flat_setup

pytestmark = pytest.mark.gpu

I, I4 = abi.T_INT64, abi.T_INT32
NP = {I: np.int64, I4: np.int32}
INT64_MAX, INT64_MIN = np.iinfo(np.int64).max, np.iinfo(np.int64).min


class Shape:
    """one plan shape of the aggregation and a generator of its input rows"""

    def __init__(self, name, types, keys, calls, append_only, nulls=False, vis=False, deletes=False):
        self.name, self.types, self.keys, self.calls, self.append_only = name, types, keys, calls, append_only
        self.nulls, self.vis, self.deletes = nulls, vis, deletes

    def __str__(self):
        return self.name

    def executor(self, be, hint=0):
        _, src = MockSource.channel()
        return HashAggExecutor(be, src.into_executor(self.types, []), self.append_only, [AggCall.from_pretty(c) for c in self.calls], 0,
                               self.keys, group_capacity_hint=hint)


SHAPES = [
    # agg_apply_fast_kernel: one int64 key; count(*), sum, max; no NULLs (bench.py's cfg2 shape)
    Shape("fast", [I, I], [0], ("(count:int8)", "(sum:int8 $1:int8)", "(max:int8 $1:int8)"), True),
    # agg_apply_kernel: two keys (int64, int32), NULL keys and arguments, a visibility bitmap, deletes
    Shape("generic", [I, I4, I, I], [0, 1], ("(count:int8)", "(count:int8 $2:int8)", "(sum:int8 $2:int8)", "(sum:int8 $3:int8)"), False,
          nulls=True, vis=True, deletes=True),
    # retractable min / max (materialized input, agg_mm_delete_kernel) with deletes
    Shape("retract", [I, I], [0], ("(count:int8)", "(min:int8 $1:int8)", "(max:int8 $1:int8)"), False, deletes=True),
]


class Source:
    """rows of one shape: the first `n` rows of a chunk are live input (inserts of new and existing groups, deletes of
    live rows), the rows past `n` look like live input too -- inserts into existing and new groups, extreme values --
    so that reading one of them changes the result"""

    def __init__(self, shape, seed, n_keys=300):
        self.s, self.rng, self.n_keys = shape, np.random.default_rng(seed), n_keys
        self.live = []  # (row values, validity) of inserted, not yet deleted rows

    def _row(self, extreme=False):
        s, rng = self.s, self.rng
        vals, valid = [], []
        for k, t in enumerate(s.types):
            if k in s.keys:
                v = int(rng.integers(0, self.n_keys if not extreme else 10 * self.n_keys))
            else:
                v = int(rng.choice([INT64_MAX // 4, INT64_MIN // 4])) if extreme else int(rng.integers(-1000, 1000))
            vals.append(v)
            valid.append(not (s.nulls and rng.random() < 0.15))
        return vals, valid

    def chunk(self, cap, n, zero_ops=0):
        """`zero_ops` rows of the prefix get op 0 (folded invisible, as the exchange expects them)"""
        s, rng = self.s, self.rng
        vis = rng.random(cap) < 0.9 if s.vis else None
        zero = set(rng.choice(n, zero_ops, replace=False).tolist()) if zero_ops else set()
        ops, rows = [], []
        for i in range(cap):
            applied = i < n and (vis is None or vis[i]) and i not in zero
            if applied and s.deletes and self.live and rng.random() < 0.3:
                r = self.live.pop(int(rng.integers(0, len(self.live))))
                ops.append(abi.OP_DELETE)
            else:
                r = self._row(extreme=i >= n and rng.random() < 0.5)
                ops.append(0 if i in zero else abi.OP_INSERT)
                if applied:
                    self.live.append(r)
            rows.append(r)
        cols = []
        for k, t in enumerate(s.types):
            data = np.array([r[0][k] for r in rows], dtype=NP[t])
            valid = np.array([r[1][k] for r in rows], dtype=bool) if s.nulls else None
            cols.append(Column(t, data, valid))
        return StreamChunk(np.array(ops, np.uint8), cols, vis)


def dev_chunk(ch):
    import torch
    from risingwave_b200 import device

    def bits(b):
        return None if b is None else torch.from_numpy(pack_bits(b).view(np.int64)).cuda()
    return device.DeviceChunk(torch.from_numpy(ch.ops.copy()).cuda(), [torch.from_numpy(c.data.copy()).cuda() for c in ch.columns], ch.types(),
                              [bits(c.valid) for c in ch.columns], bits(ch.vis))


def view_rows(view):
    """-> Counter of (op, row) of a DeviceView (None = NULL)"""
    import torch
    from risingwave_b200 import device
    n = view.n_rows
    if n == 0:
        return Counter()
    ops = view.ops().cpu().numpy()
    vis = view.visible()
    cols = []
    for k in range(view.n_cols):
        data = view.column(k).cpu().numpy()
        valid = None
        if view.valid_ptrs[k]:
            words = torch.empty((n + 63) // 64, dtype=torch.int64, device="cuda")
            device._d2d(words.data_ptr(), view.valid_ptrs[k], words.numel() * 8)
            torch.cuda.synchronize()
            valid = unpack_bits(words.cpu().numpy().view(np.uint64), n)
        cols.append(Column(view.col_types[k], data, valid))
    return Counter(StreamChunk(ops, cols, None if vis is None else vis.cpu().numpy()).rows())


def net(rows: Counter) -> Counter:
    c = Counter()
    for (op, row), m in rows.items():
        c[row] += m if op in (abi.OP_INSERT, abi.OP_UPDATE_INSERT) else -m
    return Counter({k: v for k, v in c.items() if v})


def snapshot_rows(ex):
    states, minput = ex.snapshot()
    return [sorted(map(repr, (r for ch in part for _, r in ch.rows()))) for part in (states, minput)]


def count_tensor(n):
    import torch
    return torch.tensor([n], dtype=torch.int64, device="cuda")


COUNTS = lambda cap: (0, 1, 37, cap - 1, cap)  # noqa: E731


# ------------------------------------------------------------------------------------------ 4. counted == plain on the prefix
@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_counted_push_equals_plain_push_of_the_prefix(cuda, oracle, shape):
    from risingwave_b200 import device
    cap = 1000
    src = Source(shape, seed=sum(map(ord, shape.name)))
    counted, plain, ref = shape.executor(cuda), shape.executor(cuda), shape.executor(oracle)
    for epoch in range(1, 4):
        keep = []  # buffers and counts stay unchanged until the pushes have run (the barrier waits for them)
        for n in COUNTS(cap):
            ch = src.chunk(cap, n)
            keep.append((count_tensor(n), dev_chunk(ch)))
            device.agg_push_device(counted, keep[-1][1], n_rows_dev=keep[-1][0].data_ptr())
            prefix = ch.slice(0, n)
            if n:
                keep.append(dev_chunk(prefix))
                device.agg_push_device(plain, keep[-1])
                ref.apply_chunk(prefix)
        got = view_rows(device.agg_flush_device(counted, epoch))
        want = view_rows(device.agg_flush_device(plain, epoch))
        assert got == want, f"epoch {epoch}"
        assert net(got) == net_multiset(ref.flush_data(epoch)), f"epoch {epoch}"
    assert snapshot_rows(counted) == snapshot_rows(plain)


# ------------------------------------------------------------------------------------------ 5. out-of-range counts
@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("bad", (-1, "cap+1"))
def test_count_out_of_range_is_reported_at_the_barrier(cuda, shape, bad):
    from risingwave_b200 import device
    cap = 500
    src = Source(shape, seed=7)
    counted, plain = shape.executor(cuda), shape.executor(cuda)
    good = dev_chunk(src.chunk(cap, cap))
    for ex in (counted, plain):
        device.agg_push_device(ex, good)
        device.agg_flush_device(ex, 1)
    cnt = count_tensor(cap + 1 if bad == "cap+1" else bad)
    bad_chunk = dev_chunk(src.chunk(cap, cap))
    device.agg_push_device(counted, bad_chunk, n_rows_dev=cnt.data_ptr())  # RW_OK: the count is not read here
    with pytest.raises(abi.RwError) as e:
        device.agg_flush_device(counted, 2)
    assert e.value.code == abi.RW_ERR_INVALID and "device row count out of range" in str(e.value)
    # the push applied nothing, and the operator goes on
    src.live.clear()
    nxt = dev_chunk(src.chunk(cap, cap))
    for ex in (counted, plain):
        device.agg_push_device(ex, nxt)
    assert view_rows(device.agg_flush_device(counted, 3)) == view_rows(device.agg_flush_device(plain, 3))
    assert snapshot_rows(counted) == snapshot_rows(plain)


# ------------------------------------------------------------------------------------------ 6. growth under counted pushes
@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_growth_under_counted_pushes(cuda, oracle, shape):
    """group_capacity_hint 0 (a 1024-slot table) and 3000-row capacities with many new groups: the table grows inside an
    epoch, and while two barriers are outstanding (launch / collect split)"""
    from risingwave_b200 import device
    cap = 3000
    src = Source(shape, seed=11, n_keys=40000)
    counted, ref = shape.executor(cuda, hint=0), shape.executor(oracle)
    epoch = 0
    keep = []  # the count tensors and chunks stay alive until their pushes have run
    for rnd in range(3):
        want = []
        for _ in range(2):  # two epochs enqueued, then both collected: growth happens with barriers outstanding
            epoch += 1
            for n in (cap, cap - 1, 1999):
                ch = src.chunk(cap, n)
                keep.append((count_tensor(n), dev_chunk(ch)))
                device.agg_push_device(counted, keep[-1][1], n_rows_dev=keep[-1][0].data_ptr())
                ref.apply_chunk(ch.slice(0, n))
            device.agg_flush_device_async(counted, epoch)
            want.append(net_multiset(ref.flush_data(epoch)))
        got = [net(view_rows(device.agg_flush_collect(counted))) for _ in range(2)]
        assert got == want, f"round {rnd}"
    _, capacity, _ = stats(counted)
    assert capacity > 1024


def stats(ex):
    import ctypes as C
    from risingwave_b200 import device
    a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
    device._check(device._lib().rwgpu_agg_stats(ex._h, C.byref(a), C.byref(b), C.byref(c)))
    return a.value, b.value, c.value


# ------------------------------------------------------------------------------------------ 7. no host sync in the steady state
SYNC_NAMES = ("cudaDeviceSynchronize", "cudaStreamSynchronize", "cudaEventSynchronize", "cudaMemcpy")


def calls_inside(prof, label):
    """names of the events that ran inside the `label` range (the profiler itself synchronises when the trace stops)"""
    evs = prof.events()
    win = next(e for e in evs if e.name == label).time_range
    return {e.name for e in evs if e.name != label and win.start <= e.time_range.start and e.time_range.end <= win.end}


def test_counted_pushes_never_wait_for_the_device(cuda):
    """with group_capacity_hint covering the groups plus the pushes' capacities, 8 counted pushes issue no synchronising
    call and no device-to-host copy; a push past the bound (growth) does -- the trace sees the library's calls"""
    import torch
    from torch.profiler import ProfilerActivity, profile, record_function
    from risingwave_b200 import device
    shape = SHAPES[0]
    cap, keys = 1 << 14, 4096
    ex = shape.executor(cuda, hint=keys + 10 * cap)
    rng = np.random.default_rng(5)
    chunks = []
    for _ in range(9):
        k = torch.from_numpy(rng.integers(0, keys, cap).astype(np.int64)).cuda()
        chunks.append(device.DeviceChunk(torch.ones(cap, dtype=torch.uint8, device="cuda"), [k, k * 3], [I, I]))
    cnt = count_tensor(cap - 3)
    stream = torch.cuda.Stream()
    device.agg_push_device(ex, chunks[0], stream, n_rows_dev=cnt.data_ptr())  # (module load outside the trace)
    device.agg_flush_device(ex, 1, stream)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        with record_function("counted_pushes"):
            for c in chunks[1:]:
                device.agg_push_device(ex, c, stream, n_rows_dev=cnt.data_ptr())
    names = {e.name for e in prof.events()}
    assert any("agg_apply_fast_kernel" in n for n in names), sorted(names)
    assert not [n for n in names if "DtoH" in n], sorted(names)
    inside = calls_inside(prof, "counted_pushes")
    assert "cudaLaunchKernel" in inside, sorted(inside)
    assert not [n for n in inside if any(s in n for s in SYNC_NAMES)], sorted(inside)
    device.agg_flush_device(ex, 2, stream)
    big = 1 << 20  # past the bound: agg_ensure_capacity reads the group count back
    kb = torch.zeros(big, dtype=torch.int64, device="cuda")
    big_chunk = device.DeviceChunk(torch.ones(big, dtype=torch.uint8, device="cuda"), [kb, kb], [I, I])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        with record_function("growth_push"):
            device.agg_push_device(ex, big_chunk, stream, n_rows_dev=cnt.data_ptr())
    assert "cudaDeviceSynchronize" in calls_inside(prof, "growth_push")
    device.agg_flush_device(ex, 3, stream)


# ------------------------------------------------------------------------------------------ 8. self-peer flat exchange
EX_SHAPES = [Shape("fast_retract", [I, I], [0], ("(count:int8)", "(sum:int8 $1:int8)"), False, deletes=True), SHAPES[2]]


def exchange_input(src, m):
    """a chunk of m rows, inserts and deletes, 40 of them folded invisible (op 0: the exchange drops them).
    -> (host chunk, mask of the rows the aggregation must see)"""
    ch = src.chunk(m, m, zero_ops=40)
    return ch, ch.ops != 0


@pytest.mark.parametrize("shape", EX_SHAPES, ids=str)
def test_flat_exchange_self_peer_feeds_counted_agg(cuda, oracle, shape):
    """world = 1 through rwgpu_shuffle_exchange_flat_device into the counted agg push, reading the receive buffer in
    place; the epochs shrink, so the rows of the previous, larger batch sit past the count"""
    import torch
    from risingwave_b200 import device, exchange
    src = Source(shape, seed=23, n_keys=2000)
    n = 20000
    bufs, flags, views = _flat_setup(1, shape.types, n)
    counts = torch.zeros(1, dtype=torch.int64, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    total_dev = torch.zeros(1, dtype=torch.int64, device="cuda")
    call = device.FlatExchangeCall([0], exchange.vnode_to_dest_table(1).cuda(), 1, 0, [bufs[0].data_ptr()], [flags[0].data_ptr()], n,
                                   counts, err, total_dev.data_ptr(), None)
    agg, ref = shape.executor(cuda), shape.executor(oracle)
    stream = torch.cuda.Stream()
    recv = device.DeviceChunk(views[0][0], views[0][1], shape.types)
    for epoch in (1, 2, 3):
        ch, keep = exchange_input(src, n - 1000 * epoch)
        dc = dev_chunk(ch)
        with torch.cuda.stream(stream):
            call(dc, epoch, stream)
            device.agg_push_device(agg, recv, stream, n_rows_dev=total_dev.data_ptr())
            got = net(view_rows(device.agg_flush_device(agg, epoch, stream)))
        assert int(err.item()) == 0 and int(total_dev.item()) == int(keep.sum())
        ref.apply_chunk(StreamChunk(ch.ops[keep], [Column(c.type, c.data[keep]) for c in ch.columns]))
        assert got == net_multiset(ref.flush_data(epoch)), f"epoch {epoch}"


# ------------------------------------------------------------------------------------------ 9. virtual ranks
def owner(oracle, keys, world):
    host = StreamChunk(np.ones(len(keys), np.uint8), [Column(I, np.asarray(keys, np.int64))])
    return oracle.vnode_compute(host, [0], 256).astype(np.int64) * world // 256


@pytest.mark.parametrize("shape", EX_SHAPES, ids=str)
@pytest.mark.parametrize("world", (2, 4))
def test_flat_exchange_virtual_ranks_feed_counted_aggs(cuda, oracle, shape, world):
    """W virtual ranks on one device (one stream each, exchange grids capped so the W kernels are co-resident): every
    rank's exchange of a batch is enqueued before any agg push of that batch -- a push may synchronise the device
    (growth), which would wait forever for an exchange kernel whose peers were not launched yet"""
    import torch
    from risingwave_b200 import device, exchange
    n = 9000
    cap = world * n
    bufs, flags, views = _flat_setup(world, shape.types, cap)
    v2d = exchange.vnode_to_dest_table(world).cuda()
    peers, flag_ptrs = [b.data_ptr() for b in bufs], [f.data_ptr() for f in flags]
    streams = [torch.cuda.Stream() for _ in range(world)]
    st = [dict(counts=torch.zeros(world, dtype=torch.int64, device="cuda"), err=torch.zeros(1, dtype=torch.int32, device="cuda"),
               total=torch.zeros(1, dtype=torch.int64, device="cuda")) for _ in range(world)]
    calls = [device.FlatExchangeCall([0], v2d, world, r, peers, flag_ptrs, cap, st[r]["counts"], st[r]["err"], st[r]["total"].data_ptr(),
                                     None, max_blocks=24) for r in range(world)]
    srcs = [Source(shape, seed=100 + r, n_keys=5000) for r in range(world)]
    aggs = [shape.executor(cuda, hint=5000) for _ in range(world)]
    ref = shape.executor(oracle)
    for epoch in (1, 2, 3):
        inputs = [exchange_input(srcs[r], n - 1500 * epoch) for r in range(world)]
        chunks = [dev_chunk(ch) for ch, _ in inputs]
        torch.cuda.synchronize()
        for r in range(world):
            calls[r](chunks[r], epoch, streams[r])
        for r in range(world):
            device.agg_push_device(aggs[r], device.DeviceChunk(views[r][0], views[r][1], shape.types), streams[r],
                                   n_rows_dev=st[r]["total"].data_ptr())
        deltas = [net(view_rows(device.agg_flush_device(aggs[r], epoch, streams[r]))) for r in range(world)]
        torch.cuda.synchronize()
        errs = [int(s["err"].item()) for s in st]
        if any(e & 2 for e in errs):
            pytest.skip("this device did not run the ranks' kernels side by side (barrier timed out)")
        assert errs == [0] * world
        for ch, keep in inputs:
            ref.apply_chunk(StreamChunk(ch.ops[keep], [Column(c.type, c.data[keep]) for c in ch.columns]))
        union = Counter()
        for r, d in enumerate(deltas):
            if d:
                assert set(owner(oracle, [row[0] for row in d], world).tolist()) == {r}, f"epoch {epoch}: a group off its owner rank"
            union.update(d)
        assert union == net_multiset(ref.flush_data(epoch)), f"epoch {epoch}"


# ------------------------------------------------------------------------------------------ 10. two real GPUs
def _two_gpu_agg_worker(rank, world, port, q):
    import os
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    try:
        from risingwave_b200 import device, exchange
        from risingwave_b200.executor import Backend
        shape = EX_SHAPES[1]
        n = 30000
        plan = exchange.FlatShufflePlan(world, rank, [0], shape.types, batch_rows=n)
        agg = shape.executor(Backend.cuda(), hint=20000)
        src = Source(shape, seed=300 + rank, n_keys=20000)
        stream = torch.cuda.current_stream()
        out = []
        for epoch in (1, 2, 3):
            ch, keep = exchange_input(src, n - 2000 * epoch)
            b = plan.start(dev_chunk(ch), stream)
            ops, cols = plan.output(b)
            device.agg_push_device(agg, device.DeviceChunk(ops, cols, shape.types), stream, n_rows_dev=plan.count_ptr(b))
            out.append(dict(net(view_rows(device.agg_flush_device(agg, epoch, stream)))))
            torch.cuda.synchronize()
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def test_flat_shuffle_plan_two_gpus_feeds_counted_aggs(cuda, oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world, port = 2, 29631
    procs = [ctx.Process(target=_two_gpu_agg_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
    shape = EX_SHAPES[1]
    srcs = [Source(shape, seed=300 + r, n_keys=20000) for r in range(world)]
    ref = shape.executor(oracle)
    for e, epoch in enumerate((1, 2, 3)):
        for r in range(world):
            ch, keep = exchange_input(srcs[r], 30000 - 2000 * epoch)
            ref.apply_chunk(StreamChunk(ch.ops[keep], [Column(c.type, c.data[keep]) for c in ch.columns]))
        union = Counter()
        for r in range(world):
            d = Counter(got[r][e])
            if d:
                assert set(owner(oracle, [row[0] for row in d], world).tolist()) == {r}
            union.update(d)
        assert union == net_multiset(ref.flush_data(epoch)), f"epoch {epoch}"


# ------------------------------------------------------------------------------------------ 11. Nexmark q4, second exchange
def send_delta(view, cols, batch_rows, send):
    """the inner HashAgg's barrier delta (one un-cut device chunk), projected by column pointers, in slices of at most
    `batch_rows` rows (at least one slice: every rank takes part in every exchange batch).  No U-/U+ rewrite: both rows
    of an inner-agg U-/U+ pair carry the same group key, so the same `category`, and go to the same rank together."""
    from risingwave_b200 import device
    n = view.n_rows
    lo = 0
    while True:
        hi = min(n, lo + batch_rows)
        send(device.ViewChunk(view, cols, lo, hi))
        lo = hi
        if lo >= n:
            return


@pytest.mark.parametrize("world", (2, 4))
def test_nexmark_q4_second_exchange_virtual_ranks(cuda, world):
    """q4 over W virtual ranks: auctions and bids sharded by the vnode of the join key; per rank join, filter, project and
    the inner HashAgg(max(price) GROUP BY id, category) on the CUDA backend; the inner delta of every rank goes through
    the flat exchange on `category` into the counted push of that category's owner's outer HashAgg(count, sum GROUP BY
    category).  The union of the outer deltas, applied to the MV, is the reference's expected q4 result."""
    import torch
    from decimal import Decimal
    from fractions import Fraction
    from risingwave_b200 import device, exchange
    from risingwave_b200.executor import FilterExecutor, HashJoinExecutor, JoinParams
    fx = load_golden("nexmark_q4_fixture.json")
    pred = "(and:boolean (greater_than_or_equal:boolean $2:int8 $5:int8) (less_than_or_equal:boolean $2:int8 $6:int8))"
    ranks = []
    for r in range(world):
        _, sl = MockSource.channel()
        _, sr = MockSource.channel()
        _, sf = MockSource.channel()
        _, s1 = MockSource.channel()
        _, s2 = MockSource.channel()
        ranks.append(dict(
            join=HashJoinExecutor(cuda, abi.JOIN_INNER, sl.into_executor([I] * 4, [3]), sr.into_executor([I] * 4, [0]),
                                  JoinParams([0], [3]), JoinParams([0], [0]), [False]),
            flt=FilterExecutor(cuda, sf.into_executor([I] * 8, []), pred),
            agg1=HashAggExecutor(cuda, s1.into_executor([I] * 3, []), False, [AggCall.from_pretty(c) for c in ("(count:int8)", "(max:int8 $2:int8)")],
                                 0, [0, 1]),
            agg2=HashAggExecutor(cuda, s2.into_executor([I] * 2, []), False, [AggCall.from_pretty(c) for c in ("(count:int8)", "(sum:int8 $1:int8)")],
                                 0, [0])))
    batch_rows = 16
    cap = world * batch_rows
    types2 = [I, I]
    bufs, flags, views = _flat_setup(world, types2, cap)
    v2d = exchange.vnode_to_dest_table(world).cuda()
    peers, flag_ptrs = [b.data_ptr() for b in bufs], [f.data_ptr() for f in flags]
    streams = [torch.cuda.Stream() for _ in range(world)]
    st = [dict(counts=torch.zeros(world, dtype=torch.int64, device="cuda"), err=torch.zeros(1, dtype=torch.int32, device="cuda"),
               total=torch.zeros(1, dtype=torch.int64, device="cuda")) for _ in range(world)]
    calls = [device.FlatExchangeCall([0], v2d, world, r, peers, flag_ptrs, cap, st[r]["counts"], st[r]["err"], st[r]["total"].data_ptr(),
                                     None, max_blocks=24) for r in range(world)]
    batch = [0]

    def ins(rows):
        cols = list(zip(*rows))
        return StreamChunk(np.full(len(rows), abi.OP_INSERT, np.uint8), [Column(I, np.array(c, dtype=np.int64)) for c in cols])

    def shard(rows, key):
        if not rows:
            return [[] for _ in range(world)]
        dest = cuda.vnode_compute(ins(rows), [key], 256).astype(np.int64) * world // 256
        return [[row for row, d in zip(rows, dest) if d == r] for r in range(world)]

    def after_join(rk, chunks):
        for ch in chunks:
            f = rk["flt"].filter(ch)
            if f is not None:  # Project (a.id, a.category, b.price)
                rk["agg1"].apply_chunk(StreamChunk(f.ops, [f.columns[4], f.columns[7], f.columns[1]], f.vis))

    mv = {}

    def barrier(epoch):
        deltas = [device.agg_flush_device(rk["agg1"], epoch, streams[r]) for r, rk in enumerate(ranks)]
        for v in deltas:
            assert not any(v.valid_ptrs[k] for k in (1, 3)), "q4's inner delta has no NULLs"
        # (id, category, count, max) -> Project (category, max): slices of every rank, batch by batch; all W exchanges of
        # a batch are enqueued before any push of it
        slices = []
        for v in deltas:
            s = []
            send_delta(v, [1, 3], batch_rows, s.append)
            slices.append(s)
        for b in range(max(len(s) for s in slices)):
            batch[0] += 1
            torch.cuda.synchronize()  # the previous batch's pushes are done with the receive buffers
            for r in range(world):
                sl = slices[r][b] if b < len(slices[r]) else device.ViewChunk(deltas[r], [1, 3], 0, 0)
                calls[r](sl, batch[0], streams[r])
            for r in range(world):
                device.agg_push_device(ranks[r]["agg2"], device.DeviceChunk(views[r][0], views[r][1], types2), streams[r],
                                       n_rows_dev=st[r]["total"].data_ptr())
        torch.cuda.synchronize()
        errs = [int(s["err"].item()) for s in st]
        if any(e & 2 for e in errs):
            pytest.skip("this device did not run the ranks' kernels side by side (barrier timed out)")
        assert errs == [0] * world
        for r, rk in enumerate(ranks):
            out = view_rows(device.agg_flush_device(rk["agg2"], epoch, streams[r]))
            # (one category lives on one rank and emits at most one row or U-/U+ pair: retractions first)
            for op, row in sorted(out, key=lambda x: x[0] in (abi.OP_INSERT, abi.OP_UPDATE_INSERT)):
                if op in (abi.OP_INSERT, abi.OP_UPDATE_INSERT):
                    mv[row[0]] = (row[1], row[2])
                elif mv.get(row[0]) == (row[1], row[2]):
                    del mv[row[0]]

    bids = [r + [k] for k, r in enumerate(fx["bid"])]
    auct, epoch = fx["auction"], 0
    for step in range(5):
        for r, part in enumerate(shard(auct[step * 8:(step + 1) * 8], 0)):
            if part:
                after_join(ranks[r], ranks[r]["join"].eq_join_oneside(1, ins(part)))
        for r, part in enumerate(shard(bids[step * 10:(step + 1) * 10], 0)):
            if part:
                after_join(ranks[r], ranks[r]["join"].eq_join_oneside(0, ins(part)))
        epoch += 1
        barrier(epoch)
    want = {int(c): Fraction(Decimal(v)) for c, v in fx["expected_q4"]}
    got = {c: Fraction(s, n) for c, (n, s) in mv.items()}
    assert got == want
