"""GPU: device views of a positional push point their update-side columns at the pushed chunk.

A plain chunk (no bitmaps, row count known on the host) pushed through rwgpu_join_push_device or the async pair leaves
the update-side output columns to the input: output row r is input row r, so the view's columns are the chunk's own
tensors.  Whenever that does not hold -- extra-match rows, a push with deletes (the no-op pass reads the output
columns), an output-capacity redo, a counted chunk, a chunk with bitmaps -- the output columns are written and the view
points at them.  Every case is compared with the CPU oracle fed the same rows."""
import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import HashJoinExecutor, JoinParams, MockSource
from risingwave_b200.stream_chunk import Column, StreamChunk, emitted_multiset, net_multiset

pytestmark = pytest.mark.gpu

TYPES = [abi.T_INT64] * 4
N_AUCT = 5000


def make(be):
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    # left = bids (stream key = column 1), right = auctions (stream key = the join key): the unified-table plan
    return HashJoinExecutor(be, abi.JOIN_INNER, sl.into_executor(TYPES, [1]), sr.into_executor(TYPES, [0]),
                            JoinParams([0], [1]), JoinParams([0], []), [False], capacity_hint=1000)


def host_chunk(ops, cols, vis=None):
    return StreamChunk(np.asarray(ops, np.uint8), [Column(abi.T_INT64, np.asarray(c, np.int64)) for c in cols], vis)


def dev_chunk(ch):
    import torch
    from risingwave_b200 import device
    vis = None
    if ch.vis is not None:
        words = np.packbits(np.concatenate([ch.vis, np.zeros(-len(ch.vis) % 64, bool)]), bitorder="little").view(np.int64)
        vis = torch.from_numpy(words.copy()).cuda()
    return device.DeviceChunk(torch.from_numpy(ch.ops.copy()).cuda(), [torch.from_numpy(c.data.copy()).cuda() for c in ch.columns],
                              TYPES, visibility=vis)


def view_chunk(v):
    cols = [Column(abi.T_INT64, v.column(k).cpu().numpy()) for k in range(v.n_cols)]
    vis = v.visible()
    return StreamChunk(v.ops().cpu().numpy(), cols, None if vis is None else vis.cpu().numpy())


def aliased(v, ch, first_col):
    """the view's update-side columns are the chunk's tensors (output columns first_col .. first_col + 3)"""
    return all(v.col_ptrs[first_col + k] == ch.cols[k].data_ptr() for k in range(4))


def auctions(ids):
    ids = np.asarray(ids)
    return host_chunk(np.full(len(ids), abi.OP_INSERT), [ids, ids * 3, ids * 5, ids * 7])


def bids(rng, n, pk0, key_hi=N_AUCT + 200):
    # keys above N_AUCT match nothing: holes in the positional output
    return host_chunk(np.full(n, abi.OP_INSERT), [rng.integers(0, key_hi, n), np.arange(n) + pk0,
                                                  rng.integers(0, 1 << 40, n), rng.integers(0, 1 << 40, n)])


def setup(cuda, oracle):
    from risingwave_b200 import device
    g, o = make(cuda), make(oracle)
    a = auctions(np.arange(N_AUCT))
    assert device.join_push_device(g, abi.SIDE_RIGHT, dev_chunk(a)).n_rows == 0
    assert not o.eq_join_oneside(abi.SIDE_RIGHT, a)
    return g, o


def check(v, o, side, ch, emitted=False):
    want = o.eq_join_oneside(side, ch)
    got = [view_chunk(v)]
    assert net_multiset(got) == net_multiset(want)
    if emitted:
        assert emitted_multiset(got) == emitted_multiset(want)
    return sum(net_multiset(want).values())


def test_plain_bid_pushes_alias_the_input(cuda, oracle):
    """synchronous pushes, then async pushes with two outstanding: the view's bid columns are the input tensors"""
    import torch
    from risingwave_b200 import device
    rng = np.random.default_rng(1)
    g, o = setup(cuda, oracle)
    for s in range(3):
        hc = bids(rng, 20000 + 1000 * s, 10 ** 6 * s)
        ch = dev_chunk(hc)
        v = device.join_push_device(g, abi.SIDE_LEFT, ch)
        assert v.n_rows == hc.capacity() and aliased(v, ch, 0)
        assert check(v, o, abi.SIDE_LEFT, hc) > 15000
    stream = torch.cuda.Stream()
    hcs = [bids(rng, 30000 - 1000 * s, 10 ** 7 + 10 ** 6 * s) for s in range(5)]
    chs = [dev_chunk(h) for h in hcs]
    with torch.cuda.stream(stream):
        for s in range(len(chs) + 1):
            if s < len(chs):
                device.join_push_device_async(g, abi.SIDE_LEFT, chs[s], stream)
            if s > 0:
                v = device.join_collect(g, stream)
                assert v.n_rows == hcs[s - 1].capacity() and aliased(v, chs[s - 1], 0)
                assert check(v, o, abi.SIDE_LEFT, hcs[s - 1]) > 15000


def test_multi_match_pushes_write_their_columns(cuda, oracle):
    """auctions pushed against stored bids, several per auction: extra-match rows, so the output is not aliased"""
    from risingwave_b200 import device
    rng = np.random.default_rng(2)
    g, o = setup(cuda, oracle)
    # bids on auctions that do not exist yet: stored, no output
    hb = bids(rng, 6000, 0, key_hi=N_AUCT + 1000)
    hb.columns[0].data[:] = N_AUCT + rng.integers(0, 1000, 6000)
    assert device.join_push_device(g, abi.SIDE_LEFT, dev_chunk(hb)).n_rows == 0
    assert not o.eq_join_oneside(abi.SIDE_LEFT, hb)
    ha = auctions(np.arange(N_AUCT, N_AUCT + 1000))
    ch = dev_chunk(ha)
    v = device.join_push_device(g, abi.SIDE_RIGHT, ch)
    assert v.n_rows > ha.capacity() and not aliased(v, ch, 4)
    assert check(v, o, abi.SIDE_RIGHT, ha) == 6000


def test_update_pairs_run_the_noop_pass_unaliased(cuda, oracle):
    """bid U- / U+ pairs, half of them changing nothing (the no-op pass hides those), and deletes"""
    from risingwave_b200 import device
    rng = np.random.default_rng(3)
    g, o = setup(cuda, oracle)
    hb = bids(rng, 8000, 0, key_hi=N_AUCT)
    v = device.join_push_device(g, abi.SIDE_LEFT, dev_chunk(hb))
    check(v, o, abi.SIDE_LEFT, hb)
    m = 3000
    pick = rng.permutation(8000)[:m]
    old = [c.data[pick] for c in hb.columns]
    new = [c.copy() for c in old]
    new[3][: m // 2] += 1  # the first half changes a payload column, the second half is a no-op update
    ops = np.tile([abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT], m)
    cols = [np.stack([a, b], axis=1).reshape(-1) for a, b in zip(old, new)]
    dead = rng.permutation(np.setdiff1d(np.arange(8000), pick))[:1000]
    hu = host_chunk(np.concatenate([ops, np.full(1000, abi.OP_DELETE)]), [np.concatenate([c, d.data[dead]]) for c, d in zip(cols, hb.columns)])
    ch = dev_chunk(hu)
    v = device.join_push_device(g, abi.SIDE_LEFT, ch)
    assert v.n_rows == hu.capacity() and not aliased(v, ch, 0)
    vis = v.visible()
    assert vis is not None and int((~vis[: 2 * m]).sum()) == m  # exactly the no-op pairs are hidden
    check(v, o, abi.SIDE_LEFT, hu, emitted=True)


def test_counted_and_bitmap_chunks_are_not_aliased(cuda, oracle):
    import torch
    from risingwave_b200 import device
    rng = np.random.default_rng(4)
    g, o = setup(cuda, oracle)
    # counted: the buffers hold `cap` rows, the device-resident count says n
    n, cap = 9000, 12000
    hc = bids(rng, cap, 0)
    ch = dev_chunk(hc)
    count = torch.tensor([n], dtype=torch.int64, device="cuda")
    v = device.join_push_device(g, abi.SIDE_LEFT, ch, n_rows_dev=count.data_ptr())
    assert v.n_rows == n and not aliased(v, ch, 0)
    check(v, o, abi.SIDE_LEFT, hc.slice(0, n))
    # a visibility bitmap: the chunk is not plain
    hv = bids(rng, 10000, 10 ** 6)
    hv.vis = rng.random(10000) < 0.8
    ch = dev_chunk(hv)
    v = device.join_push_device(g, abi.SIDE_LEFT, ch)
    assert v.n_rows == 10000 and not aliased(v, ch, 0)
    check(v, o, abi.SIDE_LEFT, hv)


def test_output_capacity_redo(cuda, oracle):
    """more extra-match rows than the output area reserved at launch: the push is redone with room for all of them.
    The output area holds about 11000 rows after the first auction push, and the small bid pushes do not grow it."""
    from risingwave_b200 import device
    rng = np.random.default_rng(5)
    g, o = setup(cuda, oracle)
    for s in range(20):  # ~20 bids per new auction
        hb = bids(rng, 2000, 2000 * s)
        hb.columns[0].data[:] = N_AUCT + rng.integers(0, 2000, 2000)
        assert device.join_push_device(g, abi.SIDE_LEFT, dev_chunk(hb)).n_rows == 0
        assert not o.eq_join_oneside(abi.SIDE_LEFT, hb)
    ha = auctions(np.arange(N_AUCT, N_AUCT + 2000))
    v = device.join_push_device(g, abi.SIDE_RIGHT, dev_chunk(ha))
    assert v.n_rows >= 40000
    assert check(v, o, abi.SIDE_RIGHT, ha) == 40000
    # the bid side's plain pushes alias again afterwards
    hc = bids(rng, 20000, 10 ** 6, key_hi=N_AUCT)
    ch = dev_chunk(hc)
    v = device.join_push_device(g, abi.SIDE_LEFT, ch)
    assert aliased(v, ch, 0)
    check(v, o, abi.SIDE_LEFT, hc)


def test_view_keeps_the_pushed_chunk_alive(cuda, oracle):
    """the caller drops its last reference to the chunk; tensors of the same size allocated and overwritten afterwards
    must not show up in the view"""
    import torch
    from risingwave_b200 import device
    rng = np.random.default_rng(6)
    g, o = setup(cuda, oracle)
    n = 25000

    def scribble():
        junk = [torch.full((n,), -12345, dtype=torch.int64, device="cuda") for _ in range(8)]
        junk += [torch.full((n,), 7, dtype=torch.uint8, device="cuda") for _ in range(2)]
        torch.cuda.synchronize()
        return junk

    hc = bids(rng, n, 0)
    v = device.join_push_device(g, abi.SIDE_LEFT, dev_chunk(hc))
    junk = scribble()
    assert check(v, o, abi.SIDE_LEFT, hc) > 15000
    del junk
    hc = bids(rng, n, 10 ** 6)
    device.join_push_device_async(g, abi.SIDE_LEFT, dev_chunk(hc))
    v = device.join_collect(g)
    junk = scribble()
    assert check(v, o, abi.SIDE_LEFT, hc) > 15000
    del junk
