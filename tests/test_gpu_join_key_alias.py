"""GPU: a device view of a positional unified-table push points its matched-side KEY column at the pushed chunk's key.

The unified table joins on one non-float 8-byte key compared bit for bit, and it is an inner join: every visible output
row's matched key equals the input row's key.  The hot kernel does not store that column; the view aliases the input's
key column, or, when the view cannot alias (extra-match rows, deletes, a redo), collect copies the key into it.  Every
case is compared with the CPU oracle fed the same rows."""
import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import HashJoinExecutor, JoinParams, MockSource
from risingwave_b200.stream_chunk import Column, StreamChunk, emitted_multiset, net_multiset

pytestmark = pytest.mark.gpu

TYPES = [abi.T_INT64] * 4
N_AUCT = 4000


def make(be):
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    # left = bids (key column 0, stream key column 1), right = auctions (key column 0 = stream key); output: 4 bid, 4 auction columns
    return HashJoinExecutor(be, abi.JOIN_INNER, sl.into_executor(TYPES, [1]), sr.into_executor(TYPES, [0]),
                            JoinParams([0], [1]), JoinParams([0], []), [False], capacity_hint=1000)


def host_chunk(ops, cols):
    return StreamChunk(np.asarray(ops, np.uint8), [Column(abi.T_INT64, np.asarray(c, np.int64)) for c in cols], None)


def dev_chunk(ch):
    import torch
    from risingwave_b200 import device
    return device.DeviceChunk(torch.from_numpy(ch.ops.copy()).cuda(), [torch.from_numpy(c.data.copy()).cuda() for c in ch.columns], TYPES)


def check(v, o, side, ch, emitted=False):
    cols = [Column(abi.T_INT64, v.column(k).cpu().numpy()) for k in range(v.n_cols)]
    vis = v.visible()
    got = [StreamChunk(v.ops().cpu().numpy(), cols, None if vis is None else vis.cpu().numpy())]
    want = o.eq_join_oneside(side, ch)
    assert net_multiset(got) == net_multiset(want)
    if emitted:
        assert emitted_multiset(got) == emitted_multiset(want)
    return sum(net_multiset(want).values())


def auctions(ids):
    ids = np.asarray(ids)
    return host_chunk(np.full(len(ids), abi.OP_INSERT), [ids, ids * 3, ids * 5, ids * 7])


def bids(rng, n, pk0, key_lo=0, key_hi=N_AUCT + 200):
    return host_chunk(np.full(n, abi.OP_INSERT), [rng.integers(key_lo, key_hi, n), np.arange(n) + pk0,
                                                  rng.integers(0, 1 << 40, n), rng.integers(0, 1 << 40, n)])


def setup(cuda, oracle):
    from risingwave_b200 import device
    g, o = make(cuda), make(oracle)
    a = auctions(np.arange(N_AUCT))
    assert device.join_push_device(g, abi.SIDE_RIGHT, dev_chunk(a)).n_rows == 0
    assert not o.eq_join_oneside(abi.SIDE_RIGHT, a)
    return g, o


def test_bid_push_view_aliases_the_auction_key(cuda, oracle):
    """a plain bid push: output column 4 (auction.id) is the bid chunk's key column; unmatched keys leave holes"""
    from risingwave_b200 import device
    rng = np.random.default_rng(11)
    g, o = setup(cuda, oracle)
    for s in range(2):
        hc = bids(rng, 15000, 10 ** 6 * s)
        ch = dev_chunk(hc)
        v = device.join_push_device(g, abi.SIDE_LEFT, ch)
        assert v.col_ptrs[4] == ch.cols[0].data_ptr() and v.col_ptrs[0] == ch.cols[0].data_ptr()
        assert check(v, o, abi.SIDE_LEFT, hc) > 12000


def test_auction_push_view_aliases_the_bid_key(cuda, oracle):
    """auctions pushed against one stored bid each (deferred rows, no extra rows): output column 0 (bid.auction) is the
    auction chunk's key column"""
    from risingwave_b200 import device
    rng = np.random.default_rng(12)
    g, o = setup(cuda, oracle)
    ids = np.arange(N_AUCT, N_AUCT + 3000)
    hb = bids(rng, 3000, 0)
    hb.columns[0].data[:] = ids
    assert device.join_push_device(g, abi.SIDE_LEFT, dev_chunk(hb)).n_rows == 0
    assert not o.eq_join_oneside(abi.SIDE_LEFT, hb)
    ha = auctions(ids)
    ch = dev_chunk(ha)
    v = device.join_push_device(g, abi.SIDE_RIGHT, ch)
    assert v.n_rows == ha.capacity() and v.col_ptrs[0] == ch.cols[0].data_ptr()
    assert check(v, o, abi.SIDE_RIGHT, ha) == 3000


def test_unaliased_views_carry_the_key(cuda, oracle):
    """the view is not aliased -- extra-match rows, then U- / U+ pairs with deletes -- so collect copies the key into the
    output column the hot kernel skipped"""
    from risingwave_b200 import device
    rng = np.random.default_rng(13)
    g, o = setup(cuda, oracle)
    # several bids per new auction, then the auctions: extra-match rows
    hb = bids(rng, 5000, 0, key_lo=N_AUCT, key_hi=N_AUCT + 800)
    assert device.join_push_device(g, abi.SIDE_LEFT, dev_chunk(hb)).n_rows == 0
    assert not o.eq_join_oneside(abi.SIDE_LEFT, hb)
    ha = auctions(np.arange(N_AUCT, N_AUCT + 800))
    ch = dev_chunk(ha)
    v = device.join_push_device(g, abi.SIDE_RIGHT, ch)
    assert v.n_rows > ha.capacity() and v.col_ptrs[0] != ch.cols[0].data_ptr()
    assert check(v, o, abi.SIDE_RIGHT, ha) == 5000
    # bids on existing auctions: every one matches once
    hc = bids(rng, 6000, 10 ** 6, key_hi=N_AUCT)
    check(device.join_push_device(g, abi.SIDE_LEFT, dev_chunk(hc)), o, abi.SIDE_LEFT, hc)
    m = 2000
    pick = rng.permutation(6000)[:m]
    old = [c.data[pick] for c in hc.columns]
    new = [c.copy() for c in old]
    new[3][: m // 2] += 1  # half of the pairs change a payload column, the other half are no-op updates
    ops = np.tile([abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT], m)
    cols = [np.stack([a, b], axis=1).reshape(-1) for a, b in zip(old, new)]
    dead = rng.permutation(np.setdiff1d(np.arange(6000), pick))[:500]
    hu = host_chunk(np.concatenate([ops, np.full(500, abi.OP_DELETE)]), [np.concatenate([c, d.data[dead]]) for c, d in zip(cols, hc.columns)])
    ch = dev_chunk(hu)
    v = device.join_push_device(g, abi.SIDE_LEFT, ch)
    assert v.n_rows == hu.capacity() and v.col_ptrs[4] != ch.cols[0].data_ptr()
    check(v, o, abi.SIDE_LEFT, hu, emitted=True)
