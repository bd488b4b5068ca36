"""GPU: many chained-side rows on a few keys in ONE plain chunk, through the quad-cooperative kernel (uni_hot_kernel).

Concurrent pushes on one key race between loading the bucket and exchanging its chain word (head | count); the
count must still come out exact.  The inline-side U- / U+ pairs and the deletes that follow read that count: an
update emits exactly `count` matches, so a count that is off shows up as missing or surplus rows."""
import numpy as np
import pytest

from risingwave_b200 import abi
from risingwave_b200.executor import HashJoinExecutor, JoinParams, MockSource
from risingwave_b200.stream_chunk import Column, StreamChunk, net_multiset

pytestmark = pytest.mark.gpu

TYPES = [abi.T_INT64] * 4


def make(be):
    _, sl = MockSource.channel()
    _, sr = MockSource.channel()
    # left = bids (stream key = column 1: chained side), right = auctions (stream key = the join key: inline side)
    return HashJoinExecutor(be, abi.JOIN_INNER, sl.into_executor(TYPES, [1]), sr.into_executor(TYPES, [0]),
                            JoinParams([0], [1]), JoinParams([0], []), [False], capacity_hint=1000)


def plain(ops, cols):
    return StreamChunk(np.asarray(ops, np.uint8), [Column(abi.T_INT64, np.asarray(c, np.int64)) for c in cols])


def test_contended_chain_pushes_keep_exact_counts(cuda, oracle):
    import torch
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(2024)
    n_auct, n_hot, n_bids = 64, 6, 12000
    exs = [make(cuda), make(oracle)]

    def step(side, chunk):
        outs = [net_multiset(ex.eq_join_oneside(side, chunk)) for ex in exs]
        assert outs[0] == outs[1]
        return outs[0]

    auct_ids = np.arange(n_auct)
    step(1, plain(np.full(n_auct, abi.OP_INSERT), [auct_ids, auct_ids * 3, auct_ids * 5, auct_ids * 7]))
    # 12000 bids, all but a few on 6 auctions: thousands of pushes per key inside one launch
    key = rng.integers(0, n_hot, n_bids)
    key[::97] = rng.integers(n_hot, n_auct, len(key[::97]))
    pk = np.arange(n_bids) + 10 ** 6
    bid_cols = [key, pk, rng.integers(0, 1 << 30, n_bids), rng.integers(0, 1 << 30, n_bids)]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(0, plain(np.full(n_bids, abi.OP_INSERT), bid_cols))
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    assert any("uni_hot_kernel<false, false" in n for n in names), "the bid chunk did not run through the quad-cooperative kernel"

    c3_live = auct_ids * 7

    def updates(keys, bump):  # U- names the live auction row, U+ changes its last column
        k = np.repeat(keys, 2)
        ops = np.tile([abi.OP_UPDATE_DELETE, abi.OP_UPDATE_INSERT], len(keys))
        c3 = np.stack([c3_live[keys], keys * 7 + bump], axis=1).reshape(-1)
        c3_live[keys] = keys * 7 + bump
        return plain(ops, [k, k * 3, k * 5, c3])

    hot = np.arange(n_hot)
    got = step(1, updates(hot, 1))
    assert len(got) > 0
    # delete a third of the bids (tail kernel: atomicSub on the same count), then read the counts again
    dead = rng.permutation(n_bids)[: n_bids // 3]
    step(0, plain(np.full(len(dead), abi.OP_DELETE), [c[dead] for c in bid_cols]))
    step(1, updates(np.arange(n_auct), 2))
    # a second contended push on top of the corrected counts
    more = [rng.integers(0, n_hot, 4000), np.arange(4000) + 2 * 10 ** 6, np.zeros(4000), np.ones(4000)]
    step(0, plain(np.full(4000, abi.OP_INSERT), more))
    step(1, updates(hot, 3))
