// The C++ host mirror's HashAgg watermarks (include/rwgpu_executor.hpp) on the device: the derivation of
// hash_agg.rs:628-637, 660-673 -- a watermark on a column that is not a group key is dropped, one on group key `seq` is
// renumbered to `seq` and buffered (the later one wins), and at a barrier the delta chunks go out first, then the
// watermarks in seq order, then the barrier -- and the cleaning below the window column's watermark
// (rwgpu_agg_update_watermark), seen through rwgpu_agg_stats.
#include <cstdio>

#include "rwgpu_executor.hpp"

using namespace rwgpu;

static int fails = 0;
#define EXPECT(c) do { if (!(c)) { printf("FAILED %s:%d %s\n", __FILE__, __LINE__, #c); fails++; } } while (0)

// 'c' chunk, 'w' watermark (col, val), 'b' barrier
struct Seen { char kind; int32_t col; int64_t val; };

static std::vector<Seen> drain(Execute& ex) {
  std::vector<Seen> v;
  while (auto m = ex.poll_next()) {
    if (std::holds_alternative<StreamChunk>(*m)) v.push_back({'c', 0, 0});
    else if (auto* w = std::get_if<Watermark>(&*m)) v.push_back({'w', w->col_idx, w->val});
    else v.push_back({'b', 0, (int64_t)std::get<Barrier>(*m).epoch});
  }
  return v;
}

static uint64_t groups(HashAggExecutor& ex) {
  uint64_t g = 0;
  check(rwgpu_agg_stats(ex.handle(), &g, nullptr, nullptr));
  return g;
}

int main() {
  if (rwgpu_device_check() != RW_OK) { printf("no CUDA device\n"); return 1; }
  // input (a, b, c, d); group keys [2, 0] (c = seq 0, a = seq 1); the window is group key 1 (column a)
  auto src = std::make_shared<MockSource>(std::vector<int32_t>{RW_T_INT64, RW_T_INT64, RW_T_INT64, RW_T_INT64}, std::vector<int32_t>{});
  HashAggExecutor agg(src, false, {AggCall{RW_AGG_COUNT, -1, RW_T_INT64}}, 0, {2, 0}, 1024, 1);
  src->push_barrier(1);
  auto s = drain(agg);
  EXPECT(s.size() == 1 && s[0].kind == 'b');
  src->push_chunk(StreamChunk::from_pretty(" I I I I\n + 1 0 7 0\n + 5 0 7 0\n + 9 0 7 0"));
  src->push_barrier(2);
  s = drain(agg);
  EXPECT(s.size() == 2 && s[0].kind == 'c' && s[1].kind == 'b');
  EXPECT(groups(agg) == 3);
  src->push_watermark(1, RW_T_INT64, 100);  // not a group key: dropped
  src->push_watermark(0, RW_T_INT64, 2);    // seq 1, the window: replaced below
  src->push_watermark(2, RW_T_INT64, 50);   // seq 0
  src->push_watermark(0, RW_T_INT64, 6);    // seq 1 again: the later one wins (and cleans below 6)
  src->push_chunk(StreamChunk::from_pretty(" I I I I\n + 1 0 7 0"));  // (group (7, 1) changes in the cleaning epoch)
  src->push_barrier(3);
  s = drain(agg);
  EXPECT(s.size() == 4);
  if (s.size() == 4) {
    EXPECT(s[0].kind == 'c');
    EXPECT(s[1].kind == 'w' && s[1].col == 0 && s[1].val == 50);
    EXPECT(s[2].kind == 'w' && s[2].col == 1 && s[2].val == 6);
    EXPECT(s[3].kind == 'b' && s[3].val == 3);
  }
  EXPECT(groups(agg) == 1);  // (7, 9) only: (7, 1) and (7, 5) are below 6
  src->push_barrier(4);  // nothing buffered any more
  s = drain(agg);
  EXPECT(s.size() == 1 && s[0].kind == 'b');
  printf(fails ? "agg watermarks: %d FAILED\n" : "agg watermarks: ok\n", fails);
  return fails ? 1 : 0;
}
