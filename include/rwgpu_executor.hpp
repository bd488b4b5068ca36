// rwgpu_executor.hpp -- C++ host layer above the C ABI (include/rwgpu.h), mirroring the reference's
// executor interface for the HashAgg / HashJoin path.  Header-only, C++17, links against librwgpu.so.
//
// The reference's host code is Rust (no toolchain in this image), so the host side above the ABI is
// written in C++; names and argument order follow the reference:
//   trait Execute / Message / Barrier / Watermark   src/stream/src/executor/mod.rs:240-253,403-410,1283-1299
//   MockSource + MessageSender                       src/stream/src/executor/test_utils/mock_source.rs:16-137
//   StreamChunk / Op / from_pretty                   src/common/src/array/stream_chunk.rs:45-110,650-750
//   HashAggExecutor   (new_boxed_hash_agg_executor)  src/stream/src/executor/test_utils/agg_executor.rs:224-300
//   HashJoinExecutor::new                            src/stream/src/executor/hash_join.rs:255-301
//   barrier_align                                    src/stream/src/executor/barrier_align.rs:44-165
// Errors: a non-zero ABI status becomes a StreamExecutorError exception (the Rust shim maps it to
// `StreamExecutorResult::Err`, which terminates the actor; src/stream/src/executor/error.rs).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <optional>
#include <sstream>
#include <stdexcept>
#include <string>
#include <variant>
#include <vector>

#include "rwgpu.h"

namespace rwgpu {

struct StreamExecutorError : std::runtime_error {
  int code;
  StreamExecutorError(int c, const std::string& m) : std::runtime_error("rwgpu status " + std::to_string(c) + ": " + m), code(c) {}
};
inline void check(int32_t rc) {
  if (rc != RW_OK) throw StreamExecutorError(rc, rwgpu_last_error());
}

enum class Op : uint8_t { Insert = RW_OP_INSERT, Delete = RW_OP_DELETE, UpdateInsert = RW_OP_UPDATE_INSERT, UpdateDelete = RW_OP_UPDATE_DELETE };

// one datum for tests / pretty printing: NULL or an integer-like / float value
struct Datum {
  bool null = true;
  int64_t i = 0;
  double f = 0;
  bool operator<(const Datum& o) const { return std::tie(null, i, f) < std::tie(o.null, o.i, o.f); }
  bool operator==(const Datum& o) const { return null == o.null && (null || (i == o.i && f == o.f)); }
};
using Row = std::vector<Datum>;

struct Column {
  int32_t type = RW_T_INT64;
  std::vector<uint8_t> data;     // n * width bytes
  std::vector<uint64_t> validity;  // empty = no NULLs
};

class StreamChunk {
 public:
  std::vector<uint8_t> ops;
  std::vector<Column> columns;
  std::vector<uint64_t> visibility;  // empty = all visible

  int64_t capacity() const { return (int64_t)ops.size(); }
  bool is_visible(int64_t r) const { return visibility.empty() || ((visibility[r >> 6] >> (r & 63)) & 1); }

  // the `from_pretty` test DSL (data_chunk.rs:708-790): header of type tokens (I i F f B TZ SRL D s),
  // then `op v v .. [D]` lines; `.` = NULL, trailing `D` = invisible
  static StreamChunk from_pretty(const std::string& s) {
    StreamChunk c;
    std::istringstream in(s);
    std::string line;
    bool header = true;
    std::vector<bool> vis;
    while (std::getline(in, line)) {
      std::istringstream ls(line);
      std::vector<std::string> tok;
      for (std::string t; ls >> t;) { if (t == "//") break; tok.push_back(t); }
      if (tok.empty()) continue;
      if (header) {
        for (auto& t : tok) { Column col; col.type = type_of(t); c.columns.push_back(col); }
        header = false;
        continue;
      }
      c.ops.push_back(tok[0] == "+" ? RW_OP_INSERT : tok[0] == "-" ? RW_OP_DELETE : tok[0] == "U+" ? RW_OP_UPDATE_INSERT : RW_OP_UPDATE_DELETE);
      const int64_t r = c.capacity() - 1;
      for (size_t k = 0; k < c.columns.size(); k++) c.push_value(k, r, tok[1 + k]);
      vis.push_back(!(tok.size() > 1 + c.columns.size() && tok[1 + c.columns.size()] == "D"));
    }
    bool all = true;
    for (bool v : vis) all = all && v;
    if (!all) {
      c.visibility.assign((vis.size() + 63) / 64, 0);
      for (size_t r = 0; r < vis.size(); r++) if (vis[r]) c.visibility[r >> 6] |= 1ull << (r & 63);
    }
    for (auto& col : c.columns) {  // drop all-ones validity
      bool any_null = false;
      for (int64_t r = 0; r < c.capacity(); r++) any_null = any_null || !((col.validity[r >> 6] >> (r & 63)) & 1);
      if (!any_null) col.validity.clear();
    }
    return c;
  }

  Datum datum(size_t k, int64_t r) const {
    const Column& col = columns[k];
    Datum d;
    if (!col.validity.empty() && !((col.validity[r >> 6] >> (r & 63)) & 1)) return d;
    d.null = false;
    const uint8_t* p = col.data.data() + (size_t)r * rwgpu_type_width(col.type);
    switch (col.type) {
      case RW_T_BOOL: d.i = p[0]; break;
      case RW_T_INT16: { int16_t v; memcpy(&v, p, 2); d.i = v; break; }
      case RW_T_INT32: case RW_T_DATE: { int32_t v; memcpy(&v, p, 4); d.i = v; break; }
      case RW_T_FLOAT32: { float v; memcpy(&v, p, 4); d.f = v; break; }
      case RW_T_FLOAT64: { double v; memcpy(&v, p, 8); d.f = v; break; }
      default: { int64_t v; memcpy(&v, p, 8); d.i = v; break; }
    }
    return d;
  }
  Row row(int64_t r) const {
    Row x;
    for (size_t k = 0; k < columns.size(); k++) x.push_back(datum(k, r));
    return x;
  }

  // borrowed view for one ABI call
  struct View {
    std::vector<rw_column> cols;
    rw_chunk raw;
  };
  View view() const {
    View v;
    for (auto& c : columns) v.cols.push_back(rw_column{c.type, 0, c.data.data(), c.validity.empty() ? nullptr : c.validity.data(), nullptr});
    v.raw = rw_chunk{capacity(), (int32_t)columns.size(), 0, ops.data(), visibility.empty() ? nullptr : visibility.data(), v.cols.data()};
    return v;
  }
  static StreamChunk from_abi(const rw_chunk& v) {
    StreamChunk c;
    const size_t nw = (size_t)((v.n_rows + 63) / 64);
    c.ops.assign(v.ops, v.ops + v.n_rows);
    if (v.visibility) c.visibility.assign(v.visibility, v.visibility + nw);
    for (int k = 0; k < v.n_cols; k++) {
      Column col;
      col.type = v.columns[k].type;
      const size_t bytes = (size_t)v.n_rows * rwgpu_type_width(col.type);
      col.data.assign((const uint8_t*)v.columns[k].data, (const uint8_t*)v.columns[k].data + bytes);
      if (v.columns[k].validity) col.validity.assign(v.columns[k].validity, v.columns[k].validity + nw);
      c.columns.push_back(std::move(col));
    }
    return c;
  }

 private:
  static int32_t type_of(const std::string& t) {
    if (t == "I") return RW_T_INT64;
    if (t == "i") return RW_T_INT32;
    if (t == "s") return RW_T_INT16;
    if (t == "F") return RW_T_FLOAT64;
    if (t == "f") return RW_T_FLOAT32;
    if (t == "B") return RW_T_BOOL;
    if (t == "TZ") return RW_T_TIMESTAMPTZ;
    if (t == "TS") return RW_T_TIMESTAMP;
    if (t == "SRL") return RW_T_SERIAL;
    if (t == "D") return RW_T_DATE;
    throw std::invalid_argument("unsupported type token " + t);
  }
  void push_value(size_t k, int64_t r, const std::string& tok) {
    Column& col = columns[k];
    const int w = rwgpu_type_width(col.type);
    col.data.resize((size_t)(r + 1) * w, 0);
    if (col.validity.size() <= (size_t)(r >> 6)) col.validity.resize((r >> 6) + 1, 0);
    if (tok == ".") return;
    col.validity[r >> 6] |= 1ull << (r & 63);
    uint8_t* p = col.data.data() + (size_t)r * w;
    switch (col.type) {
      case RW_T_BOOL: p[0] = (tok == "t" || tok == "true" || tok == "1"); break;
      case RW_T_INT16: { int16_t v = (int16_t)std::stoll(tok); memcpy(p, &v, 2); break; }
      case RW_T_INT32: case RW_T_DATE: { int32_t v = (int32_t)std::stoll(tok); memcpy(p, &v, 4); break; }
      case RW_T_FLOAT32: { float v = std::stof(tok); memcpy(p, &v, 4); break; }
      case RW_T_FLOAT64: { double v = std::stod(tok); memcpy(p, &v, 8); break; }
      default: { int64_t v = std::stoll(tok); memcpy(p, &v, 8); break; }
    }
  }
};

// net applied multiset of a chunk sequence: the `Store::apply_chunk` comparator of the reference's
// snapshot tests (src/stream/tests/integration_tests/snapshot.rs:219-254)
inline std::map<Row, int64_t> net_multiset(const std::vector<StreamChunk>& chunks) {
  std::map<Row, int64_t> m;
  for (auto& c : chunks)
    for (int64_t r = 0; r < c.capacity(); r++) {
      if (!c.is_visible(r)) continue;
      m[c.row(r)] += (c.ops[r] == RW_OP_INSERT || c.ops[r] == RW_OP_UPDATE_INSERT) ? 1 : -1;
    }
  for (auto it = m.begin(); it != m.end();) it = it->second == 0 ? m.erase(it) : std::next(it);
  return m;
}

// ------------------------------------------------------------------------------------ Message
struct Barrier { uint64_t epoch = 0; };
struct Watermark { int32_t col_idx = 0; int32_t data_type = 0; int64_t val = 0; };
using Message = std::variant<StreamChunk, Barrier, Watermark>;

// trait Execute: a pull-based stream of messages; std::nullopt == Poll::Pending
class Execute {
 public:
  virtual ~Execute() = default;
  virtual std::optional<Message> poll_next() = 0;
  virtual const std::vector<int32_t>& schema() const = 0;
  virtual const std::vector<int32_t>& stream_key() const = 0;
};

// MockSource::channel(): the sender half is folded into the source (push_* == MessageSender::push_*)
class MockSource : public Execute {
 public:
  MockSource(std::vector<int32_t> schema, std::vector<int32_t> stream_key) : schema_(std::move(schema)), key_(std::move(stream_key)) {}
  void push_chunk(StreamChunk c) { q_.emplace_back(std::move(c)); }
  void push_barrier(uint64_t epoch, bool /*stop*/ = false) { q_.emplace_back(Barrier{epoch}); }
  void push_watermark(int32_t col, int32_t type, int64_t val) { q_.emplace_back(Watermark{col, type, val}); }
  std::optional<Message> poll_next() override {
    if (q_.empty()) return std::nullopt;
    Message m = std::move(q_.front());
    q_.pop_front();
    return m;
  }
  const std::vector<int32_t>& schema() const override { return schema_; }
  const std::vector<int32_t>& stream_key() const override { return key_; }

 private:
  std::deque<Message> q_;
  std::vector<int32_t> schema_, key_;
};

inline std::vector<StreamChunk> take_out(rwgpu_out* out) {
  std::vector<StreamChunk> v;
  for (int32_t i = 0; i < rwgpu_out_num_chunks(out); i++) {
    rw_chunk view;
    check(rwgpu_out_chunk(out, i, &view));
    v.push_back(StreamChunk::from_abi(view));
  }
  rwgpu_out_release(out);
  return v;
}

// ------------------------------------------------------------------------------------ HashAgg
struct AggCall { int32_t kind, arg_col, ret_type; };

// window_col_idx_in_group_key: the group key leading the intermediate state table's pk (hash_agg.rs:569-570; group key 0
// in the reference's test helper, agg_executor.rs:157-171): a watermark on it cleans the state below it
class HashAggExecutor : public Execute {
 public:
  HashAggExecutor(std::shared_ptr<Execute> input, bool is_append_only, std::vector<AggCall> agg_calls, int32_t row_count_index,
                  std::vector<int32_t> group_key_indices, int32_t chunk_size = 1024, int32_t window_col_idx_in_group_key = 0)
      : input_(std::move(input)), window_seq_(window_col_idx_in_group_key) {
    std::vector<rw_agg_call> calls;
    for (auto& c : agg_calls) calls.push_back(rw_agg_call{c.kind, c.arg_col, c.ret_type, 0});
    rw_agg_desc d{};
    d.n_input_cols = (int32_t)input_->schema().size();
    d.input_types = input_->schema().data();
    d.n_group_keys = (int32_t)group_key_indices.size();
    d.group_key_indices = group_key_indices.data();
    d.n_calls = (int32_t)calls.size();
    d.calls = calls.data();
    d.row_count_index = row_count_index;
    d.is_append_only = is_append_only;
    d.chunk_size = chunk_size;
    d.strict_consistency = 1;
    check(rwgpu_agg_create(&d, &h_));
    for (int32_t k : group_key_indices) schema_.push_back(input_->schema()[k]);
    for (auto& c : agg_calls) schema_.push_back(c.ret_type);
    for (size_t seq = 0; seq < group_key_indices.size(); seq++) group_key_seq_[group_key_indices[seq]] = (int32_t)seq;
    window_col_ = group_key_indices.at((size_t)window_col_idx_in_group_key);
    buffered_.resize(group_key_indices.size());
  }
  ~HashAggExecutor() override { rwgpu_agg_destroy(h_); }
  // the Message::Watermark arm of execute_inner (hash_agg.rs:628-637): a watermark on a column that is not a group key is
  // dropped; one on group key `seq` is buffered as `seq` (the later one wins) until the barrier; one on the window
  // column also cleans the state below it at the next barrier (update_watermark at the end of flush_data, :503-507)
  void handle_watermark(const Watermark& wm) {
    auto it = group_key_seq_.find(wm.col_idx);
    if (it == group_key_seq_.end()) return;
    if (wm.col_idx == window_col_) check(rwgpu_agg_update_watermark(h_, window_seq_, wm.val));
    buffered_[(size_t)it->second] = Watermark{it->second, wm.data_type, wm.val};
  }
  // execute_inner (hash_agg.rs:561-706): chunks are applied; a barrier flushes the deltas, then the buffered group-key
  // watermarks go out in seq order, then the barrier (:651-676)
  std::optional<Message> poll_next() override {
    while (true) {
      if (!pending_.empty()) { Message m = std::move(pending_.front()); pending_.pop_front(); return m; }
      auto m = input_->poll_next();
      if (!m) return std::nullopt;
      if (auto* c = std::get_if<StreamChunk>(&*m)) {
        auto v = c->view();
        check(rwgpu_agg_push(h_, &v.raw));  // apply_chunk
      } else if (auto* b = std::get_if<Barrier>(&*m)) {
        if (first_) { first_ = false; return m; }
        rwgpu_out* out = nullptr;
        check(rwgpu_agg_flush(h_, b->epoch, &out));  // flush_data
        for (auto& ch : take_out(out)) pending_.emplace_back(std::move(ch));
        for (auto& w : buffered_)
          if (w) { pending_.emplace_back(*w); w.reset(); }
        pending_.emplace_back(*b);
      } else {
        handle_watermark(std::get<Watermark>(*m));
      }
    }
  }
  const std::vector<int32_t>& schema() const override { return schema_; }
  const std::vector<int32_t>& stream_key() const override { return key_; }
  rwgpu_agg* handle() const { return h_; }  // for diagnostics (rwgpu_agg_stats)

 private:
  std::shared_ptr<Execute> input_;
  rwgpu_agg* h_ = nullptr;
  bool first_ = true;
  std::deque<Message> pending_;
  std::vector<int32_t> schema_, key_;
  int32_t window_seq_ = 0, window_col_ = 0;
  std::map<int32_t, int32_t> group_key_seq_;  // input column -> group key seq (the last one of a column grouped twice)
  std::vector<std::optional<Watermark>> buffered_;
};

// ------------------------------------------------------------------------------------ Filter
// FilterExecutor / UpsertFilterExecutor::new(ctx, input, expr) (filter.rs:33-56) for the predicates the device
// evaluates: a conjunction of integer comparisons (col cmp col | col cmp constant).
class FilterExecutor : public Execute {
 public:
  FilterExecutor(std::shared_ptr<Execute> input, std::vector<rw_filter_term> conjuncts, bool upsert = false)
      : input_(std::move(input)), terms_(std::move(conjuncts)), upsert_(upsert) {}
  // FilterExecutorInner::filter (filter.rs:58-150): same columns, new ops / visibility; nullopt = nothing visible
  std::optional<StreamChunk> filter(const StreamChunk& c) const {
    StreamChunk out = c;
    out.visibility.assign((size_t)((c.capacity() + 63) / 64), 0);
    int64_t n_visible = 0;
    auto v = c.view();
    check(rwgpu_filter(&v.raw, terms_.data(), (int32_t)terms_.size(), upsert_ ? 1 : 0, out.ops.data(), out.visibility.data(), &n_visible));
    if (n_visible == 0) return std::nullopt;
    return out;
  }
  // execute_inner (filter.rs:172-194)
  std::optional<Message> poll_next() override {
    while (true) {
      auto m = input_->poll_next();
      if (!m) return std::nullopt;
      if (auto* c = std::get_if<StreamChunk>(&*m)) {
        auto out = filter(*c);
        if (out) return Message(std::move(*out));
        continue;
      }
      return m;
    }
  }
  const std::vector<int32_t>& schema() const override { return input_->schema(); }
  const std::vector<int32_t>& stream_key() const override { return input_->stream_key(); }

 private:
  std::shared_ptr<Execute> input_;
  std::vector<rw_filter_term> terms_;
  bool upsert_;
};

// ------------------------------------------------------------------------------------ watermarks
// BufferedWatermarks<Id> (src/stream/src/executor/watermark/mod.rs:38-115): per upstream id the smallest buffered
// watermark sits in a heap, later ones are staged behind it; a watermark is emitted when EVERY upstream has one in the
// heap (the smallest wins) and equal ones that follow are swallowed.  Order by value (mod.rs:1219-1222), equality on
// (col_idx, value).
class BufferedWatermarks {
 public:
  explicit BufferedWatermarks(std::vector<int> ids) { for (int i : ids) staged_[i]; }
  std::optional<Watermark> handle_watermark(int id, const Watermark& wm) {
    Staged& st = staged_.at(id);
    if (st.in_heap) {
      if (st.q.size() >= 1024) st.q.pop_front();
      st.q.push_back(wm);
      return std::nullopt;
    }
    st.in_heap = true;
    push(wm, id);
    return check_watermark_heap();
  }
  std::optional<Watermark> check_watermark_heap() {
    std::optional<Watermark> emit;
    while (!heap_.empty() && (heap_.size() == staged_.size() ||
                              (emit && emit->col_idx == heap_.front().wm.col_idx && emit->val == heap_.front().wm.val))) {
      std::pop_heap(heap_.begin(), heap_.end(), later);
      Entry e = heap_.back();
      heap_.pop_back();
      emit = e.wm;
      Staged& st = staged_.at(e.id);
      if (!st.q.empty()) { push(st.q.front(), e.id); st.q.pop_front(); }
      else st.in_heap = false;
    }
    return emit;
  }

 private:
  struct Entry { Watermark wm; int id; };
  struct Staged { bool in_heap = false; std::deque<Watermark> q; };
  static bool later(const Entry& a, const Entry& b) { return a.wm.val != b.wm.val ? a.wm.val > b.wm.val : a.id > b.id; }  // min-heap
  void push(const Watermark& wm, int id) { heap_.push_back(Entry{wm, id}); std::push_heap(heap_.begin(), heap_.end(), later); }
  std::vector<Entry> heap_;
  std::map<int, Staged> staged_;
};

// ------------------------------------------------------------------------------------ HashJoin
struct JoinParams { std::vector<int32_t> join_key_indices, deduped_pk_indices; };

class HashJoinExecutor : public Execute {
 public:
  HashJoinExecutor(int32_t join_type, std::shared_ptr<Execute> input_l, std::shared_ptr<Execute> input_r, JoinParams params_l,
                   JoinParams params_r, std::vector<uint8_t> null_safe, std::vector<int32_t> output_indices = {},
                   rw_join_cond cond = rw_join_cond{RW_CMP_NONE, 0, 0, 0}, bool is_append_only = false, int32_t chunk_size = 1024,
                   std::vector<std::pair<int, bool>> watermark_indices_in_jk = {})
      : in_{std::move(input_l), std::move(input_r)}, wm_in_jk_(std::move(watermark_indices_in_jk)) {
    std::vector<int32_t> nat;
    if (join_type == RW_JOIN_LEFT_SEMI || join_type == RW_JOIN_LEFT_ANTI) nat = in_[0]->schema();
    else if (join_type == RW_JOIN_RIGHT_SEMI || join_type == RW_JOIN_RIGHT_ANTI) nat = in_[1]->schema();
    else { nat = in_[0]->schema(); nat.insert(nat.end(), in_[1]->schema().begin(), in_[1]->schema().end()); }
    if (output_indices.empty()) for (size_t i = 0; i < nat.size(); i++) output_indices.push_back((int32_t)i);
    rw_join_desc d{};
    d.join_type = join_type;
    d.n_keys = (int32_t)params_l.join_key_indices.size();
    const JoinParams* ps[2] = {&params_l, &params_r};
    rw_join_side_desc* sd[2] = {&d.left, &d.right};
    for (int s = 0; s < 2; s++) {
      sd[s]->n_cols = (int32_t)in_[s]->schema().size();
      sd[s]->types = in_[s]->schema().data();
      sd[s]->key_indices = ps[s]->join_key_indices.data();
      sd[s]->n_pk = (int32_t)ps[s]->deduped_pk_indices.size();
      sd[s]->pk_indices = ps[s]->deduped_pk_indices.data();
      sd[s]->n_stream_key = (int32_t)in_[s]->stream_key().size();
      sd[s]->stream_key = in_[s]->stream_key().data();
    }
    d.null_safe = null_safe.data();
    d.n_output = (int32_t)output_indices.size();
    d.output_indices = output_indices.data();
    d.cond = cond;
    d.is_append_only = is_append_only;
    d.chunk_size = chunk_size;
    d.strict_consistency = 1;
    check(rwgpu_join_create(&d, &h_));
    for (int32_t i : output_indices) schema_.push_back(nat[i]);
    // i2o_mapping_indexed per side (input column -> output positions), for the watermarks
    const int32_t n_l = (int32_t)in_[0]->schema().size();
    const bool semi_l = join_type == RW_JOIN_LEFT_SEMI || join_type == RW_JOIN_LEFT_ANTI;
    const bool semi_r = join_type == RW_JOIN_RIGHT_SEMI || join_type == RW_JOIN_RIGHT_ANTI;
    for (size_t o = 0; o < output_indices.size(); o++) {
      const int32_t i = output_indices[o];
      if (semi_l || (!semi_r && i < n_l)) i2o_[0][i].push_back((int32_t)o);
      else i2o_[1][semi_r ? i : i - n_l].push_back((int32_t)o);
    }
    jk_[0] = params_l.join_key_indices;
    jk_[1] = params_r.join_key_indices;
  }
  // HashJoinExecutor::handle_watermark, the join-key part (hash_join.rs:791-842); inequality pairs stay on the CPU executor
  std::vector<Watermark> handle_watermark(int side, const Watermark& wm) {
    std::vector<Watermark> out;
    const int upd = side, mat = 1 - side;
    for (size_t idx = 0; idx < jk_[upd].size(); idx++) {
      if (jk_[upd][idx] != wm.col_idx) continue;
      auto it = wm_buffers_.find((int)idx);
      if (it == wm_buffers_.end()) it = wm_buffers_.emplace((int)idx, BufferedWatermarks({RW_SIDE_LEFT, RW_SIDE_RIGHT})).first;
      auto sel = it->second.handle_watermark(side, wm);
      if (!sel) continue;
      for (auto& pc : wm_in_jk_)
        if (pc.first == (int)idx && pc.second) {  // JoinHashMap::update_watermark on both sides, applied at the next barrier
          check(rwgpu_join_update_watermark(h_, mat, (int32_t)idx, sel->val));
          check(rwgpu_join_update_watermark(h_, upd, (int32_t)idx, sel->val));
          break;
        }
      for (int s2 : {upd, mat}) {
        auto f = i2o_[s2].find(jk_[s2][idx]);
        if (f == i2o_[s2].end()) continue;
        for (int32_t o : f->second) out.push_back(Watermark{o, sel->data_type, sel->val});
      }
    }
    return out;
  }
  ~HashJoinExecutor() override { rwgpu_join_destroy(h_); }
  // into_stream over barrier_align: a side that delivered its barrier is blocked until the other
  // side's barrier arrives; the left side is preferred (one legal schedule of barrier_align.rs:67)
  std::optional<Message> poll_next() override {
    while (true) {
      if (!pending_.empty()) { Message m = std::move(pending_.front()); pending_.pop_front(); return m; }
      bool progressed = false;
      for (int s = 0; s < 2 && !progressed; s++) {
        if (blocked_[s]) continue;
        auto m = in_[s]->poll_next();
        if (!m) continue;
        progressed = true;
        if (auto* c = std::get_if<StreamChunk>(&*m)) {
          auto v = c->view();
          rwgpu_out* out = nullptr;
          check(rwgpu_join_push(h_, s, &v.raw, &out));  // eq_join_oneside::<SIDE>
          for (auto& ch : take_out(out)) pending_.emplace_back(std::move(ch));
        } else if (auto* b = std::get_if<Barrier>(&*m)) {
          blocked_[s] = *b;
          if (blocked_[0] && blocked_[1]) {
            Barrier bar = *blocked_[0];
            blocked_[0].reset();
            blocked_[1].reset();
            check(rwgpu_join_barrier(h_, bar.epoch));
            pending_.emplace_back(bar);
          }
        } else if (auto* w = std::get_if<Watermark>(&*m)) {  // AlignedMessage::WatermarkLeft / Right (hash_join.rs:711-722)
          for (auto& o : handle_watermark(s, *w)) pending_.emplace_back(o);
        }
      }
      if (!progressed && pending_.empty()) return std::nullopt;
    }
  }
  const std::vector<int32_t>& schema() const override { return schema_; }
  const std::vector<int32_t>& stream_key() const override { return key_; }

 private:
  std::shared_ptr<Execute> in_[2];
  rwgpu_join* h_ = nullptr;
  std::optional<Barrier> blocked_[2];
  std::deque<Message> pending_;
  std::vector<int32_t> schema_, key_;
  std::vector<std::pair<int, bool>> wm_in_jk_;
  std::map<int32_t, std::vector<int32_t>> i2o_[2];
  std::vector<int32_t> jk_[2];
  std::map<int, BufferedWatermarks> wm_buffers_;
};

}  // namespace rwgpu
