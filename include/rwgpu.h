/*
 * rwgpu.h -- C ABI of the H100-native streaming HashAgg / HashJoin / hash-shuffle path.
 *
 * The reference (risingwavelabs/risingwave) has NO extern "C" surface on this path: the
 * operators are Rust types behind `trait Execute` (src/stream/src/executor/mod.rs:240-253)
 * built by `ExecutorBuilder::new_boxed_executor` (src/stream/src/from_proto/mod.rs:131-140).
 * This header is therefore what a thin Rust shim (`GpuHashAggExecutor` / `GpuHashJoinExecutor`,
 * see INTEGRATION.md) binds with `extern "C"`; every entry point cites the reference
 * function whose work it replaces.
 *
 * Conventions
 *  - every function returns an int32 status (RW_OK == 0); `rwgpu_last_error()` gives a
 *    thread-local message.  No exceptions / longjmp cross the boundary.
 *  - a handle is single-owner (one actor == one tokio task polls it; actor.rs:272); different
 *    handles may be used concurrently from different threads.
 *  - input chunks are BORROWED for the duration of the call; output objects are LIBRARY-OWNED
 *    until `rwgpu_out_release`.
 *  - all layouts are little-endian; bitmaps are uint64 words, LSB first
 *    (bit i = words[i/64] >> (i%64) & 1, src/common/src/bitmap.rs:363-369); a NULL bitmap
 *    pointer means "all ones" (Bitmap.bits == None, bitmap.rs:220-224).
 */
#ifndef RWGPU_H_
#define RWGPU_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- status codes */
#define RW_OK 0
#define RW_ERR_INVALID 1       /* bad argument / malformed descriptor                          */
#define RW_ERR_UNSUPPORTED 2   /* plan shape not offloadable: shim falls back to CPU executor */
#define RW_ERR_OOM 3
#define RW_ERR_NUMERIC_OUT_OF_RANGE 4 /* ExprError::NumericOutOfRange (general.rs:32-40)       */
#define RW_ERR_INCONSISTENT 5  /* strict-consistency violation (src/stream/src/lib.rs:58-127)  */
#define RW_ERR_CUDA 6
#define RW_ERR_NO_DEVICE 7

/* ---------------------------------------------------------------- Op (stream_chunk.rs:84-91, to_i16) */
#define RW_OP_INSERT 1
#define RW_OP_DELETE 2
#define RW_OP_UPDATE_INSERT 3
#define RW_OP_UPDATE_DELETE 4

/* ---------------------------------------------------------------- column types.  Fixed-width types everywhere; the
 * two VARLEN types (BytesArray{offset, bitmap, data}, src/common/src/array/bytes_array.rs:30-34) cross the ABI as
 * PAYLOAD: a join carries them from input to output (stored in a per-side byte heap in HBM), HashAgg / Filter /
 * Project ignore columns they do not reference.  A varlen column cannot be a join key, a pk column, a group key, an
 * aggregate argument or a predicate operand here (`KeySerialized` keys stay on the CPU executor, SURVEY §8a).   */
#define RW_T_BOOL 1        /* 1 byte / row (BoolArray bit-unpacked by the shim)         */
#define RW_T_INT16 2
#define RW_T_INT32 3
#define RW_T_INT64 4
#define RW_T_FLOAT32 5
#define RW_T_FLOAT64 6
#define RW_T_DATE 7        /* int32 days                                               */
#define RW_T_TIME 8        /* int64 microseconds                                       */
#define RW_T_TIMESTAMP 9   /* int64 microseconds since epoch                           */
#define RW_T_TIMESTAMPTZ 10/* int64 microseconds                                       */
#define RW_T_SERIAL 11     /* int64 row id                                             */
#define RW_T_DECIMAL 12    /* 16 bytes: little-endian two's-complement i128 mantissa,
                              scale fixed per column by agreement (SURVEY §8b)          */
#define RW_T_VARCHAR 13    /* varlen: offsets[n_rows + 1] (uint32) into `data` bytes   */
#define RW_T_BYTEA 14      /* varlen, same layout                                      */

/* width in bytes of one value of a fixed-width `type`; 0 if unknown or varlen */
int32_t rwgpu_type_width(int32_t type);

/* ---------------------------------------------------------------- StreamChunk view
 * mirrors StreamChunk{ops, DataChunk{columns, visibility}} (stream_chunk.rs:106-110,
 * data_chunk.rs:65-68) and PrimitiveArray{bitmap,data} (primitive_array.rs:137-140). */
typedef struct rw_column {
  int32_t type;              /* RW_T_*                                                  */
  int32_t reserved;
  const void* data;          /* n_rows * width bytes; NULL slots hold any value.  Varlen: the bytes */
  const uint64_t* validity;  /* 1 = non-NULL; NULL pointer = no NULLs                   */
  const uint32_t* offsets;   /* varlen types only: value i = data[offsets[i] .. offsets[i+1]); else NULL.
                                offsets[0] need not be 0 (chunk views cut from one buffer share `data`) */
} rw_column;

typedef struct rw_chunk {
  int64_t n_rows;            /* capacity(): rows incl. invisible ones                   */
  int32_t n_cols;
  int32_t reserved;
  const uint8_t* ops;        /* RW_OP_* per row                                         */
  const uint64_t* visibility;/* NULL = all visible                                      */
  const rw_column* columns;
} rw_chunk;

/* ---------------------------------------------------------------- output object */
typedef struct rwgpu_out rwgpu_out;
/* number of StreamChunks produced by the call that returned `out` (0 is legal). */
int32_t rwgpu_out_num_chunks(const rwgpu_out* out);
/* total rows (capacity) over all chunks. */
int64_t rwgpu_out_num_rows(const rwgpu_out* out);
/* fill `view` with host pointers valid until rwgpu_out_release(out). */
int32_t rwgpu_out_chunk(const rwgpu_out* out, int32_t idx, rw_chunk* view);
void rwgpu_out_release(rwgpu_out* out);

/* ================================================================ HashAgg ===================
 * replaces HashAggExecutor (src/stream/src/executor/aggregate/hash_agg.rs):
 *   rwgpu_agg_push   <-> apply_chunk            hash_agg.rs:332-409
 *   rwgpu_agg_flush  <-> flush_data at barrier  hash_agg.rs:412-514, 651-676
 * Offloaded states (agg_state.rs:49-56): the value states count, sum, and min/max on append-only input, and
 * -- is_append_only == 0 -- RETRACTABLE min/max, the reference's MaterializedInput state (minput.rs): the call's
 * non-NULL input values are kept as a chained multiset in HBM; a retraction kills one record, and if it was the
 * group's extreme the barrier recomputes it from the live records.  string_agg / array_agg / DISTINCT / EOWC
 * => RW_ERR_UNSUPPORTED.  (The value log only grows between restarts; 2^31 values per operator.)            */
#define RW_AGG_COUNT 1     /* count(*) when arg_col < 0, else count(col)   general.rs:155-162 */
#define RW_AGG_SUM 2       /* general.rs:28-41                                                 */
#define RW_AGG_MIN 3       /* general.rs:91-108 (append-only) / minput.rs (retractable)        */
#define RW_AGG_MAX 4       /* general.rs:110-125 (append-only) / minput.rs (retractable)       */
#define RW_AGG_SUM0 5      /* sum0(int8)->int8, init 0     general.rs:28                      */

typedef struct rw_agg_call {
  int32_t kind;       /* RW_AGG_*                                                        */
  int32_t arg_col;    /* input column index, -1 for count(*)                             */
  int32_t ret_type;   /* RW_T_*: sum(int2|int4)->INT64, sum(int8)->DECIMAL (scale 0) or the
                         internal sum(int8)->INT64 form; sum(float)->same float; count->INT64;
                         min/max -> arg type                                             */
  int32_t reserved;
} rw_agg_call;

typedef struct rw_agg_desc {
  int32_t n_input_cols;
  const int32_t* input_types;       /* RW_T_* per input column                            */
  int32_t n_group_keys;
  const int32_t* group_key_indices; /* hash_agg.rs:338                                    */
  int32_t n_calls;
  const rw_agg_call* calls;
  int32_t row_count_index;          /* index into calls of the count(*) used by
                                       OnlyOutputIfHasInput (agg_group.rs:131-166)        */
  int32_t is_append_only;           /* input has no Delete/UpdateDelete                   */
  int32_t chunk_size;               /* output chunk rows (config/mod.rs:213-215)          */
  int32_t strict_consistency;       /* 1: negative row count => RW_ERR_INCONSISTENT
                                       (agg_group.rs:55-79); 0: clamp to 0               */
  uint64_t group_capacity_hint;     /* expected distinct groups (table grows on demand)   */
} rw_agg_desc;

typedef struct rwgpu_agg rwgpu_agg;

int32_t rwgpu_agg_create(const rw_agg_desc* desc, rwgpu_agg** out_handle);
void rwgpu_agg_destroy(rwgpu_agg* h);
/* HOST chunk: staged into pinned memory, copied H2D and applied asynchronously on the handle's
 * stream; rows are coalesced across calls into one device batch until flush (SURVEY §7.2). */
int32_t rwgpu_agg_push(rwgpu_agg* h, const rw_chunk* chunk);
/* DEVICE chunk: every pointer inside `chunk` (ops, visibility, column data/validity) is a device
 * pointer; the rw_chunk/rw_column structs themselves are host memory.  The kernel is enqueued on
 * `cuda_stream` (a cudaStream_t; NULL = the handle's own stream) and the call does not sync.  */
int32_t rwgpu_agg_push_device(rwgpu_agg* h, const rw_chunk* chunk, void* cuda_stream);
/* barrier: emit one +, - or U-/U+ pair per changed group, outputs copied to host. */
int32_t rwgpu_agg_flush(rwgpu_agg* h, uint64_t epoch, rwgpu_out** out);
/* barrier with the delta left in HBM: `view` receives DEVICE pointers to one un-cut chunk
 * (valid until the next flush on this handle); *n_rows is read back (one 8-byte D2H).       */
int32_t rwgpu_agg_flush_device(rwgpu_agg* h, uint64_t epoch, rw_chunk* view, void* cuda_stream);
/* the same barrier split in two, so that a caller never waits for the GPU between a barrier and the next epoch's
 * pushes: `_async` only ENQUEUES the delta computation (one launch on `cuda_stream`, nothing is waited for);
 * `_collect` waits for the OLDEST outstanding barrier and returns its delta like rwgpu_agg_flush_device.  At most two
 * barriers may be outstanding (two output sets); a view stays valid until the second `_async` after its own.  All
 * work of one handle forms ONE logical stream: a call on another cuda_stream than the previous call's is ordered
 * behind it on the device (event), whichever streams are used.                                                */
int32_t rwgpu_agg_flush_device_async(rwgpu_agg* h, uint64_t epoch, void* cuda_stream);
int32_t rwgpu_agg_flush_collect(rwgpu_agg* h, rw_chunk* view, void* cuda_stream);
/* ---- state persistence (checkpoint / recovery).  What the reference persists per group is the INTERMEDIATE STATE row
 * `group key | one state datum per call` (AggGroup::build_states_change, agg_group.rs:473-538; a group whose row count
 * is 0 has no row) and, per retractable min / max call, the rows of its materialized input (minput.rs); on recovery
 * AggGroup::create (agg_group.rs:260-316) loads the row and derives prev_outputs from it.
 *   rwgpu_agg_snapshot: between a barrier and the next push.  `*states`: all-Insert chunks, schema = the operator's
 *     OUTPUT schema (group key columns, then per call its state datum: count int8, sum in its return type, min / max
 *     in the argument type; NULL = no input yet).  `*minput`: group key columns | int4 call index | int8 value (float
 *     arguments: the IEEE-754 bits of the f64), one row per live input value of a retractable min / max (0 rows
 *     otherwise).  The shim hands both to StateTable::write_chunk, which does the value / memcomparable encoding and
 *     the vnode prefix (state_table.rs:1451-1560).  Release both with rwgpu_out_release.
 *   rwgpu_agg_restore: into an idle operator; chunks of the same two schemas (HOST).  Afterwards the operator emits
 *     exactly what the snapshotted one would.                                                                     */
int32_t rwgpu_agg_snapshot(rwgpu_agg* h, rwgpu_out** states, rwgpu_out** minput);
int32_t rwgpu_agg_restore(rwgpu_agg* h, const rw_chunk* states, const rw_chunk* minput);
/* number of groups currently held / table capacity (diagnostics, join_cached_entry_count-like) */
int32_t rwgpu_agg_stats(rwgpu_agg* h, uint64_t* n_groups, uint64_t* capacity, uint64_t* kernel_launches);
/* device-time accounting of the dominant kernel (the fused group-by + aggregate apply kernel):
 * enable != 0 starts bracketing every launch with CUDA events on the launching stream; the call
 * returns the accumulated milliseconds / launch count since the previous call and resets them
 * (feeds the `join_match_duration_ns`-style metrics, streaming_stats.rs:94-100, and bench.py).  */
int32_t rwgpu_agg_profile(rwgpu_agg* h, int32_t enable, double* kernel_ms, uint64_t* kernel_launches);

/* ================================================================ HashJoin ==================
 * replaces HashJoinExecutor (src/stream/src/executor/hash_join.rs):
 *   rwgpu_join_push    <-> eq_join_oneside::<SIDE>   hash_join.rs:925-1062 (+1072-1357)
 *   rwgpu_join_barrier <-> flush_data / commit       hash_join.rs:754-766                     */
#define RW_JOIN_INNER 0
#define RW_JOIN_LEFT_OUTER 1
#define RW_JOIN_RIGHT_OUTER 2
#define RW_JOIN_FULL_OUTER 3
#define RW_JOIN_LEFT_SEMI 4
#define RW_JOIN_LEFT_ANTI 5
#define RW_JOIN_RIGHT_SEMI 6
#define RW_JOIN_RIGHT_ANTI 7

#define RW_SIDE_LEFT 0
#define RW_SIDE_RIGHT 1

/* restricted non-equi condition: `concat_row[lhs] <cmp> concat_row[rhs]` over the
 * (left cols || right cols) row, compared as integers: both operands int2 / int4 / int8 (mixed
 * widths are fine), or both of one and the same other non-float, non-decimal, fixed-width type
 * (date with date, timestamp with timestamp ...).  Anything else -- float, decimal or varlen
 * operands, date against timestamp, bool against int -- makes create return RW_ERR_UNSUPPORTED
 * and stays on the CPU executor (hash_join.rs:1362-1384 evaluates a general expression).  Filter
 * terms follow the same rule.                                                                   */
#define RW_CMP_NONE 0
#define RW_CMP_LT 1
#define RW_CMP_LE 2
#define RW_CMP_GT 3
#define RW_CMP_GE 4
#define RW_CMP_EQ 5
#define RW_CMP_NE 6
typedef struct rw_join_cond {
  int32_t cmp;   /* RW_CMP_*                                       */
  int32_t lhs;   /* index into left||right concatenated columns    */
  int32_t rhs;
  int32_t reserved;
} rw_join_cond;

typedef struct rw_join_side_desc {
  int32_t n_cols;
  const int32_t* types;             /* RW_T_* per input column                               */
  const int32_t* key_indices;       /* JoinParams.join_key_indices (hash_join.rs:75-89)      */
  int32_t n_pk;
  const int32_t* pk_indices;        /* JoinParams.deduped_pk_indices                         */
  int32_t n_stream_key;
  const int32_t* stream_key;        /* input.stream_key(): decides pk_contained_in_jk
                                       (hash_join.rs:377-381)                               */
  uint64_t row_capacity_hint;       /* expected distinct join keys of this side (index grows on demand) */
  uint64_t stored_rows_hint;        /* expected rows STORED on this side (0 = two per expected key); the row store
                                       grows on demand, one 200 MB segment at a time                          */
} rw_join_side_desc;

typedef struct rw_join_desc {
  int32_t join_type;                /* RW_JOIN_*  (join/mod.rs:43-52)                        */
  int32_t n_keys;
  rw_join_side_desc left, right;
  const uint8_t* null_safe;         /* n_keys flags, IS NOT DISTINCT FROM (stream_plan.proto:639) */
  int32_t n_output;
  const int32_t* output_indices;    /* projection of the natural output (hash_join.rs:337-359) */
  rw_join_cond cond;                /* cmp == RW_CMP_NONE => no condition                    */
  int32_t is_append_only;           /* enables append_only_optimize when pk ⊆ jk both sides  */
  int32_t chunk_size;               /* output chunk rows, clamped to >= 2 (join/builder.rs:44-47) */
  int32_t strict_consistency;
  int32_t reserved;
} rw_join_desc;

typedef struct rwgpu_join rwgpu_join;

int32_t rwgpu_join_create(const rw_join_desc* desc, rwgpu_join** out_handle);
void rwgpu_join_destroy(rwgpu_join* h);
/* HOST chunk from `side`; `out` receives 0..k output chunks (host buffers).
 * ALIASING: for an inner join whose output is positional (output row r belongs to input row r), the
 * output columns that are plain copies of `chunk`'s columns are NOT shipped back over PCIe: the output
 * chunk views point into `chunk`'s own column buffers.  Keep `chunk`'s buffers alive and unmodified
 * until rwgpu_out_release(*out).                                                                   */
int32_t rwgpu_join_push(rwgpu_join* h, int32_t side, const rw_chunk* chunk, rwgpu_out** out);
/* DEVICE chunk; output left in HBM as one un-cut chunk `view` (device pointers, valid until the
 * next push on this handle).  *view.n_rows is read back (one 8-byte D2H).
 * ALIASING: when the output is positional (output row r belongs to input row r) the view's columns
 * that are plain copies of `chunk`'s columns may point into `chunk`'s own device buffers instead of
 * a copy.  Keep `chunk`'s buffers alive and unmodified for as long as the view is used: until the
 * next push on this handle (for the _async / collect pair below: until the second _async after
 * the push).  A chunk with a device-resident row count is never aliased.                      */
int32_t rwgpu_join_push_device(rwgpu_join* h, int32_t side, const rw_chunk* chunk, rw_chunk* view,
                               void* cuda_stream);
/* same, for a chunk whose row count is produced ON THE DEVICE by earlier work of `cuda_stream` (the
 * exchange's unpack kernel): chunk->n_rows is the capacity of its buffers, *n_rows_dev (DEVICE int64,
 * 0 <= *n_rows_dev <= n_rows) the rows to process.  No host round trip between producer and join.
 * n_rows_dev == NULL behaves like rwgpu_join_push_device.                                     */
int32_t rwgpu_join_push_device_counted(rwgpu_join* h, int32_t side, const rw_chunk* chunk,
                                       const int64_t* n_rows_dev, rw_chunk* view, void* cuda_stream);
/* LAUNCH / COLLECT split of rwgpu_join_push_device_counted, so that the caller never sits between two launches:
 * `_async` only ENQUEUES the push on `cuda_stream` (n_rows_dev may be NULL) and returns; `rwgpu_join_collect` waits
 * for the OLDEST outstanding push and returns its output like the synchronous call.  Rules:
 *  - at most two pushes outstanding (two output sets); a view stays valid until the second `_async` after its own;
 *  - `chunk`'s DEVICE buffers (and *n_rows_dev) stay valid and unmodified until the push is collected, and as long as
 *    its view is used when the view aliases them (see rwgpu_join_push_device);
 *  - pushes of DIFFERENT sides are never outstanding together (RW_ERR_INVALID): a side's probe reads the other side's
 *    state, and the collect step may have to re-run that probe when the output area was too small;
 *  - errors of the push (RW_ERR_INCONSISTENT ...) are reported by its collect;
 *  - all work of one handle is ONE logical stream: a call on another cuda_stream than the previous call's is ordered
 *    behind it on the device.
 * Plan shapes without an asynchronous kernel path complete inside `_async`; the protocol is the same.           */
int32_t rwgpu_join_push_device_async(rwgpu_join* h, int32_t side, const rw_chunk* chunk, const int64_t* n_rows_dev,
                                     void* cuda_stream);
int32_t rwgpu_join_collect(rwgpu_join* h, rw_chunk* view, void* cuda_stream);
/* The same split for HOST chunks -- what the executor shim uses per message (INTEGRATION.md section 9): the launch
 * enqueues the input's H2D copy, the push, and the D2H copy of the positional output rows (one per input row: the
 * common case) on three streams and returns; while the caller launches the NEXT chunk (its input travels host -> device)
 * this chunk's output travels device -> host, so both PCIe directions stay busy across calls (rwgpu_join_push overlaps
 * them only inside one call).  `rwgpu_join_collect_out` waits for the OLDEST outstanding push, copies what the status
 * block says is still missing (extra matches, NULL / visibility bytes) and returns the rwgpu_out (release it as usual).
 * Rules as above (two outstanding, one side, errors at collect), and
 *  - the chunk's HOST buffers stay valid and unmodified until the push is collected -- and, when output columns alias
 *    them (see rwgpu_join_push), until the rwgpu_out is released;
 *  - device-chunk and host-chunk pushes each have their own collect call; collect them in launch order.
 * Plan shapes without an asynchronous kernel path (and chunks with varlen payload) complete inside the launch.  */
int32_t rwgpu_join_push_async(rwgpu_join* h, int32_t side, const rw_chunk* chunk);
int32_t rwgpu_join_collect_out(rwgpu_join* h, rwgpu_out** out);
int32_t rwgpu_join_barrier(rwgpu_join* h, uint64_t epoch);
int32_t rwgpu_join_stats(rwgpu_join* h, uint64_t* left_rows, uint64_t* right_rows,
                         uint64_t* kernel_launches);
/* Watermark-driven state cleaning (HashJoinExecutor::handle_watermark, hash_join.rs:791-891 -> JoinHashMap::
 * update_watermark): the host keeps the BufferedWatermarks logic (take the smaller of the two sides' watermarks,
 * derive the output watermarks) and tells the operator which side's state may drop every row whose join key column
 * `key_pos` is below `value` (integer-typed key columns).  Like the reference's state table the rows leave at the next
 * rwgpu_join_barrier.  By the watermark contract no later row can match them, so results are unchanged; the
 * state stops growing.                                                                                     */
int32_t rwgpu_join_update_watermark(rwgpu_join* h, int32_t side, int32_t key_pos, int64_t value);
/* ---- state persistence (checkpoint / recovery).  A side's persistent state is the set of its stored input rows: the
 * reference writes every stored row to the side's StateTable (JoinHashMap::insert, join/hash_join.rs:591-625; table
 * pk = join key | deduped input pk, stream_plan.proto:628-637), so on the write path the shim passes the INPUT chunks
 * on to StateTable::write_chunk exactly as the CPU executor does -- nothing has to come back from the GPU.
 *   rwgpu_join_snapshot: the live rows of `side` as all-Insert chunks in the side's input schema (for a checkpoint of
 *     an operator that was running without a StateTable, and for moving state when vnodes are re-assigned).
 *   rwgpu_join_restore: replays state rows (HOST chunk) as inserts with the output discarded -- restore BOTH sides;
 *     the incremental algorithm itself re-derives the degrees of outer / semi / anti joins.                        */
int32_t rwgpu_join_snapshot(rwgpu_join* h, int32_t side, rwgpu_out** rows);
int32_t rwgpu_join_restore(rwgpu_join* h, int32_t side, const rw_chunk* rows);
/* State reclamation: a delete marks the stored row dead; rwgpu_join_barrier rebuilds a side's row log from its live
 * rows once more than half of it is dead (the reference frees the entry at delete time, join/hash_join.rs:659-681).
 * -> number of such rebuilds so far (diagnostics).  State-lifetime limit: a side holds < 2^31 - 16 log rows between
 * two rebuilds (RW_ERR_OOM beyond).                                                                      */
uint64_t rwgpu_join_compactions(rwgpu_join* h);
/* TEST HOOK: set the operator's arrival counter (rows pushed so far, both sides).  Stored rows carry their 64-bit
 * arrival number; the own-side delete rule compares them.  Tests move the counter next to 2^31 / 2^32 to pin
 * the behaviour across those boundaries without pushing billions of rows.                              */
int32_t rwgpu_join_debug_set_seq(rwgpu_join* h, uint64_t seq);
/* same as rwgpu_agg_profile for the join's dominant kernel (probe + emit). */
int32_t rwgpu_join_profile(rwgpu_join* h, int32_t enable, double* kernel_ms, uint64_t* kernel_launches);

/* ================================================================ hash shuffle ==============
 * replaces VirtualNode::compute_chunk (src/common/src/hash/consistent_hash/vnode.rs:151-182)
 * and the routing half of HashDataDispatcher::dispatch_data (src/stream/src/executor/
 * dispatch.rs:961-1053).  vnode = crc32(IEEE, bytes of key datums) % vnode_count.             */
/* HOST: vnode per row (invisible rows still get a value, as in the reference).               */
int32_t rwgpu_vnode_compute(const rw_chunk* chunk, const int32_t* key_indices, int32_t n_keys,
                            int32_t vnode_count, uint16_t* out_vnodes);
/* HOST: the op rewrite of dispatch.rs:976-1023 (U-/U+ whose dist key changed -> -/+).  Over the visible rows, a U+
 * pairs with the last U- that no earlier U+ has taken, whatever + / - rows lie between them; a U- that a later U-
 * replaces before any U+ keeps its op.  The key compares as a Datum (NULL == NULL, -0 == +0, every NaN equal).
 * RW_ERR_INCONSISTENT: a U+ with no U- to take ("missing U- before U+"), or a U- that no U+ follows anywhere in the
 * chunk ("missing U+ after U-").  Invisible rows keep their op.  Key arguments as for rwgpu_vnode_compute.      */
int32_t rwgpu_dispatch_rewrite_ops(const rw_chunk* chunk, const int32_t* key_indices, int32_t n_keys,
                                   uint8_t* out_ops);
/* DEVICE: partition the visible rows of a device chunk by destination
 *   dest = vnode_to_dest[vnode]   (vnode_to_dest: DEVICE array of vnode_count int32)
 * into per-destination contiguous regions of caller-provided DEVICE output columns
 * (same types as input; capacity n_rows each), ops included; counts[n_dest] / offsets[n_dest]
 * are DEVICE int64 arrays.  This is the send-side of the NCCL all-to-all-v that replaces the
 * Dispatch/Exchange pair for the hash-shuffle path.                                          */
int32_t rwgpu_shuffle_partition_device(const rw_chunk* chunk, const int32_t* key_indices,
                                       int32_t n_keys, int32_t vnode_count,
                                       const int32_t* vnode_to_dest, int32_t n_dest,
                                       uint8_t* out_ops, void* const* out_cols,
                                       uint8_t* const* out_valid_bytes, /* 1 byte/row, may be NULL */
                                       int64_t* counts, int64_t* offsets, void* cuda_stream);

/* ---- fused partition + transfer over NVLink peer memory (no NCCL call on the data path) ----------------
 * Every rank owns a receive buffer of n_rank REGIONS (one per source rank), symmetric across ranks and
 * peer-mapped (e.g. torch.distributed._symmetric_memory); region = [256 B header: int64 row count]
 * [ops: cap_rows bytes][column k: cap_rows * width_k], each 256-B aligned.                              */
int32_t rwgpu_shuffle_p2p_region_bytes(const int32_t* types, int32_t n_cols, int64_t cap_rows,
                                       int64_t* region_bytes);
/* sender: stable-partition the visible rows of a DEVICE chunk by destination and store them straight into
 * region `my_rank` of each destination's buffer (`peer_bases`: HOST array of n_dest peer-mapped device
 * pointers), then publish the row counts in the region headers.  `counts`: DEVICE int64[n_dest];
 * `overflow`: DEVICE int32 set to 1 if some (src,dst) pair exceeded cap_rows (rows beyond it are dropped and the
 * receiver's total reads -1): size cap_rows for the worst case -- every row of a source batch going to ONE
 * destination -- and it cannot happen.  Columns with validity bitmaps => RW_ERR_UNSUPPORTED (the regions carry ops
 * and column data only).  The caller runs a cross-rank barrier on the same stream before anybody unpacks.   */
int32_t rwgpu_shuffle_partition_p2p_device(const rw_chunk* chunk, const int32_t* key_indices, int32_t n_keys,
                                           int32_t vnode_count, const int32_t* vnode_to_dest, int32_t n_dest,
                                           int32_t my_rank, void* const* peer_bases, int64_t cap_rows,
                                           int64_t* counts, int32_t* overflow, void* cuda_stream);
/* receiver: concatenate the n_src regions of `recv_base` (source-rank order, row order preserved) into
 * contiguous DEVICE ops / columns; *total (DEVICE int64) receives the row count.                         */
int32_t rwgpu_shuffle_unpack_device(const void* recv_base, int32_t n_src, const int32_t* types, int32_t n_cols,
                                    int64_t cap_rows, uint8_t* out_ops, void* const* out_cols, int64_t* total,
                                    void* cuda_stream);

/* one call = one batch of the exchange: partition + peer stores + count publication (as above), a
 * cross-rank barrier, and the unpack -- five launches on `cuda_stream`, no library call in between.
 *   peer_flags : HOST array of n_dest peer-mapped device pointers to each rank's flag block
 *                (1024 bytes, zero-initialised, symmetric: uint64 flag[64] + scratch); the barrier of batch `epoch` (1, 2, ...
 *                strictly increasing per flag array) stores `epoch` into slot my_rank of every rank's
 *                array and waits until every slot of its own array holds >= epoch.
 *   recv_base  : this rank's receive buffer (== peer_bases[my_rank]).
 *                The DEVICE copy of the unpacked row count is the int64 at byte 512 + 8 * (epoch & 1) of this
 *                rank's flag block (feed it to rwgpu_join_push_device_counted: no host round trip).
 *   total_host : PINNED host int64 (device-addressable): receives the row count (-1 = a region
 *                overflowed) when the unpack kernel has run; the caller waits on the stream / an event. */
int32_t rwgpu_shuffle_exchange_p2p_device(const rw_chunk* chunk, const int32_t* key_indices, int32_t n_keys,
                                          int32_t vnode_count, const int32_t* vnode_to_dest, int32_t n_dest,
                                          int32_t my_rank, void* const* peer_bases, void* const* peer_flags,
                                          uint64_t epoch, int64_t cap_rows, const void* recv_base,
                                          uint8_t* out_ops, void* const* out_cols, int64_t* counts,
                                          int32_t* overflow, int64_t* total_host, void* cuda_stream);

/* ---- the exchange as ONE kernel, rows stored straight into their final place ------------------
 * Flat receive buffer (symmetric, peer-mapped, two alternate): [header: int64 M[64][64], M[s][d] = rows source s sends
 * to destination d][ops: cap_rows bytes][column k: cap_rows * width_k], parts 256-B aligned (rwgpu_shuffle_flat_layout
 * returns the offsets).  One launch per batch: per-block histograms -> scan -> every source writes its count row into
 * every rank's header -> cross-rank barrier -> every source scatters its rows over NVLink to
 *     first row of (s -> d) = sum of M[s'][d] over s' < s        (source-rank order, row order kept inside a source)
 * -> cross-rank barrier -> the received row count is stored to *total_dev (DEVICE int64, feed it to
 * rwgpu_join_push_device_counted / _async) and, if given, *total_host (pinned).  Nothing is unpacked: the consumer
 * reads ops / columns of the buffer in place.  Size cap_rows = n_dest x (rows per batch): no batch can overflow.
 *   peer_bases : HOST array of n_dest peer-mapped pointers to THIS batch's receive buffer of every rank
 *   peer_flags : as for rwgpu_shuffle_exchange_p2p_device; batch `epoch` (1, 2, ...) uses the values 2*epoch-1, 2*epoch
 *   err        : DEVICE int32, bit 0 = a destination buffer was too small, bit 1 = a peer did not reach the barrier
 *                within ~10 s (the count then reads -1)
 *   max_blocks : 0 = as many blocks as are co-resident; > 0 caps the grid (several ranks sharing one device in tests)
 * The kernel meets in grid-wide barriers of its own (plain launch, grid sized to be resident: at most three blocks per SM),
 * so at most TWO exchange launches may be in flight on one device at a time (different plans on different streams); a third
 * could keep the others' remaining blocks off the SMs.
 * Caller contract: batch e is launched after this rank's consumer of batch e - 2 (same buffer) has finished; that is
 * all the cross-rank ordering needed -- a peer writes into the buffer only after barrier 1 of batch e, which this
 * rank enters inside its own launch.  Replaces dispatch.rs:961-1053 + the exchange channel + merge for N GPUs.     */
int32_t rwgpu_shuffle_flat_layout(const int32_t* types, int32_t n_cols, int64_t cap_rows, int64_t* total_bytes,
                                  int64_t* ops_off, int64_t* col_off /* [n_cols] */);
int32_t rwgpu_shuffle_exchange_flat_device(const rw_chunk* chunk, const int32_t* key_indices, int32_t n_keys,
                                           int32_t vnode_count, const int32_t* vnode_to_dest, int32_t n_dest,
                                           int32_t my_rank, void* const* peer_bases, void* const* peer_flags,
                                           uint64_t epoch, int64_t cap_rows, int64_t* counts, int32_t* err,
                                           int64_t* total_dev, int64_t* total_host, int32_t max_blocks,
                                           void* cuda_stream);

/* ================================================================ Filter (operator chaining on the device)
 * Replaces FilterExecutorInner::filter           src/stream/src/executor/filter.rs:58-150
 * for predicates that are a CONJUNCTION of integer comparisons `col cmp col` / `col cmp constant`,
 * compared as raw integers under the operand rule of join conditions (above): int2 / int4 / int8
 * mix, and bool, serial, date, time, timestamp and timestamptz compare only with themselves; a
 * constant has the left operand's type.  Any other pair (date against timestamp, bool against int8,
 * a float, decimal or varlen operand) is RW_ERR_UNSUPPORTED and stays on the CPU FilterExecutor, as
 * does everything else the expression framework can evaluate.  A bad comparison or column index is
 * RW_ERR_INVALID.  A NULL operand makes its term NULL and the row's result false (filter.rs:79
 * `res.unwrap_or(false)`).  Project with InputRef expressions (project_scalar.rs:100-120) is a
 * re-ordering of column pointers in the caller and needs no kernel.
 *
 * Output: out_ops[n_rows] and the packed visibility out_visibility[(n_rows+63)/64] of a chunk that
 * has the input's columns; every word is written, the bits past n_rows zero.  Rows that were
 * invisible in the input -- a cleared visibility bit or op 0 -- stay invisible with their op
 * unchanged (the reference compacts them away first, filter.rs:182); the visible rows carry exactly
 * the ops / visibility the reference produces, U-/U+ pairs included (filter.rs:107-141).  A visible
 * U- pairs with the next visible row only if that row is a U+; a U- or U+ without its partner (which
 * well-formed streams never carry) is filtered like a - or + and keeps its op.  upsert != 0 selects
 * the UPSERT rules (filter.rs:82-106).  *n_visible (may be NULL) receives the number of visible
 * output rows (0 => the reference yields no chunk, filter.rs:146-150).  rwgpu_filter_device reads
 * neighbouring rows' input ops and visibility while it writes: outputs that alias the chunk's ops
 * or visibility are RW_ERR_INVALID.                                                               */
typedef struct rw_filter_term {
  int32_t cmp;       /* RW_CMP_LT .. RW_CMP_NE                                  */
  int32_t lhs_col;
  int32_t rhs_col;   /* >= 0: column; -1: rhs_const                             */
  int32_t reserved;
  int64_t rhs_const;
} rw_filter_term;
/* HOST chunk, host outputs */
int32_t rwgpu_filter(const rw_chunk* chunk, const rw_filter_term* terms, int32_t n_terms, int32_t upsert,
                     uint8_t* out_ops, uint64_t* out_visibility, int64_t* n_visible);
/* DEVICE chunk (e.g. the view a join push returned), DEVICE outputs; *n_visible_dev: DEVICE int64 or NULL */
int32_t rwgpu_filter_device(const rw_chunk* chunk, const rw_filter_term* terms, int32_t n_terms, int32_t upsert,
                            uint8_t* out_ops, uint64_t* out_visibility, int64_t* n_visible_dev,
                            void* cuda_stream);

/* ================================================================ Project (operator chaining on the device)
 * Replaces apply_project_exprs                   src/stream/src/executor/project/project_scalar.rs:91-108
 * for INTEGER expressions in postfix form.  An InputRef projection needs no call at all (re-order the column
 * pointers).  Evaluation is non-strict like the reference's (`eval_infallible`): a NULL operand, a numeric overflow
 * (checked_add / checked_sub / checked_mul / checked_div / checked_neg of the OPERATION's result type), MIN % -1
 * (checked_rem) or a division by zero makes the ROW's value NULL, never an error.  Ops and visibility of the chunk
 * pass through unchanged.
 *   RW_EX_COL    push column `arg` (Int16/32/64, Date, Time, Timestamp(tz), Serial)      RW_EX_CONST  push `value`
 *   RW_EX_ADD / SUB / MUL / DIV / MOD (b = pop, a = pop, push a op b; Rust semantics: truncating /, sign of a for %)
 *   RW_EX_NEG    RW_EX_TUMBLE_START / RW_EX_TUMBLE_END  (a = timestamp in us, or a DATE operand (days), which becomes
 *                the timestamp of its midnight; b = window in us; tumble.rs:34-112)
 * Every operator (RW_EX_ADD..RW_EX_NEG) carries its result type in `arg`: an integer-typed RW_T_*, 0 = RW_T_INT64.
 * The result of the operation must fit that type (Int16 / Int32 / Date: 2 / 4 / 4 bytes, the others 8), else the row is
 * NULL.  An `arg` that is no RW_T_* is RW_ERR_INVALID.  The device evaluates at most 16 expressions of at most 24
 * operations and a stack depth of 8 (RW_ERR_UNSUPPORTED beyond).
 * Everything else the expression framework can evaluate stays on the CPU ProjectExecutor.                       */
#define RW_EX_COL 1
#define RW_EX_CONST 2
#define RW_EX_ADD 3
#define RW_EX_SUB 4
#define RW_EX_MUL 5
#define RW_EX_DIV 6
#define RW_EX_MOD 7
#define RW_EX_TUMBLE_START 8
#define RW_EX_TUMBLE_END 9
#define RW_EX_NEG 10
typedef struct rw_expr_op {
  int32_t op;     /* RW_EX_*                         */
  int32_t arg;    /* RW_EX_COL: input column; operator: result RW_T_* (0 = INT64) */
  int64_t value;  /* RW_EX_CONST                     */
} rw_expr_op;
typedef struct rw_project_expr {
  const rw_expr_op* ops;  /* postfix program, leaves exactly one value */
  int32_t n_ops;
  int32_t ret_type;       /* RW_T_* (integer-typed)                    */
} rw_project_expr;
/* HOST chunk; out_data[e]: n_rows values of expression e; out_validity[e]: (n_rows+63)/64 words, written only when
 * has_null[e] comes back non-zero (else every value is non-NULL).                                              */
int32_t rwgpu_project(const rw_chunk* chunk, const rw_project_expr* exprs, int32_t n_exprs, void* const* out_data,
                      uint64_t* const* out_validity, uint32_t* has_null);
/* DEVICE chunk, DEVICE outputs: out_valid_bytes[e] = 1 byte per row (1 = non-NULL), has_null = DEVICE uint32[n_exprs]. */
int32_t rwgpu_project_device(const rw_chunk* chunk, const rw_project_expr* exprs, int32_t n_exprs, void* const* out_data,
                             uint8_t* const* out_valid_bytes, uint32_t* has_null, void* cuda_stream);

/* ================================================================ misc */
const char* rwgpu_last_error(void);
/* 0 if a CUDA device is usable, else RW_ERR_NO_DEVICE (and every create() fails loudly). */
int32_t rwgpu_device_check(void);
/* "rwgpu <version> sm_90a" */
const char* rwgpu_version(void);

#ifdef __cplusplus
}
#endif
#endif /* RWGPU_H_ */
