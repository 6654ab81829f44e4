// libb200exec host side: the GPU ExecutionEngine / QueryStageExecutor.
//
// Mirrors (reference file:line):
//   DefaultExecutionEngine::create_query_stage_exec     ballista/executor/src/execution_engine.rs:106-169
//   DefaultQueryStageExec::execute_query_stage          ballista/executor/src/execution_engine.rs:235-254
//   ShuffleWriterExec::execute_shuffle_write            ballista/core/src/execution_plans/shuffle_writer.rs:203-402
//   SortShuffleWriterExec::execute_shuffle_write        ballista/core/src/execution_plans/sort_shuffle/writer.rs:199-373
//   ShuffleReaderExec::execute                          ballista/core/src/execution_plans/shuffle_reader.rs:248-318
//   collect_plan_metrics                                ballista/core/src/utils.rs:328-339
// The operator tree below the writer (FilterExec/ProjectionExec/AggregateExec/HashJoinExec/SortExec,
// DataFusion 53.1 [EXT]) is executed by the CUDA kernels in csrc/device.  There is no CPU path:
// every operator either runs on the GPU or fails with B200_ERR_UNSUPPORTED.
#include <sched.h>
#include <sys/stat.h>

#include <algorithm>
#include <atomic>
#include <cctype>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <map>
#include <mutex>
#include <functional>
#include <set>

#include "../common/arrow_host.hpp"
#include "../common/tpch_gen.hpp"
#include "../device/kernels.h"
#include "host_pool.hpp"
#include "lower.hpp"
#include "nccl_dyn.hpp"
#include "../common/plan_proto.hpp"
#include "../common/plan_dump.hpp"
#include "parquet_meta.hpp"
#include "arrow_ipc.hpp"
#include "shuffle_store.hpp"

using namespace b200;

namespace {

thread_local std::string g_err;

struct OpMetrics {
  std::string name;
  uint64_t output_rows = 0, input_rows = 0, elapsed_ns = 0, bytes_read = 0, bytes_written = 0, launches = 0;
};

}  // namespace

struct b200_engine {
  int device = 0;
  int rank = 0, world = 1;
  int sm_count = 132;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  std::map<std::string, std::map<int, DevBatchPtr>> tables;
  ShuffleStore shuffle;                      // its own lock: take mu first when both are held
  std::atomic<uint64_t> launches{0};
  std::atomic<uint64_t> n_fused{0}, n_fused_static{0}, n_vm{0}, n_groupby{0}, n_groupby_pf{0}, n_fastfilter{0};  // pipelines per kernel family (b200_engine_counter)
  int64_t batch_size = 8192;
  std::map<std::string, std::string> config;
  std::map<std::string, int> agg_hint;       // plan fingerprint -> sink that worked (0 reg, >0 log2 cap)
  uint64_t pf_bucket_slots = (uint64_t)1 << 19;  // partition-first aggregation: table slots per bucket (power of two; 0 = off)
  int64_t pf_min_rows = (int64_t)1 << 22;
  std::map<std::string, uint64_t> agg_groups;  // plan fingerprint -> most groups any task of that shape produced (sizes the table)
  void* pinned_stage = nullptr;              // small pinned buffer for status read-backs
  // ingest narrowing (import_batch): host pool + two pinned staging slots with their device mirrors
  std::unique_ptr<HostPool> pool;
  std::mutex ingest_mu;                      // one narrowing pipeline at a time (pool and staging slots are shared)
  struct NarrowSlot {
    void* pinned = nullptr;
    void* dev = nullptr;
    cudaEvent_t done = nullptr;
    bool used = false;
    size_t bytes = 0;
  } nslot[4];
  int64_t ingest_chunk_rows = (int64_t)1 << 22;
  int ingest_slots = 3;
  // per-kernel device timing (b200.metrics.kernel_timing = on): CUDA event pairs on the launching stream, resolved
  // when the statistics are read (b200_engine_kernel_stats)
  bool kernel_timing = false;
  struct KernelSample { std::string name; cudaEvent_t e0, e1; uint64_t bytes; };
  std::vector<KernelSample> ksamples;
  struct KernelStat { double ms = 0; uint64_t launches = 0, bytes = 0; };
  std::map<std::string, KernelStat> kstats;
  ncclComm_t comm = nullptr;                 // exchange communicator (b200_engine_comm_init); nullptr = single executor
  std::mutex comm_mu;                        // one collective at a time
  uint64_t exch_sent_bytes = 0, exch_recv_bytes = 0;
  // fused shuffle (b200_stage_execute_exchange): one window of HBM per executor, mapped into every peer process through
  // CUDA IPC at b200_engine_comm_init, so the partition scatter kernel stores each row straight into the HBM of the executor
  // that owns its output partition (NVLink / NVSwitch peer stores) -- no staging copy, no separate transfer
  size_t win_config_bytes = 0;               // b200.exchange.window_bytes
  uint8_t* win_local = nullptr;
  size_t win_bytes = 0, win_used = 0;
  std::vector<uint8_t*> win_peer;            // [rank] -> this process's mapping of that rank's window (own rank: win_local)
  uint64_t fused_exchanges = 0;
  std::mutex export_mu;                      // small-result export arena (pinned), one export at a time
  uint8_t* export_arena = nullptr;
  std::atomic<uint64_t> narrowed_bytes_saved{0};         // PCIe bytes not sent thanks to narrowing (b200_engine_counter)
  std::atomic<uint64_t> n_window_sorts{0};               // sorts the window operator ran itself (b200_engine_counter)
  std::atomic<uint64_t> nlj_pairs{0};                    // (build row, probe row) pairs the nested-loop join evaluated (b200_engine_counter)
  std::atomic<uint64_t> string_arena_retries{0};         // launches re-run because their character arena was too small
  std::atomic<uint64_t> host_syncs{0};                   // host waits on the stream inside tasks, exchanges and exports (host_wait)
  // parsed stage plans by plan text with the job id taken out (b200_stage_prepare): the next job that runs the same stage
  // plan shares the parsed tree instead of parsing and typing the JSON again.  Plans are read-only once parsed.
  std::map<std::string, std::shared_ptr<const PlanNode>> plan_cache;
  RegexCache regex;                          // device copies of compiled regex DFAs, by pattern and flags
};

struct b200_stage {
  b200_engine* eng = nullptr;
  std::string job_id;
  int64_t stage_id = 0;
  std::shared_ptr<const PlanNode> plan;  // possibly shared with other stages of the same plan text (b200_engine::plan_cache)
  std::string fingerprint;
  std::vector<OpMetrics> metrics;  // pre-order
  std::map<const PlanNode*, int> metric_index;
};

#define NCCL_CHECK(expr)                                                                                              \
  do {                                                                                                                \
    ncclResult_t _r = (expr);                                                                                         \
    if (_r != 0) throw EngineError(B200_ERR_CUDA, std::string("NCCL error: ") + NcclApi::get().GetErrorString(_r) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
  } while (0)

static void release_window(b200_engine* e);
static void setup_window(b200_engine* e);

namespace {

// ------------------------------------------------------------------------------------------------
// Small helpers
// ------------------------------------------------------------------------------------------------
// Per-thread read-back arena: scalars the host needs from the device (row counts, status words, string
// byte totals) are queued as asynchronous copies into one pinned buffer and become readable after the next
// Exec::sync().  Checks that only have to hold before the task RETURNS (arithmetic-overflow flags of kernels
// whose output size is already known) are deferred to that same synchronisation instead of costing their own.
struct TaskCtx {
  uint8_t* arena = nullptr;
  size_t pos = 0;
  bool drained = true;
  std::vector<std::function<void()>> checks;
};
static const size_t TASK_ARENA_BYTES = (size_t)1 << 16;
inline TaskCtx& task_ctx() {
  static thread_local TaskCtx t;
  if (!t.arena && cudaHostAlloc((void**)&t.arena, TASK_ARENA_BYTES, cudaHostAllocDefault) != cudaSuccess) t.arena = nullptr;
  return t;
}

// Blocks the host until the stream has drained.  Every such wait of a task, an exchange or an export goes through here and
// is counted (b200_engine_counter "host_syncs"): the tail of a small query is bound by these round trips, not by its kernels.
inline cudaError_t host_wait(b200_engine* e, cudaStream_t st) {
  e->host_syncs++;
  return cudaStreamSynchronize(st);
}

struct Exec {
  b200_engine* e;
  b200_stage* s;
  const volatile int32_t* cancel;
  cudaStream_t st() const { return e->stream; }
  void check_cancel() const {
    if (cancel && *cancel) throw EngineError(B200_ERR_CANCELLED, "task cancelled");
  }
  OpMetrics* m(const PlanNode* n) const {
    if (!s) return nullptr;
    auto it = s->metric_index.find(n);
    return it == s->metric_index.end() ? nullptr : &s->metrics[(size_t)it->second];
  }
  // queue a device->host copy of `bytes` bytes; the returned pointer is readable after sync()
  const void* fetch_bytes(const void* dptr, size_t bytes) const {
    TaskCtx& t = task_ctx();
    if (!t.arena) throw EngineError(B200_ERR_OOM, "pinned read-back arena unavailable");
    if (t.drained) {
      t.pos = 0;
      t.drained = false;
    }
    const size_t at = (t.pos + 15) & ~(size_t)15;
    if (at + bytes > TASK_ARENA_BYTES) {  // rare: flush what is queued, then start over
      sync();
      return fetch_bytes(dptr, bytes);
    }
    CUDA_CHECK(cudaMemcpyAsync(t.arena + at, dptr, bytes, cudaMemcpyDeviceToHost, st()));
    t.pos = at + bytes;
    return t.arena + at;
  }
  // pinned host scratch for an asynchronous host->device upload; valid until the next sync()
  void* stage_bytes(size_t bytes) const {
    TaskCtx& t = task_ctx();
    if (!t.arena) throw EngineError(B200_ERR_OOM, "pinned staging arena unavailable");
    if (t.drained) {
      t.pos = 0;
      t.drained = false;
    }
    size_t at = (t.pos + 15) & ~(size_t)15;
    if (at + bytes > TASK_ARENA_BYTES) {
      sync();
      t.pos = 0;
      t.drained = false;
      at = 0;
      if (bytes > TASK_ARENA_BYTES) throw EngineError(B200_ERR_INVALID, "staging request larger than the arena");
    }
    t.pos = at + bytes;
    return t.arena + at;
  }
  template <class T>
  const T* fetch(const void* dptr) const {
    return (const T*)fetch_bytes(dptr, sizeof(T));
  }
  void defer(std::function<void()> fn) const { task_ctx().checks.push_back(std::move(fn)); }
  // wait for everything enqueued so far, then run the deferred checks (they may throw)
  void sync() const {
    TaskCtx& t = task_ctx();
    cudaError_t se = host_wait(e, st());
    t.drained = true;
    std::vector<std::function<void()>> cs;
    cs.swap(t.checks);
    CUDA_CHECK(se);
    for (auto& c : cs) c();
    check_cancel();
  }
  // drop deferred checks without running them (error unwinding)
  static void abandon() {
    TaskCtx& t = task_ctx();
    t.checks.clear();
    t.drained = true;
  }
  template <class T>
  T get(const void* dptr) const {
    const T* p = fetch<T>(dptr);
    sync();
    return *p;
  }
};

// Brackets one kernel (or one short sequence) with CUDA events when kernel timing is on; `bytes` = algorithmic bytes
// (SURVEY.md 8(d) formulas) so that achieved GB/s per kernel family can be reported next to the HBM roofline.
struct KernelTimer {
  b200_engine* e;
  cudaStream_t st;
  b200_engine::KernelSample ks;
  bool on;
  KernelTimer(const Exec& x, const char* name, uint64_t bytes) : e(x.e), st(x.st()), on(x.e->kernel_timing) {
    if (!on) return;
    ks.name = name;
    ks.bytes = bytes;
    if (cudaEventCreate(&ks.e0) != cudaSuccess || cudaEventCreate(&ks.e1) != cudaSuccess) {
      on = false;
      return;
    }
    cudaEventRecord(ks.e0, st);
  }
  ~KernelTimer() {
    if (!on) return;
    cudaEventRecord(ks.e1, st);
    std::lock_guard<std::mutex> g(e->mu);
    e->ksamples.push_back(ks);
  }
};

// B200_TIMING=1: host wall time of the phases of a task (diagnostic; stderr)
struct ScopeTimer {
  const char* name;
  std::chrono::steady_clock::time_point t0;
  bool on;
  explicit ScopeTimer(const char* n) : name(n) {
    static const bool enabled = getenv("B200_TIMING") != nullptr;
    on = enabled;
    if (on) t0 = std::chrono::steady_clock::now();
  }
  ~ScopeTimer() {
    if (on) fprintf(stderr, "[b200-time] %s host_ms=%.3f\n", name, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
  }
};

uint64_t next_pow2(uint64_t v) {
  uint64_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

DevColumn make_out_column(const std::string& name, const DataType& t, Phys phys, int64_t cap, bool with_valid, cudaStream_t st) {
  DevColumn c;
  c.name = name;
  c.type = t;
  c.phys = phys;
  c.n = cap;
  DevPtr d = dev_alloc((size_t)std::max<int64_t>(cap, 1) * phys_width(phys), st);
  c.data = (const uint8_t*)d->ptr;
  c.keep.push_back(d);
  if (with_valid) {
    DevPtr v = dev_alloc((size_t)std::max<int64_t>(cap, 1), st);
    c.valid = (const uint8_t*)v->ptr;
    c.keep.push_back(v);
  }
  c.nullable = with_valid;
  return c;
}

// A batch of small copy / string-conversion jobs executed by ONE kernel (shuffle.cu pack_jobs_kernel): the tail of
// a query moves a handful of rows through a dozen columns and is bound by launch count, not bytes.
struct PackList {
  std::vector<PackJob> jobs;
  void copy(const void* src, void* dst, uint64_t bytes) {
    if (!bytes) return;
    PackJob j;
    memset(&j, 0, sizeof j);
    j.kind = PK_COPY;
    j.src = src;
    j.dst = dst;
    j.bytes = bytes;
    jobs.push_back(j);
  }
  // string column slice (views or Arrow offsets positioned at the first row) -> offsets (rows + 1, from 0) + chars
  void bitmap(const uint8_t* bytes, int64_t rows, void* bitmap_out, void* zero_count_out) {
    PackJob j;
    memset(&j, 0, sizeof j);
    j.kind = PK_BITMAP;
    j.src = bytes;
    j.dst = bitmap_out;
    j.dst2 = zero_count_out;
    j.rows = rows;
    jobs.push_back(j);
  }
  // Arrow Utf8 slice -> views written at `views_out` (rows x 16 bytes)
  void utf8_views(const DevColumn& c, void* views_out) {
    PackJob j;
    memset(&j, 0, sizeof j);
    j.kind = PK_UTF8_VIEWS;
    j.src = c.data;
    j.chars = c.chars;
    j.dst = views_out;
    j.rows = c.n;
    jobs.push_back(j);
  }
  void strings(const DevColumn& c, void* offsets_out, void* chars_out, uint64_t chars_cap = ~0ull) {
    PackJob j;
    memset(&j, 0, sizeof j);
    j.bytes = chars_cap;
    j.kind = c.phys == PH_STRVIEW ? PK_STR_VIEWS : PK_STR_UTF8;
    j.src = c.data;
    j.valid = c.valid;
    j.chars = c.chars;
    j.dst = offsets_out;
    j.dst2 = chars_out;
    j.rows = c.n;
    jobs.push_back(j);
  }
  void run(const Exec& x, std::vector<DevPtr>* keep = nullptr) {
    if (jobs.empty()) return;
    const size_t bytes = jobs.size() * sizeof(PackJob);
    DevPtr d = dev_alloc(bytes, x.st());
    if (bytes <= TASK_ARENA_BYTES / 4) {
      void* h = x.stage_bytes(bytes);
      memcpy(h, jobs.data(), bytes);
      CUDA_CHECK(cudaMemcpyAsync(d->ptr, h, bytes, cudaMemcpyHostToDevice, x.st()));
    } else {
      CUDA_CHECK(cudaMemcpyAsync(d->ptr, jobs.data(), bytes, cudaMemcpyHostToDevice, x.st()));  // pageable: staged by the driver before returning
    }
    launch_pack_jobs((const PackJob*)d->ptr, (int)jobs.size(), x.st());
    if (keep) keep->push_back(d);
    jobs.clear();
  }
};

// strings as views (needed for gather / scatter / sort / join); zero-copy for non-strings
DevColumn as_views(const Exec& x, const DevColumn& c) {
  if (c.phys != PH_UTF8) return c;
  DevColumn o = c;
  DevPtr v = dev_alloc((size_t)std::max<int64_t>(c.n, 1) * 16, x.st());
  launch_utf8_to_views((const int32_t*)c.data, c.chars, (unsigned long long*)v->ptr, c.n, x.st());
  o.phys = PH_STRVIEW;
  o.data = (const uint8_t*)v->ptr;
  o.chars = nullptr;
  o.keep.push_back(v);
  return o;
}

// views -> Arrow Utf8 (offsets + chars), contiguous
DevColumn as_utf8(const Exec& x, const DevColumn& c, int64_t known_total = -1) {
  if (c.phys != PH_STRVIEW) return c;
  const int64_t n = c.n;
  if (known_total >= 0 && n <= 4096) {
    // small column whose character count the host already knows: offsets + chars in ONE launch, no read-back
    DevPtr offsets = dev_alloc((size_t)(n + 1) * 4, x.st());
    DevPtr chars = dev_alloc((size_t)known_total + 16, x.st());
    PackList pl;
    pl.strings(c, offsets->ptr, chars->ptr);
    pl.run(x);
    DevColumn o;
    o.name = c.name;
    o.type = c.type;
    o.nullable = c.nullable;
    o.phys = PH_UTF8;
    o.n = n;
    o.data = (const uint8_t*)offsets->ptr;
    o.chars = (const uint8_t*)chars->ptr;
    o.chars_bytes = known_total;
    o.valid = c.valid;
    o.keep.push_back(offsets);
    o.keep.push_back(chars);
    if (c.valid)
      for (auto& k : c.keep) o.keep.push_back(k);
    return o;
  }
  DevPtr lens = dev_alloc((size_t)(n + 1) * 4, x.st());
  DevPtr offs64 = dev_alloc((size_t)(n + 2) * 8, x.st());
  DevPtr scratch = dev_alloc((size_t)(n / 1024 + 4) * 8, x.st());
  launch_view_lengths((const unsigned long long*)c.data, c.valid, (uint32_t*)lens->ptr, n, x.st());
  launch_scan_u32_to_u64((const uint32_t*)lens->ptr, (uint64_t*)offs64->ptr, n, (uint64_t*)scratch->ptr, x.st());
  uint64_t total = known_total >= 0 ? (uint64_t)known_total : x.get<uint64_t>((const uint64_t*)offs64->ptr + n);
  if (total > 0x7FFFFFFFull) throw EngineError(B200_ERR_UNSUPPORTED, "string column exceeds 2 GiB (LargeUtf8 not supported)");
  DevPtr offsets = dev_alloc((size_t)(n + 1) * 4, x.st());
  DevPtr chars = dev_alloc((size_t)total + 16, x.st());
  launch_views_to_utf8((const unsigned long long*)c.data, c.valid, (const uint64_t*)offs64->ptr, (int32_t*)offsets->ptr, (uint8_t*)chars->ptr, n, x.st());
  DevColumn o;
  o.name = c.name;
  o.type = c.type;
  o.nullable = c.nullable;
  o.phys = PH_UTF8;
  o.n = n;
  o.data = (const uint8_t*)offsets->ptr;
  o.chars = (const uint8_t*)chars->ptr;
  o.chars_bytes = (int64_t)total;
  o.valid = c.valid;
  o.keep.push_back(offsets);
  o.keep.push_back(chars);
  if (c.valid)
    for (auto& k : c.keep) o.keep.push_back(k);  // validity lives in the old allocations
  return o;
}

// Registered tables get 4-byte companion images of the non-null columns that allow one, all or nothing per column:
//  * Utf8 whose strings are all at most 3 bytes long (TPC-H flags, status, ...): key images len << 24 | bytes.  An
//    aggregate that groups by such a column streams 4 bytes per row through the same TMA ring as its other operands
//    instead of gathering characters behind the offsets.
//  * Decimal128 whose values all fit int32 (TPC-H money and quantity columns): the value as int32.  The fused aggregate
//    kernel streams 4 of the 16 bytes per row.
// The table itself stays Arrow; the images cost 4 bytes per row and column of HBM.  One read-back for all columns.
void build_column_images(const Exec& x, DevBatch& b) {
  std::vector<size_t> cands;
  for (size_t ci = 0; ci < b.cols.size(); ci++) {
    const DevColumn& c = b.cols[ci];
    if (c.valid || c.img32 || c.n == 0) continue;
    if (c.phys == PH_UTF8 && c.chars_bytes >= 0 && c.chars_bytes <= 3 * c.n) cands.push_back(ci);  // else some string is longer
    if (c.phys == PH_DEC128) cands.push_back(ci);
  }
  if (cands.empty()) return;
  DevPtr flags = dev_alloc(cands.size() * 4, x.st());
  CUDA_CHECK(cudaMemsetAsync(flags->ptr, 0, cands.size() * 4, x.st()));
  std::vector<DevPtr> imgs;
  for (size_t k = 0; k < cands.size(); k++) {
    const DevColumn& c = b.cols[cands[k]];
    DevPtr img = dev_alloc((size_t)c.n * 4 + 64, x.st());  // slack: a TMA bulk copy of the last tile stays inside
    unsigned int* flag = (unsigned int*)flags->ptr + k;
    if (c.phys == PH_UTF8) launch_prepack3((const int32_t*)c.data, c.chars, c.n, (uint32_t*)img->ptr, flag, x.st());
    else launch_dec128_image(c.data, c.n, (int32_t*)img->ptr, flag, x.st());
    imgs.push_back(img);
  }
  const unsigned int* h = (const unsigned int*)x.fetch_bytes(flags->ptr, cands.size() * 4);
  x.sync();
  for (size_t k = 0; k < cands.size(); k++) {
    if (h[k]) continue;
    DevColumn& c = b.cols[cands[k]];
    c.img32 = (const uint32_t*)imgs[k]->ptr;
    c.keep.push_back(imgs[k]);
  }
}

DevBatchPtr gather_batch(const Exec& x, const DevBatch& in, const int64_t* idx, int64_t n_out, bool may_be_null) {
  auto out = std::make_shared<DevBatch>();
  out->n = n_out;
  GatherCols gc;
  gc.n = 0;
  auto flush = [&]() {
    if (gc.n) {
      uint64_t b = 8;
      for (int k = 0; k < gc.n; k++) b += 2ull * (uint64_t)gc.c[k].width;
      KernelTimer kt(x, "gather", (uint64_t)n_out * b);
      launch_gather_multi(gc, idx, n_out, x.st());
      gc.n = 0;
    }
  };
  for (auto& c0 : in.cols) {
    DevColumn c = as_views(x, c0);
    bool with_valid = c.valid != nullptr || may_be_null;
    DevColumn o = make_out_column(c.name, c.type, c.phys, n_out, with_valid, x.st());
    o.n = n_out;
    GatherCol& g = gc.c[gc.n++];
    g.in = c.data;
    g.valid_in = c.valid;
    g.out = (void*)o.data;
    g.valid_out = (uint8_t*)o.valid;
    g.width = c.width();
    if (gc.n == GATHER_MAX_COLS) flush();
    for (auto& k : c.keep) o.keep.push_back(k);
    out->cols.push_back(o);
  }
  flush();
  return out;
}

// the rows of `parts`, one after the other, as one batch of `schema`: a single piece is sliced without a copy
DevBatchPtr concat_slices(const Exec& x, const std::vector<Piece>& parts, const Schema& schema) {
  auto out = std::make_shared<DevBatch>();
  int64_t total = 0;
  for (auto& p : parts) total += p.r1 - p.r0;
  out->n = total;
  if (parts.size() == 1) {
    const DevBatch& b = *parts[0].batch;
    for (auto& c : b.cols) out->cols.push_back(slice_column(c, parts[0].r0, parts[0].r1));
    return out;
  }
  // few rows (the tail of a query, reduce side of a small shuffle): all copies in one kernel launch
  const bool batched = total <= 65536;
  PackList pl;
  for (size_t ci = 0; ci < schema.size(); ci++) {
    bool any_valid = false;
    for (auto& p : parts) any_valid |= p.batch->cols[ci].valid != nullptr;
    const DataType& t = schema[ci].type;
    Phys ph = t.id == TypeId::Utf8 ? PH_STRVIEW : phys_of(t);
    DevColumn oc = make_out_column(schema[ci].name, t, ph, total, any_valid, x.st());
    oc.n = total;
    int64_t pos = 0;
    for (auto& p : parts) {
      int64_t r0 = p.r0, r1 = p.r1, n = r1 - r0;
      if (n == 0) continue;
      DevColumn sc = slice_column(p.batch->cols[ci], r0, r1);
      if (sc.type != t) throw EngineError(B200_ERR_INVALID, "concat: type mismatch in column " + schema[ci].name);
      if (batched && sc.phys == PH_UTF8) {
        // offsets + characters -> views, straight into the concatenated column (no temporary, no extra launch)
        pl.utf8_views(sc, (uint8_t*)oc.data + pos * oc.width());
        if (any_valid) {
          if (sc.valid) pl.copy(sc.valid, (uint8_t*)oc.valid + pos, (uint64_t)n);
          else CUDA_CHECK(cudaMemsetAsync((uint8_t*)oc.valid + pos, 1, (size_t)n, x.st()));
        }
        for (auto& k : sc.keep) oc.keep.push_back(k);
        pos += n;
        continue;
      }
      DevColumn v = as_views(x, sc);
      if (batched) pl.copy(v.data, (uint8_t*)oc.data + pos * oc.width(), (uint64_t)n * oc.width());
      else CUDA_CHECK(cudaMemcpyAsync((uint8_t*)oc.data + pos * oc.width(), v.data, (size_t)n * oc.width(), cudaMemcpyDeviceToDevice, x.st()));
      if (any_valid) {
        if (v.valid && batched) pl.copy(v.valid, (uint8_t*)oc.valid + pos, (uint64_t)n);
        else if (v.valid) CUDA_CHECK(cudaMemcpyAsync((uint8_t*)oc.valid + pos, v.valid, (size_t)n, cudaMemcpyDeviceToDevice, x.st()));
        else CUDA_CHECK(cudaMemsetAsync((uint8_t*)oc.valid + pos, 1, (size_t)n, x.st()));
      }
      if (ph == PH_STRVIEW)
        for (auto& k : v.keep) oc.keep.push_back(k);
      pos += n;
    }
    out->cols.push_back(oc);
  }
  pl.run(x);
  return out;
}

DevBatchPtr concat(const Exec& x, const std::vector<DevBatchPtr>& parts, const Schema& schema) {
  std::vector<Piece> v;
  for (auto& p : parts) v.push_back(Piece{0, p, 0, p->n});
  return concat_slices(x, v, schema);
}

// character bytes of every Utf8 column of `b` (rows [0, b.n)), one read-back for all of them; known values are reused
std::vector<int64_t> string_bytes(const Exec& x, const DevBatch& b) {
  std::vector<int64_t> out;
  PartStrCols sc;
  sc.n = 0;
  std::vector<size_t> unknown;
  for (auto& c : b.cols) {
    if (c.type.id != TypeId::Utf8) continue;
    if (c.phys == PH_UTF8 && c.chars_bytes >= 0) {
      out.push_back(c.chars_bytes);
      continue;
    }
    out.push_back(-1);
    if (b.n == 0) {
      out.back() = 0;
      continue;
    }
    if (sc.n == PART_MAX_STR_COLS) throw EngineError(B200_ERR_UNSUPPORTED, "more than 16 string columns in one shuffle output");
    sc.c[sc.n++] = PartStrCol{c.data, c.valid, c.phys == PH_STRVIEW ? 1 : 0, 0};
    unknown.push_back(out.size() - 1);
  }
  if (sc.n) {
    DevPtr acc = dev_alloc((size_t)(1 + sc.n) * 8, x.st());
    CUDA_CHECK(cudaMemsetAsync(acc->ptr, 0, (size_t)(1 + sc.n) * 8, x.st()));
    PidSrc none;
    memset(&none, 0, sizeof none);
    CUDA_CHECK(launch_partition_hist(none, b.n, 1, nullptr, (unsigned long long*)acc->ptr, sc, (unsigned long long*)acc->ptr + 1, x.st()));
    const unsigned long long* h = (const unsigned long long*)x.fetch_bytes((const unsigned long long*)acc->ptr + 1, (size_t)sc.n * 8);
    x.sync();
    for (size_t k = 0; k < unknown.size(); k++) out[unknown[k]] = (int64_t)h[k];
  }
  return out;
}

// One column moved by the radix partition's scatter: to `out`, partition after partition, or -- part_base set -- to
// part_base[p] + row * width for the rows of partition p
struct ScatterCol {
  const void* in;
  void* out;
  const unsigned long long* part_base;
  int width;
};

// The radix partition after launch_partition_hist: scans the per-tile histogram into every tile's first destination
// row, then moves the columns, GATHER_MAX_COLS per launch (each timed as `timer`)
void partition_scatter(const Exec& x, const char* timer, const PidSrc& pid, int64_t n, uint32_t P, uint32_t n_tiles, const DevPtr& tile_hist,
                       const std::vector<ScatterCol>& cols) {
  const int64_t hn = (int64_t)P * n_tiles;
  DevPtr offs = dev_alloc((size_t)(hn + 2) * 8, x.st());
  DevPtr scratch = dev_alloc((size_t)(hn / 1024 + 4) * 8, x.st());
  if (hn > 0) launch_scan_u32_to_u64((const uint32_t*)tile_hist->ptr, (uint64_t*)offs->ptr, hn, (uint64_t*)scratch->ptr, x.st());
  if (n == 0) return;
  for (size_t c0 = 0; c0 < cols.size(); c0 += GATHER_MAX_COLS) {
    GatherCols gc;
    memset(&gc, 0, sizeof gc);
    uint64_t b = 0;
    for (; gc.n < GATHER_MAX_COLS && c0 + (size_t)gc.n < cols.size(); gc.n++) {
      const ScatterCol& c = cols[c0 + gc.n];
      GatherCol& g = gc.c[gc.n];
      g.in = c.in;
      g.out = c.out;
      g.part_base = c.part_base;
      g.width = c.width;
      b += (uint64_t)c.width;
    }
    KernelTimer kt(x, timer, (uint64_t)n * (2 * b + 4));
    CUDA_CHECK(launch_partition_scatter(pid, n, P, (const uint64_t*)offs->ptr, gc, nullptr, x.st()));
  }
}

// ------------------------------------------------------------------------------------------------
// Arrow import (host -> HBM)
// ------------------------------------------------------------------------------------------------
// Decimal128 ingest with the sign-extension bytes squeezed out on the host (see host_pool.hpp).
// `src` = n 16-byte values in host memory, `dst` = n 16-byte slots in HBM.  Chunks are narrowed by the
// host pool into one of two pinned staging slots while the previous chunk is still on the bus; a chunk
// whose values do not fit int32 is retried as int64 and finally copied as is.  Bit-exact by construction.
static const int64_t NARROW_CHUNK_ROWS_DEFAULT = (int64_t)1 << 22;  // 64 MiB of source per chunk (b200.ingest.chunk_rows)
static const int64_t NARROW_BLOCK_ROWS = (int64_t)1 << 16;          // one pool task
static const int NARROW_SLOTS = 4;                                  // staging buffers in flight (b200.ingest.slots: 2..4)

void ingest_decimal_narrowed(b200_engine* e, const uint8_t* src, uint8_t* dst, int64_t n, cudaStream_t st) {
  std::lock_guard<std::mutex> ingest_guard(e->ingest_mu);
  if (!e->pool) {
    // default pool size: 1.5 x the CPUs this process may use (cgroup quota if there is one; the loops
    // are memory-latency bound, a few more threads than cores help, many more get throttled)
    int cpus = (int)std::thread::hardware_concurrency();
    if (cpus <= 0) cpus = 8;
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
      long long quota = 0, period = 0;
      if (fscanf(f, "%lld %lld", &quota, &period) == 2 && quota > 0 && period > 0) cpus = std::min<int>(cpus, (int)std::max<long long>(1, quota / period));
      fclose(f);
    }
    int want = std::max(2, cpus + cpus / 2);
    {
      std::lock_guard<std::mutex> g(e->mu);
      auto it = e->config.find("b200.ingest.threads");
      if (it != e->config.end() && atoi(it->second.c_str()) > 0) want = atoi(it->second.c_str());
    }
    e->pool.reset(new HostPool(std::min(want, 256)));
  }
  const int64_t NARROW_CHUNK_ROWS = std::max<int64_t>(NARROW_BLOCK_ROWS, e->ingest_chunk_rows);
  const int n_slots = std::min(NARROW_SLOTS, std::max(2, e->ingest_slots));
  for (int si = 0; si < n_slots; si++) {
    auto& sl = e->nslot[si];
    const size_t need = (size_t)NARROW_CHUNK_ROWS * 8;
    if (sl.pinned && sl.bytes < need) {
      CUDA_CHECK(cudaStreamSynchronize(st));
      cudaFreeHost(sl.pinned);
      cudaFree(sl.dev);
      sl.pinned = sl.dev = nullptr;
      sl.used = false;
    }
    if (!sl.pinned) {
      CUDA_CHECK(cudaHostAlloc(&sl.pinned, need, cudaHostAllocDefault));
      CUDA_CHECK(cudaMalloc(&sl.dev, need));
      if (!sl.done) CUDA_CHECK(cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
      sl.bytes = need;
    }
  }
  int which = 0;
  for (int64_t r0 = 0; r0 < n; r0 += NARROW_CHUNK_ROWS, which = (which + 1) % n_slots) {
    const int64_t rows = std::min(NARROW_CHUNK_ROWS, n - r0);
    b200_engine::NarrowSlot& sl = e->nslot[which];
    if (sl.used) CUDA_CHECK(cudaEventSynchronize(sl.done));  // its previous chunk has left the staging buffer
    const int64_t* p = (const int64_t*)(src + r0 * 16);
    const int n_blocks = (int)((rows + NARROW_BLOCK_ROWS - 1) / NARROW_BLOCK_ROWS);
    int width = 0;
    for (int w : {4, 8}) {
      std::atomic<int> failed{0};
      e->pool->parallel_for(n_blocks, [&](int b) {
        if (failed.load(std::memory_order_relaxed)) return;
        const int64_t b0 = (int64_t)b * NARROW_BLOCK_ROWS, bn = std::min(NARROW_BLOCK_ROWS, rows - b0);
        const bool ok = w == 4 ? narrow_i128_to_i32(p + 2 * b0, bn, (int32_t*)sl.pinned + b0) : narrow_i128_to_i64(p + 2 * b0, bn, (int64_t*)sl.pinned + b0);
        if (!ok) failed.store(1, std::memory_order_relaxed);
      });
      if (!failed.load()) {
        width = w;
        break;
      }
    }
    if (width == 0) {  // genuinely wide values: ship the chunk unchanged
      CUDA_CHECK(cudaMemcpyAsync(dst + r0 * 16, src + r0 * 16, (size_t)rows * 16, cudaMemcpyHostToDevice, st));
      continue;
    }
    CUDA_CHECK(cudaMemcpyAsync(sl.dev, sl.pinned, (size_t)rows * width, cudaMemcpyHostToDevice, st));
    launch_widen_to_i128(sl.dev, width, dst + r0 * 16, rows, st);
    CUDA_CHECK(cudaEventRecord(sl.done, st));
    sl.used = true;
    e->narrowed_bytes_saved += (uint64_t)rows * (uint64_t)(16 - width);
  }
}

DevBatchPtr import_batch_impl(b200_engine* e, ArrowArray* arr, ArrowSchema* sch);

// Ownership of `arr` / `sch` moves to the engine on entry: they are released on success AND on failure (after the copies
// already issued from their buffers have drained), as the Arrow C Data Interface asks of a consumer.
DevBatchPtr import_batch(b200_engine* e, ArrowArray* arr, ArrowSchema* sch) {
  try {
    return import_batch_impl(e, arr, sch);
  } catch (...) {
    cudaStreamSynchronize(e->stream);
    if (arr && arr->release) arr->release(arr);
    if (sch && sch->release) sch->release(sch);
    throw;
  }
}

DevBatchPtr import_batch_impl(b200_engine* e, ArrowArray* arr, ArrowSchema* sch) {
  int64_t n = 0;
  std::vector<ImportedCol> ics = import_record_batch(arr, sch, &n);
  auto b = std::make_shared<DevBatch>();
  b->n = n;
  cudaStream_t st = e->stream;
  // Decimal128 columns of large batches go last, through the narrowing pipeline, so that the host pool
  // works while the plain copies of the other columns are on the bus
  bool narrow_on = n >= ((int64_t)1 << 20);
  {
    std::lock_guard<std::mutex> g(e->mu);
    auto it = e->config.find("b200.ingest.narrow_decimals");
    if (it != e->config.end()) narrow_on = it->second == "on" || (it->second != "off" && narrow_on);
  }
  struct Deferred { const uint8_t* src; uint8_t* dst; };
  std::vector<Deferred> deferred;
  for (auto& ic : ics) {
    DevColumn c;
    c.name = ic.name;
    c.type = ic.type;
    c.phys = phys_of(ic.type);
    c.n = n;
    c.nullable = ic.null_count > 0;
    if (ic.type.id == TypeId::Null) throw EngineError(B200_ERR_UNSUPPORTED, "Null-typed columns are not supported");
    if (ic.null_count > 0 && ic.validity) {
      int64_t b0 = ic.offset >> 3, b1 = (ic.offset + n + 7) >> 3;
      DevPtr bm = dev_alloc((size_t)(b1 - b0) + 16, st);
      CUDA_CHECK(cudaMemcpyAsync(bm->ptr, ic.validity + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, st));
      DevPtr v = dev_alloc((size_t)n + 16, st);
      launch_bitmap_to_bytes((const uint8_t*)bm->ptr, ic.offset & 7, (uint8_t*)v->ptr, n, st);
      c.valid = (const uint8_t*)v->ptr;
      c.keep.push_back(v);
      c.keep.push_back(bm);
    }
    if (ic.type.id == TypeId::Bool) {
      int64_t b0 = ic.offset >> 3, b1 = (ic.offset + n + 7) >> 3;
      DevPtr bm = dev_alloc((size_t)(b1 - b0) + 16, st);
      CUDA_CHECK(cudaMemcpyAsync(bm->ptr, ic.data + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, st));
      DevPtr v = dev_alloc((size_t)n + 16, st);
      launch_bitmap_to_bytes((const uint8_t*)bm->ptr, ic.offset & 7, (uint8_t*)v->ptr, n, st);
      c.data = (const uint8_t*)v->ptr;
      c.keep.push_back(v);
      c.keep.push_back(bm);
    } else if (ic.type.id == TypeId::Utf8) {
      if (ic.large_offsets) throw EngineError(B200_ERR_UNSUPPORTED, "LargeUtf8/LargeBinary input: cast to Utf8 on the host side");
      const int32_t* off = (const int32_t*)ic.data + ic.offset;
      int32_t first = off[0], last = off[n];
      DevPtr d_off = dev_alloc((size_t)(n + 1) * 4 + 64, st);
      CUDA_CHECK(cudaMemcpyAsync(d_off->ptr, off, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, st));
      DevPtr d_chars = dev_alloc((size_t)(last - first) + 64, st);
      if (last > first) CUDA_CHECK(cudaMemcpyAsync(d_chars->ptr, ic.extra + first, (size_t)(last - first), cudaMemcpyHostToDevice, st));
      c.data = (const uint8_t*)d_off->ptr;
      c.chars = (const uint8_t*)d_chars->ptr - first;
      c.chars_bytes = last - first;
      c.keep.push_back(d_off);
      c.keep.push_back(d_chars);
    } else {
      int w = c.width();
      DevPtr d = dev_alloc((size_t)n * w + 64, st);
      if (n && narrow_on && ic.type.id == TypeId::Decimal128 && w == 16) deferred.push_back(Deferred{ic.data + ic.offset * w, (uint8_t*)d->ptr});
      else if (n) CUDA_CHECK(cudaMemcpyAsync(d->ptr, ic.data + ic.offset * w, (size_t)n * w, cudaMemcpyHostToDevice, st));
      c.data = (const uint8_t*)d->ptr;
      c.keep.push_back(d);
    }
    b->cols.push_back(c);
  }
  for (auto& d : deferred) ingest_decimal_narrowed(e, d.src, d.dst, n, st);
  // the copies above read host memory owned by the Arrow arrays: wait before releasing them
  CUDA_CHECK(cudaStreamSynchronize(st));
  if (arr->release) arr->release(arr);
  if (sch->release) sch->release(sch);
  return b;
}

// ------------------------------------------------------------------------------------------------
// Arrow export (HBM -> host)
// ------------------------------------------------------------------------------------------------
// Small results (the tail of most queries is a handful of rows): ONE kernel packs every buffer of the batch
// (bitmaps + null counts, fixed-width values, string offsets and characters) into a device arena, one copy
// brings the arena to pinned host memory, one synchronisation in total.  Character areas are sized optimistically;
// a column that needs more sends the batch down the general path.
static const int64_t SMALL_EXPORT_ROWS = 4096;
static const size_t SMALL_EXPORT_ARENA = (size_t)1 << 20;
static const size_t SMALL_EXPORT_CHARS = (size_t)32 << 10;  // per string column

bool download_small(const Exec& x, const DevBatch& b, int64_t r0, int64_t r1, std::vector<HostCol>& hcs_out) {
  const int64_t n = r1 - r0;
  std::lock_guard<std::mutex> eg(x.e->export_mu);
  if (!x.e->export_arena && cudaHostAlloc((void**)&x.e->export_arena, SMALL_EXPORT_ARENA, cudaHostAllocDefault) != cudaSuccess) {
    x.e->export_arena = nullptr;
    return false;
  }
  uint8_t* arena = x.e->export_arena;
  cudaStream_t st = x.st();
  struct Slot { size_t validity = 0, count = 0, data = 0, chars = 0, chars_cap = 0; bool has_valid = false; };
  std::vector<Slot> slots(b.cols.size());
  std::vector<HostCol> hcs(b.cols.size());
  std::vector<DevColumn> cs(b.cols.size());
  size_t pos = 0;
  auto take = [&](size_t bytes) {
    size_t p = pos;
    pos += (bytes + 63) & ~(size_t)63;
    return p;
  };
  for (size_t ci = 0; ci < b.cols.size(); ci++) {
    cs[ci] = slice_column(b.cols[ci], r0, r1);
    const DevColumn& c = cs[ci];
    HostCol& h = hcs[ci];
    Slot& sl = slots[ci];
    h.name = c.name;
    h.type = c.type;
    h.nullable = true;
    h.n = n;
    if (c.valid && n) {
      sl.has_valid = true;
      sl.validity = take((size_t)(n + 7) / 8);
      sl.count = take(8);
    }
    if (c.type.id == TypeId::Bool) {
      h.data.assign((size_t)(n + 7) / 8, 0);
      sl.data = take(h.data.size());
    } else if (c.type.id == TypeId::Utf8) {
      h.data.resize((size_t)(n + 1) * 4);
      sl.data = take(h.data.size());
      sl.chars_cap = (c.phys == PH_UTF8 && c.chars_bytes >= 0) ? (size_t)c.chars_bytes : SMALL_EXPORT_CHARS;
      sl.chars = take(sl.chars_cap);
    } else {
      h.data.resize((size_t)n * c.width());
      sl.data = take(h.data.size());
    }
    if (pos > SMALL_EXPORT_ARENA) return false;
  }
  if (pos == 0) {
    hcs_out = std::move(hcs);
    return true;
  }
  DevPtr dev = dev_alloc(pos, st);
  uint8_t* d = (uint8_t*)dev->ptr;
  PackList pl;
  for (size_t ci = 0; ci < b.cols.size(); ci++) {
    const DevColumn& c = cs[ci];
    const Slot& sl = slots[ci];
    if (sl.has_valid) pl.bitmap(c.valid, n, d + sl.validity, d + sl.count);
    if (c.type.id == TypeId::Bool) {
      if (n) pl.bitmap(c.data, n, d + sl.data, nullptr);
    } else if (c.type.id == TypeId::Utf8) {
      pl.strings(c, d + sl.data, d + sl.chars, sl.chars_cap);
    } else if (n) {
      pl.copy(c.data, d + sl.data, (uint64_t)n * c.width());
    }
  }
  pl.run(x);
  CUDA_CHECK(cudaMemcpyAsync(arena, d, pos, cudaMemcpyDeviceToHost, st));
  x.sync();
  for (size_t ci = 0; ci < b.cols.size(); ci++)
    if (hcs[ci].type.id == TypeId::Utf8) {
      int32_t total = 0;
      memcpy(&total, arena + slots[ci].data + (size_t)n * 4, 4);
      if ((size_t)total > slots[ci].chars_cap) return false;  // optimistic character area too small: general path
    }
  for (size_t ci = 0; ci < b.cols.size(); ci++) {
    HostCol& h = hcs[ci];
    const Slot& sl = slots[ci];
    if (sl.has_valid) {
      unsigned long long nulls = 0;
      memcpy(&nulls, arena + sl.count, 8);
      h.null_count = (int64_t)nulls;
      if (nulls) h.validity.assign(arena + sl.validity, arena + sl.validity + (size_t)(n + 7) / 8);
    }
    if (!h.data.empty()) memcpy(h.data.data(), arena + sl.data, h.data.size());
    if (h.type.id == TypeId::Utf8) {
      const int32_t total = ((const int32_t*)h.data.data())[n];
      h.extra.assign(arena + sl.chars, arena + sl.chars + (size_t)total);
    }
  }
  hcs_out = std::move(hcs);
  return true;
}

// rows [r0, r1) of a device batch as host columns (Arrow buffers: bitmaps, values, offsets + characters)
std::vector<HostCol> download_batch(const Exec& x, const DevBatch& b, int64_t r0, int64_t r1) {
  const int64_t n = r1 - r0;
  std::vector<HostCol> hcs;
  if (n <= SMALL_EXPORT_ROWS && download_small(x, b, r0, r1, hcs)) return hcs;
  hcs.clear();
  cudaStream_t st = x.st();
  for (auto& c0 : b.cols) {
    DevColumn c = slice_column(c0, r0, r1);
    HostCol h;
    h.name = c.name;
    h.type = c.type;
    h.nullable = true;
    h.n = n;
    if (c.valid && n) {
      DevPtr bm = dev_alloc((size_t)(n + 7) / 8 + 16, st);
      DevPtr cnt = dev_alloc(8, st);
      CUDA_CHECK(cudaMemsetAsync(cnt->ptr, 0, 8, st));
      launch_bytes_to_bitmap(c.valid, (uint8_t*)bm->ptr, n, (unsigned long long*)cnt->ptr, st);
      h.validity.resize((size_t)(n + 7) / 8);
      CUDA_CHECK(cudaMemcpyAsync(h.validity.data(), bm->ptr, h.validity.size(), cudaMemcpyDeviceToHost, st));
      h.null_count = (int64_t)x.get<unsigned long long>(cnt->ptr);
      if (h.null_count == 0) h.validity.clear();
    }
    if (c.type.id == TypeId::Bool) {
      h.data.assign((size_t)(n + 7) / 8, 0);
      if (n) {
        DevPtr bm = dev_alloc((size_t)(n + 7) / 8 + 16, st);
        launch_bytes_to_bitmap(c.data, (uint8_t*)bm->ptr, n, nullptr, st);
        CUDA_CHECK(cudaMemcpyAsync(h.data.data(), bm->ptr, h.data.size(), cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(host_wait(x.e, st));
      }
    } else if (c.type.id == TypeId::Utf8) {
      DevColumn u = c.phys == PH_STRVIEW ? as_utf8(x, c) : c;
      h.data.resize((size_t)(n + 1) * 4);
      CUDA_CHECK(cudaMemcpyAsync(h.data.data(), u.data, h.data.size(), cudaMemcpyDeviceToHost, st));
      CUDA_CHECK(host_wait(x.e, st));
      int32_t* off = (int32_t*)h.data.data();
      int32_t first = off[0], last = off[n];
      h.extra.resize((size_t)(last - first));
      if (last > first) CUDA_CHECK(cudaMemcpyAsync(h.extra.data(), u.chars + first, h.extra.size(), cudaMemcpyDeviceToHost, st));
      CUDA_CHECK(host_wait(x.e, st));
      for (int64_t i = 0; i <= n; i++) off[i] -= first;
    } else {
      h.data.resize((size_t)n * c.width());
      if (n) CUDA_CHECK(cudaMemcpyAsync(h.data.data(), c.data, h.data.size(), cudaMemcpyDeviceToHost, st));
      CUDA_CHECK(host_wait(x.e, st));
    }
    hcs.push_back(std::move(h));
  }
  return hcs;
}

void export_batch(const Exec& x, const DevBatch& b, int64_t r0, int64_t r1, ArrowArray* out, ArrowSchema* out_schema) {
  std::vector<HostCol> hcs = download_batch(x, b, r0, r1);
  export_record_batch(std::move(hcs), r1 - r0, out, out_schema);
}

// ------------------------------------------------------------------------------------------------
// Pipeline execution
// ------------------------------------------------------------------------------------------------
struct RunOutcome {
  RunStatus status;
  float ms = 0;
};

// the fused kernel's description of a program it can run instead of the tile VM (match_fused)
struct FusedPlan {
  FusedSpec spec;
  FusedShape shape;
  int block = 0;
  size_t smem = 0;
};

static void throw_run_error(unsigned int error) {
  if (error == 1) throw EngineError(B200_ERR_EXECUTION, "Arithmetic overflow");
  if (error == 2) throw EngineError(B200_ERR_EXECUTION, "Divide by zero");
  if (error == 4) throw EngineError(B200_ERR_EXECUTION, "concat: a result row is longer than 2147483647 bytes");
  if (error == 5) throw EngineError(B200_ERR_EXECUTION, "repeat: a result row is longer than 2147483647 bytes");
  if (error == 6) throw EngineError(B200_ERR_EXECUTION, "CAST(Date32 AS Utf8): a date outside chrono's range (years -262144..262143)");
  if (error == 7) throw EngineError(B200_ERR_EXECUTION, "regexp_replace: a result row is longer than 2147483647 bytes");
  if (error) throw EngineError(B200_ERR_EXECUTION, "execution error in expression");
}

static bool program_filters(const Program& P) {
  for (int i = 0; i < P.n_instr; i++)
    if (P.code[i].op == OP_FILTER || (P.code[i].flags & IF_FILTER)) return true;
  return false;
}

// Enqueues the pipeline kernel.  wait == true: synchronises, checks the status word and returns it
// (`extra_fetch`, if given, is a device word read back in the same synchronisation).  wait == false:
// the caller already knows the output size; the status check (and the kernel time for the metrics)
// is deferred to the task's next synchronisation.
bool match_groupby(const Program& P, GroupBySpec& S);
bool match_fast_filter(const Program& P, FastFilterSpec& S);

// Partition-first aggregation (AggregateExec with more groups than the L2 can hold a table for): radix-partition the
// referenced columns by hash(keys) % K with the shuffle writer's kernels, so that bucket b's groups live in their own
// region of the table (cap / K slots, ~32 MB of touched cells) that stays in L2 while that bucket's CTAs run -- the
// random accesses of the upsert become L2 hits instead of 32-byte DRAM sectors.  Bytes: one extra read + write of the
// referenced columns (sequential) against three random sectors per row saved.  The bucket ranges are resolved on the
// device (launch_groupby_plan): no host synchronisation between the partition and the aggregation.
bool partition_for_groupby(const Exec& x, GroupBySpec& S, std::vector<DevPtr>& keep) {
  // b200.agg.partition_first.bucket_slots (default 2^19 slots ~ 32 MB of touched cells; 0 = never partition),
  // b200.agg.partition_first.min_rows (default 2^22).  On an H100 SXM (700 W limit), GROUP BY l_partkey (2 M groups) /
  // l_orderkey (15 M groups) over SF10 lineitem, SUM + COUNT, median of 3: 2^19 slots 4.99 / 7.88 ms, 2^18 5.05 / 7.74 ms,
  // 2^17 5.46 / 7.95 ms, never partitioned 11.16 / 8.75 ms.  The min_rows threshold has not been measured on an H100.
  const uint64_t GB_PF_BUCKET_SLOTS = x.e->pf_bucket_slots;
  if (!GB_PF_BUCKET_SLOTS || S.n_keys < 1 || S.table.cap < GB_PF_BUCKET_SLOTS * 8 || S.n_rows < x.e->pf_min_rows || S.n_rows >= ((int64_t)1 << 32)) return false;
  for (int k = 0; k < S.n_keys; k++) {
    const uint32_t w = S.cols[S.key_col[k]].width;
    if (w != 4 && w != 8) return false;
  }
  const uint32_t K = (uint32_t)std::min<uint64_t>(S.table.cap / GB_PF_BUCKET_SLOTS, PART_MAX_FANOUT);
  const int64_t n = S.n_rows;
  PidSrc ps;
  memset(&ps, 0, sizeof ps);
  ps.salt = 0x5bd1e995;  // not the shuffle's partition function: the input may BE one shuffle partition of these very keys
  for (int k = 0; k < S.n_keys; k++) {
    const FusedCol& c = S.cols[S.key_col[k]];
    ps.keys[ps.n_keys++] = KeyCol{c.data, nullptr, (uint8_t)(c.width == 4 ? PH_I32 : PH_I64), (uint8_t)c.width};
  }
  const uint32_t n_tiles = partition_n_tiles(n);
  DevPtr acc = dev_alloc((size_t)K * 8 + 64, x.st());
  CUDA_CHECK(cudaMemsetAsync(acc->ptr, 0, (size_t)K * 8, x.st()));
  DevPtr tile_hist = dev_alloc((size_t)K * n_tiles * 4 + 64, x.st());
  PartStrCols sc;
  sc.n = 0;
  CUDA_CHECK(launch_partition_hist(ps, n, K, (uint32_t*)tile_hist->ptr, (unsigned long long*)acc->ptr, sc, (unsigned long long*)acc->ptr + K, x.st()));
  std::vector<ScatterCol> cols;
  for (int c = 0; c < S.n_cols; c++) {
    DevPtr out = dev_alloc((size_t)n * S.cols[c].width + 64, x.st());
    cols.push_back(ScatterCol{S.cols[c].data, out->ptr, nullptr, (int)S.cols[c].width});
    S.cols[c].data = out->ptr;
    keep.push_back(out);
  }
  partition_scatter(x, "partition_scatter_agg", ps, n, K, n_tiles, tile_hist, cols);
  DevPtr row_start = dev_alloc((size_t)(K + 1) * 8 + 64, x.st()), cta_start = dev_alloc((size_t)(K + 1) * 4 + 64, x.st());
  CUDA_CHECK(launch_groupby_plan((const unsigned long long*)acc->ptr, (int)K, (unsigned long long*)row_start->ptr, (unsigned int*)cta_start->ptr, x.st()));
  S.pf_K = (int)K;
  S.pf_slots = S.table.cap / K;
  S.pf_row_start = (const unsigned long long*)row_start->ptr;
  S.pf_cta_start = (const unsigned int*)cta_start->ptr;
  keep.push_back(row_start);
  keep.push_back(cta_start);
  keep.push_back(acc);
  keep.push_back(tile_hist);
  x.e->n_groupby_pf++;
  return true;
}

RunOutcome launch_program(const Exec& x, PipelineBuilder& pb, int reg_groups, const FusedPlan* fused = nullptr, bool wait = true, OpMetrics* met = nullptr,
                          const unsigned int* extra_fetch = nullptr, unsigned int* extra_out = nullptr, const GroupBySpec* gb = nullptr,
                          const FastFilterSpec* ff = nullptr) {
  Program& P = pb.prog;
  DevPtr dstat = dev_alloc(sizeof(RunStatus), x.st());
  CUDA_CHECK(cudaMemsetAsync(dstat->ptr, 0, sizeof(RunStatus), x.st()));
  P.status = (RunStatus*)dstat->ptr;
  // string builders: a character arena of its own for every launch (a second pass must not overwrite the bytes the
  // first one published).  Its views join the outputs' lifetimes through pb.keep.  Without a sound bound the caller
  // must learn the need, so the launch waits.
  P.arena = nullptr;
  P.arena_cap = 0;
  if (pb.arena_ops) {
    const uint64_t cap = pb.arena_capacity();
    DevPtr arena = dev_alloc(cap + 16, x.st());
    P.arena = (uint8_t*)arena->ptr;
    P.arena_cap = cap;
    pb.keep.push_back(arena);
    if (!pb.arena_sound()) wait = true;
  }
  DevPtr tstate;
  if (P.sink == SINK_MATERIALIZE) {
    const int64_t tile_rows = ff ? 1024 : (int64_t)pb.block * VM_R;
    const int64_t nt = (P.n_rows + tile_rows - 1) / tile_rows;
    tstate = dev_alloc((size_t)std::max<int64_t>(nt, 1) * 8, x.st());
    CUDA_CHECK(cudaMemsetAsync(tstate->ptr, 0, (size_t)std::max<int64_t>(nt, 1) * 8, x.st()));
    P.tile_state = (unsigned long long*)tstate->ptr;
  }
  int grid;
  if (fused) {
    const int64_t warp_tile = 32 * fused->spec.rows_per_thread, nw = fused->block / 32;
    const int64_t n_wt = (P.n_rows + warp_tile - 1) / warp_tile;
    grid = (int)std::min<int64_t>(std::max<int64_t>((n_wt + nw - 1) / nw, 1), x.e->sm_count);
    if (!fused_rows_ok(P, grid, fused->block, fused->spec.rows_per_thread)) fused = nullptr;
  }
  if (!fused) {
    const int tile = pb.block * VM_R;
    int64_t n_tiles = (P.n_rows + tile - 1) / tile;
    grid = (int)std::min<int64_t>(std::max<int64_t>(n_tiles, 1), x.e->sm_count);
  }
  static const bool debug = getenv("B200_DEBUG") != nullptr;
  if (debug)
    fprintf(stderr, "[b200] pipeline sink=%d rows=%lld cols=%d instr=%d regs=%d block=%d stages=%u stage_bytes=%u regs_bytes=%u tma=%u grid=%d\n", (int)P.sink,
            (long long)P.n_rows, P.n_cols, P.n_instr, P.n_regs, pb.block, P.n_stages, P.stage_bytes, P.regs_bytes, P.use_tma, grid);
  if (debug) {
    for (int i = 0; i < P.n_instr; i++) {
      const VInstr& v = P.code[i];
      fprintf(stderr, "[b200]   %2d: op=%d t=%d fl=%d aux=%d dst=(%d,%d,%d) a=(%d,%d,%d) b=(%d,%d,%d) imm=%d\n", i, v.op, v.t, v.flags, v.aux, v.dst.kind, v.dst.vk,
              v.dst.idx, v.a.kind, v.a.vk, v.a.idx, v.b.kind, v.b.vk, v.b.idx, v.imm);
    }
    for (int i = 0; i < P.n_regs; i++) fprintf(stderr, "[b200]   reg %d: vk=%d off=%u valid_off=%u\n", i, P.regs[i].vk, P.regs[i].smem_off, P.regs[i].valid_off);
  }
  uint64_t kt_bytes = 0;
  for (int i = 0; i < P.n_cols; i++) kt_bytes += (uint64_t)(fused ? fused->spec.cols[i].width : P.cols[i].width) * (uint64_t)P.n_rows;  // fused: images when streamed
  if (P.sink == SINK_MATERIALIZE)
    for (int j = 0; j < P.n_out; j++) kt_bytes += (uint64_t)phys_width((Phys)P.out[j].phys) * (uint64_t)P.n_rows;  // upper bound: every row kept
  KernelTimer kt(x, ff ? "filter_compact" : gb ? "groupby_hash_agg" : fused ? "pipeline_fused_agg" : P.sink == SINK_MATERIALIZE ? "pipeline_materialize"
                   : P.mom_pass ? (P.sink == SINK_AGG_REG ? "pipeline_agg_reg_pass2" : "pipeline_agg_global_pass2")
                   : P.sink == SINK_AGG_REG ? "pipeline_agg_reg" : P.n_sets ? "pipeline_agg_gsets" : "pipeline_agg_global", kt_bytes);
  cudaEvent_t e0, e1;
  CUDA_CHECK(cudaEventCreate(&e0));
  CUDA_CHECK(cudaEventCreate(&e1));
  CUDA_CHECK(cudaEventRecord(e0, x.st()));
  cudaError_t le;
  if (ff) {
    FastFilterSpec S = *ff;
    S.status = P.status;
    S.tile_state = P.tile_state;
    le = launch_fast_filter(S, x.e->sm_count, x.st());
    x.e->n_fastfilter++;
  } else if (gb) {
    GroupBySpec S = *gb;
    S.status = P.status;
    S.table = P.table;
    const bool allow_pf = gb->pf_K != -1;
    S.pf_K = 0;
    std::vector<DevPtr> pf_keep;  // stream-ordered: released after the launch below is enqueued
    if (allow_pf) partition_for_groupby(x, S, pf_keep);
    le = launch_groupby(S, x.e->sm_count, x.st());
    x.e->n_groupby++;
  } else if (fused) {
    int is_static = 0;
    le = launch_fused_pipeline(P, fused->spec, fused->shape, reg_groups, grid, fused->block, fused->smem, x.st(), &is_static);
    x.e->n_fused++;
    if (is_static) x.e->n_fused_static++;
    if (debug) {
      const FusedSpec& F = fused->spec;
      fprintf(stderr, "[b200]   fused kernel: static=%d shape=(%#llx,%#llx) block=%d R=%d stages=%d stage_bytes=%u smem=%zu grid=%d tma=%u\n", is_static,
              (unsigned long long)fused->shape.a, (unsigned long long)fused->shape.b, fused->block, F.rows_per_thread, F.n_stages, F.stage_bytes, fused->smem, grid,
              F.use_tma);
      for (int i = 0; i < F.n_filters; i++) fprintf(stderr, "[b200]     filter %d: w=%d op=%d\n", i, F.f[i].w, F.f[i].op - OP_CMP_EQ);
      for (int k = 0; k < F.n_keys; k++) fprintf(stderr, "[b200]     key %d: kind=%d w=%d max_len=%d shift=%d\n", k, F.k[k].kind, F.k[k].w, F.k[k].max_len, F.k[k].shift);
      for (int j = 0; j < F.n_prod; j++) fprintf(stderr, "[b200]     prod %d: kind=%d a_src=%d a_w=%d b_w=%d\n", j, F.p[j].kind, F.p[j].a_src, F.p[j].a_w, F.p[j].b_w);
      for (int a = 0; a < F.n_acc; a++) fprintf(stderr, "[b200]     acc %d: src=%d w=%d\n", a, F.a[a].src, F.a[a].w);
      fprintf(stderr, "[b200]     combine=%d\n", F.combine);
    }
  } else {
    le = launch_pipeline(P, reg_groups, grid, pb.block, pb.smem_bytes(), x.st());
    x.e->n_vm++;
  }
  if (le != cudaSuccess) {
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    CUDA_CHECK(le);
  }
  CUDA_CHECK(cudaEventRecord(e1, x.st()));
  RunOutcome o;
  const RunStatus* hs = x.fetch<RunStatus>(dstat->ptr);
  const unsigned int* he = extra_fetch ? x.fetch<unsigned int>(extra_fetch) : nullptr;
  if (!wait) {
    const unsigned long long arena_cap = P.arena ? P.arena_cap : ~0ull;
    x.defer([hs, e0, e1, met, dstat, tstate, arena_cap]() {
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      cudaEventDestroy(e0);
      cudaEventDestroy(e1);
      if (met) met->elapsed_ns += (uint64_t)(ms * 1e6);
      throw_run_error(hs->error);
      if (hs->arena_need > arena_cap) throw EngineError(B200_ERR_EXECUTION, "string arena: the bytes built exceed their bound");
    });
    memset(&o.status, 0, sizeof o.status);
    return o;
  }
  try {
    x.sync();
  } catch (...) {
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    throw;
  }
  o.status = *hs;
  if (he && extra_out) *extra_out = *he;
  cudaEventElapsedTime(&o.ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (met) met->elapsed_ns += (uint64_t)(o.ms * 1e6);
  throw_run_error(o.status.error);
  return o;
}

uint64_t source_bytes(const PipelineBuilder& pb) {
  uint64_t b = 0;
  for (int i = 0; i < pb.prog.n_cols; i++) b += (uint64_t)pb.prog.cols[i].width * (uint64_t)pb.prog.n_rows + (pb.prog.cols[i].valid ? (uint64_t)pb.prog.n_rows : 0);
  return b;
}

// materialise `outs` (current builder columns) -> new batch
DevBatchPtr run_materialize(const Exec& x, PipelineBuilder& pb, const std::vector<ColRef>& outs, const DevBatchPtr& src, OpMetrics* met) {
  Program& P = pb.prog;
  if (outs.size() > (size_t)VM_MAX_OUT) throw EngineError(B200_ERR_UNSUPPORTED, "too many output columns in one pipeline");
  auto out = std::make_shared<DevBatch>();
  const int64_t cap = src->n;
  P.sink = SINK_MATERIALIZE;
  P.n_out = (uint8_t)outs.size();
  for (size_t j = 0; j < outs.size(); j++) {
    const ColRef& c = outs[j];
    Phys ph = c.type.id == TypeId::Utf8 ? PH_STRVIEW : phys_of(c.type);
    DevColumn oc = make_out_column(c.name, c.type, ph, cap, c.nullable, x.st());
    for (auto& k : c.keep) oc.keep.push_back(k);
    OutCol& d = P.out[j];
    memset(&d, 0, sizeof d);
    d.src = pb.resolve(c);
    d.data = (void*)oc.data;
    d.valid = (uint8_t*)oc.valid;
    d.phys = ph;
    out->cols.push_back(oc);
  }
  pb.finalize_layout(4096);
  // without a filter every input row comes out: no need to wait for the row count
  const bool filters = program_filters(P);
  FastFilterSpec ffs;
  const bool use_ff = filters && match_fast_filter(P, ffs);
  RunOutcome r = launch_program(x, pb, 1, nullptr, filters, met, nullptr, nullptr, nullptr, use_ff ? &ffs : nullptr);
  // the character arena was too small: run again with what it needed (the launch rewrites every output row).  The need
  // is exact unless a CASE / COALESCE moved an unwritten intermediate, so the loop ends after one re-run in practice.
  while (P.arena && r.status.arena_need > P.arena_cap) {
    pb.arena_floor = r.status.arena_need;
    x.e->string_arena_retries++;
    r = launch_program(x, pb, 1, nullptr, filters, met, nullptr, nullptr, nullptr, use_ff ? &ffs : nullptr);
  }
  out->n = filters ? (int64_t)r.status.out_rows : src->n;
  uint64_t wbytes = 0;
  for (auto& c : out->cols) {
    c.n = out->n;
    wbytes += (uint64_t)c.width() * (uint64_t)out->n;
  }
  // the views may point into the source batch's character buffers
  for (auto& c : out->cols)
    if (c.phys == PH_STRVIEW)
      for (auto& sc : src->cols)
        if (sc.phys == PH_UTF8 || sc.phys == PH_STRVIEW)
          for (auto& k : sc.keep) c.keep.push_back(k);
  for (auto& k : pb.keep)
    for (auto& c : out->cols)
      if (c.phys == PH_STRVIEW) c.keep.push_back(k);
  if (met) {
    met->bytes_read += source_bytes(pb);
    met->bytes_written += wbytes;
  }
  return out;
}

// ---- aggregate ------------------------------------------------------------------------------------
struct AggLowered {
  std::vector<ColRef> keys;          // what the group table stores (packed strings are Int64 values)
  std::vector<int> key_pack_shift;   // 0: plain key; 56 / 24: packed short string (bit position of the length)
  bool fast = false;                 // key_hash is an injective 64-bit image of the whole key
  ColRef combined;                   // valid when fast
  std::vector<AccDesc> accs;
  std::vector<ColRef> acc_src;
  std::vector<MomDesc> moms;         // VAR / STDDEV / COVAR / CORR: co-moments of pass 2 (table columns after the accs)
  std::vector<ColRef> key_hashes;    // grouping sets: the hash of each key on its own
  struct OutRecipe {
    uint8_t kind, a, b;
    Phys phys;
    int imm;
    DataType type;
    std::string name;
    bool with_valid;
    int key_idx;
    uint8_t st[6];  // AO_STAT: count, sum x, sum y accumulators; xx, yy, xy co-moments (indices into `moms` until lowered)
  };
  std::vector<OutRecipe> outs;
};

int add_acc(PipelineBuilder& pb, AggLowered& L, uint8_t kind, const ColRef* src) {
  Operand so;
  memset(&so, 0, sizeof so);
  bool nullable = false;
  if (src) {
    so = pb.resolve(*src);
    nullable = src->nullable;
  }
  for (size_t i = 0; i < L.accs.size(); i++) {
    const AccDesc& a = L.accs[i];
    if (a.kind == kind && (kind == ACC_COUNT_STAR || (a.src.kind == so.kind && a.src.idx == so.idx && a.src.vk == so.vk))) return (int)i;
  }
  if (L.accs.size() >= (size_t)VM_MAX_ACC) throw EngineError(B200_ERR_UNSUPPORTED, "too many aggregates in one AggregateExec");
  AccDesc a;
  memset(&a, 0, sizeof a);
  a.kind = kind;
  a.src = so;
  a.nullable = nullable ? 1 : 0;
  a.zext = (src && src->type.id == TypeId::UInt64 && (kind == ACC_MIN_I128 || kind == ACC_MAX_I128)) ? 1 : 0;
  L.accs.push_back(a);
  if (src) {
    pb.pin(*src);
    L.acc_src.push_back(*src);
  }
  return (int)L.accs.size() - 1;
}

// a co-moment sum w * (x - mx) * (y - my) + b of pass 2 (w, b optional); returns its index in L.moms
int add_mom(PipelineBuilder& pb, AggLowered& L, const ColRef& x, const ColRef& y, const ColRef* w, const ColRef* b, int cnt, int sx, int sy) {
  MomDesc m;
  memset(&m, 0, sizeof m);
  m.x = pb.resolve(x);
  m.y = pb.resolve(y);
  if (w) m.w = pb.resolve(*w);
  if (b) m.b = pb.resolve(*b);
  m.cnt = (uint8_t)cnt;
  m.sx = (uint8_t)sx;
  m.sy = (uint8_t)sy;
  for (size_t i = 0; i < L.moms.size(); i++)
    if (memcmp(&L.moms[i], &m, sizeof m) == 0) return (int)i;
  if (L.moms.size() >= (size_t)VM_MAX_MOM) throw EngineError(B200_ERR_UNSUPPORTED, "too many VAR / STDDEV / COVAR / CORR co-moments in one AggregateExec");
  for (const ColRef* c : {&x, &y, w, b})
    if (c) pb.pin(*c);
  L.moms.push_back(m);
  return (int)L.moms.size() - 1;
}

static bool narrowable(const DataType& t) {
  switch (t.id) {
    case TypeId::Utf8:
    case TypeId::Bool:
    case TypeId::Int8:
    case TypeId::Int16:
    case TypeId::Int32:
    case TypeId::UInt8:
    case TypeId::UInt16:
    case TypeId::UInt32:
    case TypeId::Date32: return true;
    default: return false;
  }
}

// pack_mode: 0 = keys as they are; 1 = short strings packed into Int64 (len<<56 | <=7 bytes);
//            2 = every key squeezed into 32 bits and combined injectively into one 64-bit value
// The packed forms are optimistic: the kernel raises pack_overflow when a string does not fit and
// the caller re-lowers with a smaller pack_mode.
void lower_aggregate(PipelineBuilder& pb, const PlanNode& node, AggLowered& L, int pack_mode) {
  const bool from_states = agg_mode_consumes_states(node.agg_mode);
  const bool emit_states = agg_mode_emits_states(node.agg_mode);
  const bool scalar = node.group_by.empty();
  const bool gsets = !node.grouping_sets.empty();
  std::vector<ColRef> narrow32;  // pack_mode 2: non-negative 32-bit images of the keys
  for (size_t g = 0; g < node.group_by.size(); g++) {
    ColRef k0 = pb.compile(*node.group_by[g].expr);
    pb.pin(k0);
    ColRef k = k0;
    int shift = 0;
    if (k0.type.id == TypeId::Utf8 && pack_mode > 0) {
      shift = pack_mode == 2 ? 24 : 56;
      k = pb.str_pack(k0, pack_mode == 2 ? 3 : 7, shift);
      pb.pin(k);
    }
    if (pack_mode == 2) {
      ColRef n32 = k;
      if (shift == 0 && (k0.type.is_signed_int() || k0.type.id == TypeId::Date32)) {
        n32 = pb.add_literal_i64(k, 2147483648ll);
        pb.pin(n32);
      }
      narrow32.push_back(n32);
    }
    k.name = node.group_by[g].name;
    L.keys.push_back(k);
    L.key_pack_shift.push_back(shift);
    AggLowered::OutRecipe r{};
    r.kind = shift ? AO_KEY_PACKED : AO_KEY;
    r.a = (uint8_t)g;
    r.b = 255;
    r.type = k0.type;
    r.phys = k0.type.id == TypeId::Utf8 ? PH_STRVIEW : phys_of(k0.type);
    r.name = k.name;
    r.with_valid = k0.nullable || gsets;
    r.key_idx = (int)g;
    r.imm = shift;
    L.outs.push_back(r);
  }
  if (gsets) {
    // __grouping_id: table key n_keys (written by the grouping-set sink), narrowed to its type by the extraction
    AggLowered::OutRecipe r{};
    r.kind = AO_KEY;
    r.a = (uint8_t)node.group_by.size();
    r.b = 255;
    r.type = grouping_id_type(node.group_by.size());
    r.phys = phys_of(r.type);
    r.name = "__grouping_id";
    r.with_valid = false;
    r.key_idx = -1;
    L.outs.push_back(r);
    // the sink hashes each set's keys itself, from one hash register per key
    for (auto& k : L.keys) L.key_hashes.push_back(pb.hash_of({k}));
  }
  // injective 64-bit key image => the register-cached group directory can be used
  {
    bool all_i64 = !L.keys.empty(), any_null = false;
    for (auto& k : L.keys) {
      all_i64 &= (k.type.pk() == PK::I64 || k.type.pk() == PK::Bool);
      any_null |= k.nullable;
    }
    if (all_i64 && !any_null && !gsets) {
      if (L.keys.size() == 1) {
        L.fast = true;
        L.combined = L.keys[0];
      } else if (pack_mode == 2 && L.keys.size() == 2) {
        L.fast = true;
        L.combined = pb.combine32(narrow32[0], narrow32[1]);
        pb.pin(L.combined);
      }
    }
  }
  const int star = add_acc(pb, L, ACC_COUNT_STAR, nullptr);
  size_t state_col = node.group_by.size();
  (void)emit_states;
  auto push = [&](uint8_t kind, int a, int b, const DataType& t, const std::string& name, bool with_valid, int imm = 0) {
    AggLowered::OutRecipe r{};
    r.kind = kind;
    r.a = (uint8_t)a;
    r.b = (uint8_t)b;
    r.type = t;
    r.phys = phys_of(t);
    r.name = name;
    r.with_valid = with_valid;
    r.imm = imm;
    r.key_idx = -1;
    L.outs.push_back(r);
  };
  auto sum_out_kind = [](const DataType& t) -> uint8_t { return t.pk() == PK::F64 ? AO_ACC_F64 : (t.pk() == PK::I128 ? AO_ACC_I128 : AO_ACC_I64); };
  // MIN / MAX of a value (raw rows or a partial state column): strings as views, floats by their total-order key,
  // everything else (integers, UInt64 zero-extended, decimals, bools) as 128-bit integers
  auto push_minmax = [&](bool mn, const ColRef& v, const DataType& t, const std::string& name) {
    const bool s = v.type.pk() == PK::Str, f = v.type.pk() == PK::F64;
    const uint8_t kind = s ? (mn ? ACC_MIN_STR : ACC_MAX_STR) : f ? (mn ? ACC_MIN_F64 : ACC_MAX_F64) : (mn ? ACC_MIN_I128 : ACC_MAX_I128);
    int a = add_acc(pb, L, kind, &v);
    int c = v.nullable ? add_acc(pb, L, ACC_COUNT, &v) : star;
    push(s ? AO_MINMAX_STR : f ? AO_MINMAX_F64 : sum_out_kind(t), a, c, t, name, v.nullable || scalar);
    if (s) L.outs.back().phys = PH_STRVIEW;  // copied into a buffer of its own after the extraction
  };
  // VAR / STDDEV / COVAR / CORR: the group's count and f64 sums (pass 1) and its centred co-moments (pass 2), then the
  // result or the partial state columns computed from them at extraction
  auto f64_expr = [](const ExprPtr& e) -> ExprPtr {
    if (e->type.id == TypeId::Float64) return e;
    auto c = std::make_shared<Expr>();
    c->kind = Expr::Cast;
    c->type = DataType(TypeId::Float64);
    c->nullable = e->nullable;
    c->args = {e};
    return c;
  };
  auto col_expr = [&](size_t i) {
    auto c = std::make_shared<Expr>();
    c->kind = Expr::Col;
    c->col = (int)i;
    c->type = pb.cols.at(i).type;
    c->nullable = pb.cols.at(i).nullable;
    return c;
  };
  auto push_stat = [&](const AggExpr& ae, int cnt, int sx, int sy, int mxx, int myy, int mxy) {
    const std::string& nm = ae.name;
    const uint8_t st[6] = {(uint8_t)cnt, (uint8_t)sx, (uint8_t)sy, (uint8_t)mxx, (uint8_t)myy, (uint8_t)mxy};
    auto out = [&](int code, const std::string& name) {
      push(AO_STAT, 0, 0, DataType(TypeId::Float64), name, true, code);
      memcpy(L.outs.back().st, st, sizeof st);
    };
    if (emit_states) {
      push(AO_COUNT, cnt, 255, DataType(TypeId::UInt64), nm + "[count]", false);
      if (ae.fn == AggFn::Corr) {
        out(SO_MEAN_X, nm + "[mean1]");
        out(SO_M2_X, nm + "[m2_1]");
        out(SO_MEAN_Y, nm + "[mean2]");
        out(SO_M2_Y, nm + "[m2_2]");
        out(SO_CO, nm + "[algo_const]");
      } else if (agg_is_bivariate(ae.fn)) {
        out(SO_MEAN_X, nm + "[mean1]");
        out(SO_MEAN_Y, nm + "[mean2]");
        out(SO_CO, nm + "[algo_const]");
      } else {
        out(SO_MEAN_X, nm + "[mean]");
        out(SO_M2_X, nm + "[m2]");
      }
      return;
    }
    switch (ae.fn) {
      case AggFn::VarSamp: out(SO_VAR_SAMP, nm); break;
      case AggFn::VarPop: out(SO_VAR_POP, nm); break;
      case AggFn::StddevSamp: out(SO_STDDEV_SAMP, nm); break;
      case AggFn::StddevPop: out(SO_STDDEV_POP, nm); break;
      case AggFn::CovarSamp: out(SO_COVAR_SAMP, nm); break;
      case AggFn::CovarPop: out(SO_COVAR_POP, nm); break;
      default: out(SO_CORR, nm); break;
    }
  };
  auto lower_stat_states = [&](const AggExpr& ae) {
    // Chan's merge: n = sum n_i, mean = sum n_i * mean_i / n, m2 = sum (m2_i + n_i * (mean_i - mean)^2), and the same for the
    // co-moment with both means.  Pass 1 sums n_i and n_i * mean_i, pass 2 the rest around the merged means.
    const size_t c0 = state_col;
    ColRef n_i = pb.cols.at(c0);
    const int cnt = add_acc(pb, L, ACC_SUM_I128, &n_i);
    ColRef w = pb.cast_to(n_i, DataType(TypeId::Float64));
    pb.pin(w);
    auto weighted = [&](size_t mean_col) {
      auto e = std::make_shared<Expr>();
      e->kind = Expr::Bin;
      e->op = BinOp::Mul;
      e->type = DataType(TypeId::Float64);
      e->args = {f64_expr(col_expr(c0)), col_expr(mean_col)};
      e->nullable = e->args[0]->nullable || e->args[1]->nullable;
      ColRef v = pb.compile(*e);
      return add_acc(pb, L, ACC_SUM_F64, &v);
    };
    if (!agg_is_bivariate(ae.fn)) {  // [count] [mean] [m2]
      ColRef mean = pb.cols.at(c0 + 1), m2 = pb.cols.at(c0 + 2);
      const int sx = weighted(c0 + 1);
      const int mxx = add_mom(pb, L, mean, mean, &w, &m2, cnt, sx, sx);
      push_stat(ae, cnt, sx, sx, mxx, mxx, mxx);
      return;
    }
    const bool corr = ae.fn == AggFn::Corr;  // corr: [count] [mean1] [m2_1] [mean2] [m2_2] [algo_const]; covar: [count] [mean1] [mean2] [algo_const]
    const size_t i_mean2 = corr ? c0 + 3 : c0 + 2, i_co = corr ? c0 + 5 : c0 + 3;
    ColRef mean1 = pb.cols.at(c0 + 1), mean2 = pb.cols.at(i_mean2), co = pb.cols.at(i_co);
    const int sx = weighted(c0 + 1), sy = weighted(i_mean2);
    const int mxy = add_mom(pb, L, mean1, mean2, &w, &co, cnt, sx, sy);
    int mxx = mxy, myy = mxy;
    if (corr) {
      ColRef m2_1 = pb.cols.at(c0 + 2), m2_2 = pb.cols.at(c0 + 4);
      mxx = add_mom(pb, L, mean1, mean1, &w, &m2_1, cnt, sx, sx);
      myy = add_mom(pb, L, mean2, mean2, &w, &m2_2, cnt, sy, sy);
    }
    push_stat(ae, cnt, sx, sy, mxx, myy, mxy);
  };
  // the Float64 argument values, compiled once per distinct argument (pair), so that e.g. VAR and STDDEV of one column, or
  // COVAR and CORR of one pair, share their accumulators and co-moments
  std::map<std::string, ColRef> stat_args;
  auto lower_stat_rows = [&](const AggExpr& ae) {
    // covar / corr count a row only when both arguments are non-NULL: each argument is masked by the other's validity
    auto arg = [&](const ExprPtr& v, const ExprPtr& other) {
      const bool mask = other && other->nullable;
      const std::string key = dump_expr(v) + (mask ? "|" + dump_expr(other) : std::string());
      auto it = stat_args.find(key);
      if (it != stat_args.end()) return it->second;
      ExprPtr e = f64_expr(v);
      if (mask) {
        auto nn = std::make_shared<Expr>();
        nn->kind = Expr::IsNotNull;
        nn->type = DataType(TypeId::Bool);
        nn->nullable = false;
        nn->args = {other};
        auto c = std::make_shared<Expr>();
        c->kind = Expr::Case;
        c->type = DataType(TypeId::Float64);
        c->nullable = true;
        c->args = {nn, e};
        e = c;
      }
      ColRef r = pb.compile(*e);
      pb.pin(r);
      stat_args.emplace(key, r);
      return r;
    };
    const ColRef x = arg(ae.arg, ae.arg2);
    const int cnt = x.nullable ? add_acc(pb, L, ACC_COUNT, &x) : star;
    const int sx = add_acc(pb, L, ACC_SUM_F64, &x);
    if (!ae.arg2) {
      const int mxx = add_mom(pb, L, x, x, nullptr, nullptr, cnt, sx, sx);
      push_stat(ae, cnt, sx, sx, mxx, mxx, mxx);
      return;
    }
    const ColRef y = arg(ae.arg2, ae.arg);
    const int sy = add_acc(pb, L, ACC_SUM_F64, &y);
    const int mxy = add_mom(pb, L, x, y, nullptr, nullptr, cnt, sx, sy);
    int mxx = mxy, myy = mxy;
    if (ae.fn == AggFn::Corr) {
      mxx = add_mom(pb, L, x, x, nullptr, nullptr, cnt, sx, sx);
      myy = add_mom(pb, L, y, y, nullptr, nullptr, cnt, sy, sy);
    }
    push_stat(ae, cnt, sx, sy, mxx, myy, mxy);
  };
  for (size_t ai = 0; ai < node.aggs.size(); ai++) {
    const AggExpr& ae = node.aggs[ai];
    const std::string& nm = ae.name;
    if (agg_is_stat(ae.fn)) {
      if (from_states) {
        lower_stat_states(ae);
        state_col += (size_t)ae.n_state_cols();
      } else {
        lower_stat_rows(ae);
      }
      continue;
    }
    if (from_states) {
      ColRef s0 = pb.cols.at(state_col);
      switch (ae.fn) {
        case AggFn::Count: {
          int a = add_acc(pb, L, ACC_SUM_I128, &s0);
          push(AO_COUNT, a, 255, DataType(TypeId::Int64), nm, false);
          break;
        }
        case AggFn::Sum: {
          bool f = s0.type.pk() == PK::F64;
          int a = add_acc(pb, L, f ? ACC_SUM_F64 : ACC_SUM_I128, &s0);
          int c = s0.nullable ? add_acc(pb, L, ACC_COUNT, &s0) : star;
          push(sum_out_kind(ae.result_type), a, c, ae.result_type, nm, s0.nullable || scalar);
          break;
        }
        case AggFn::Min:
        case AggFn::Max: {
          push_minmax(ae.fn == AggFn::Min, s0, ae.result_type, nm);
          break;
        }
        case AggFn::Avg: {
          ColRef s1 = pb.cols.at(state_col + 1);
          int c = add_acc(pb, L, ACC_SUM_I128, &s0);
          bool f = s1.type.pk() == PK::F64;
          int a = add_acc(pb, L, f ? ACC_SUM_F64 : ACC_SUM_I128, &s1);
          if (f) push(AO_AVG_F64, a, c, ae.result_type, nm, true);
          else push(AO_AVG_DEC, a, c, ae.result_type, nm, true, ae.result_type.scale - ae.sum_type.scale);
          break;
        }
        default: break;
      }
      state_col += (size_t)ae.n_state_cols();
      continue;
    }
    ColRef arg;
    bool has_arg = ae.arg != nullptr;
    if (has_arg) arg = pb.compile(*ae.arg);
    switch (ae.fn) {
      case AggFn::Count: {
        int a = (has_arg && arg.nullable) ? add_acc(pb, L, ACC_COUNT, &arg) : star;
        push(AO_COUNT, a, 255, DataType(TypeId::Int64), emit_states ? nm + "[count]" : nm, false);
        break;
      }
      case AggFn::Sum: {
        ColRef v = arg;
        bool f = ae.sum_type.pk() == PK::F64;
        if (f) v = pb.cast_to(arg, DataType(TypeId::Float64));
        int a = add_acc(pb, L, f ? ACC_SUM_F64 : ACC_SUM_I128, &v);
        int c = v.nullable ? add_acc(pb, L, ACC_COUNT, &v) : star;
        push(sum_out_kind(ae.sum_type), a, c, ae.sum_type, emit_states ? nm + "[sum]" : nm, v.nullable || scalar);
        break;
      }
      case AggFn::Min:
      case AggFn::Max: {
        const bool mn = ae.fn == AggFn::Min;
        push_minmax(mn, arg, ae.sum_type, emit_states ? nm + (mn ? "[min]" : "[max]") : nm);
        break;
      }
      case AggFn::Avg: {
        ColRef v = arg;
        bool f = !arg.type.is_decimal();
        if (f) v = pb.cast_to(arg, DataType(TypeId::Float64));
        int a = add_acc(pb, L, f ? ACC_SUM_F64 : ACC_SUM_I128, &v);
        int c = v.nullable ? add_acc(pb, L, ACC_COUNT, &v) : star;
        if (emit_states) {
          push(AO_COUNT, c, 255, DataType(TypeId::UInt64), nm + "[count]", false);
          push(sum_out_kind(ae.sum_type), a, c, ae.sum_type, nm + "[sum]", v.nullable || scalar);
        } else if (f) {
          push(AO_AVG_F64, a, c, ae.result_type, nm, true);
        } else {
          push(AO_AVG_DEC, a, c, ae.result_type, nm, true, ae.result_type.scale - ae.sum_type.scale);
        }
        break;
      }
      default: break;
    }
  }
  // the co-moments occupy three table columns each after the accumulators
  const size_t n_acc = L.accs.size();
  for (size_t m = 0; m < L.moms.size(); m++) L.moms[m].col = (uint8_t)(n_acc + 3 * m);
  for (auto& r : L.outs)
    if (r.kind == AO_STAT)
      for (int k = 3; k < 6; k++) r.st[k] = (uint8_t)(n_acc + 3 * r.st[k]);
}

// ------------------------------------------------------------------------------------------------
// Pattern match of a lowered register-aggregate program against the fused fast path
// (filters on integer-like tile columns -> up to two decimal products -> <= 2 packed/integer keys ->
// SUM/COUNT accumulators).  Anything outside the pattern keeps the general VM path.
// ------------------------------------------------------------------------------------------------
static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v && *v ? atoi(v) : dflt;
}

// Recognise the scan -> filter -> decimal products -> small SUM/COUNT aggregate shape in a lowered
// program and lay out the per-warp stage buffers of the fused kernel (fused.cuh).
bool match_fused(const Program& P, FusedPlan& FP) {
  FusedSpec& F = FP.spec;
  memset(&F, 0, sizeof F);
  if (P.sink != SINK_AGG_REG) return false;
  if (P.n_mom) return false;  // VAR / STDDEV / COVAR / CORR need the second pass of the VM sinks
  if (P.n_sets) return false;  // grouping sets run on the global sink's grouping-set variant only
  if (getenv("B200_NO_FUSED")) return false;
  for (int a = 0; a < P.n_acc; a++)
    if (!(P.acc[a].kind == ACC_SUM_I128 || P.acc[a].kind == ACC_COUNT || P.acc[a].kind == ACC_COUNT_STAR)) return false;
  // stage layout: every column of the program, one warp tile of 32*R rows each
  // 4 rows per thread amortise the per-tile work (claim, TMA issue, barrier wait); grouped shapes then fit
  // 8 warps of up to 255 registers next to their shared-memory partials, scalar shapes 12 warps.  On an
  // H100 SXM (700 W limit) stage 1 of q1 at SF10 took 1.62-1.73 ms at R=4 / 256 threads against
  // 1.69-1.83 ms for R=4 / 384 and R=2 / 256, 384, 512 (Arrow widths, 76 B/row).
  // With every column streamed as a 4-byte image (28 B/row) the kernel is no longer bandwidth-bound at 8 warps:
  // on an H100 80GB HBM3 (700 W limit), median of 10 runs, stage 1 of q1 at SF10 took 1.09 ms at R=4 / 256
  // threads (1.05-1.08 ms with 2-4 stages), 0.80 ms at R=4 / 384 (3 stages), 0.90 ms at R=8 / 256 (not kept), 1.39, 1.13
  // and 1.01 ms at R=2 / 256, 384, 512.  So narrow tiles run 12 warps of R=4.
  const int R = env_int("B200_FUSED_R", 4);
  if (!(R == 2 || R == 4)) return false;
  const uint32_t TR = 32u * (uint32_t)R;
  if (P.n_cols > FUSED_MAX_COLS || P.n_cols == 0) return false;
  uint32_t fused_off[VM_MAX_COLS];
  uint32_t cur = 0, tx = 0, tx_utf8 = 0;
  bool aligned = true, narrow = true;
  // columns with a 4-byte companion image (build_column_images) stream the image: short-string keys are read as 4-byte
  // integer key columns, decimals as int32 (every use of a decimal column in a matched program is a filter, a product
  // operand or a SUM source, and all of them sign-extend 4-byte tile values)
  bool imaged[VM_MAX_COLS] = {false};
  if (!getenv("B200_NO_PREPACK")) {
    for (int i = 0; i < P.n_instr; i++) {
      const VInstr& v = P.code[i];
      if (v.op == OP_STR_PACK8 && v.a.kind == OPD_COL && v.imm == 24 && v.aux <= 3 && P.cols[v.a.idx].phys == PH_UTF8 && P.cols[v.a.idx].img32)
        imaged[v.a.idx] = true;
    }
    for (int c = 0; c < P.n_cols; c++)
      if (P.cols[c].phys == PH_DEC128 && P.cols[c].img32) imaged[c] = true;
    for (int c = 0; c < P.n_cols; c++)
      if (((uintptr_t)P.cols[c].img32) & 15) imaged[c] = false;  // the bulk copies need 16-byte aligned sources
  }
  for (int c = 0; c < P.n_cols; c++) {
    const ColDesc& cd = P.cols[c];
    if (cd.valid) return false;
    FusedCol& fc = F.cols[c];
    fc.data = imaged[c] ? cd.img32 : cd.data;
    fc.width = imaged[c] ? 4 : cd.width;
    fc.utf8 = (cd.phys == PH_UTF8 && !imaged[c]) ? 1u : 0u;
    fc.tile_bytes = TR * fc.width + (fc.utf8 ? 16u : 0u);
    if (fc.tile_bytes & 15u) return false;
    fc.off = cur;
    fused_off[c] = cur;
    cur += fc.tile_bytes;
    if (fc.utf8) tx_utf8 += fc.tile_bytes;
    else tx += fc.tile_bytes;
    if (((uintptr_t)fc.data & 15) != 0) aligned = false;
    narrow &= fc.width <= 4 && !fc.utf8;
  }
  int block = env_int("B200_FUSED_B", (R == 4 && P.n_keys && !narrow) ? 256 : 384);
  if (block > (R == 4 ? 384 : 512) || block < 32 || (block & 31)) return false;
  F.n_cols = P.n_cols;
  F.rows_per_thread = R;
  F.stage_bytes = (cur + 127u) & ~127u;
  F.tile_tx = tx;
  F.tile_tx_utf8 = tx_utf8;
  F.use_tma = (aligned && !getenv("B200_NO_TMA")) ? 1u : 0u;
  {
    // shared memory: per-warp rings, then (grouped shapes) 8 bytes per (group, accumulator, thread)
    const size_t budget = 216 * 1024;
    const size_t acc_per_thread = P.n_keys ? (size_t)VM_REG_GROUPS * VM_REG_ACC * 8 : 0;
    const int want_S = std::min(env_int("B200_FUSED_S", FUSED_MAX_STAGES), (int)FUSED_MAX_STAGES);
    int S = 0;
    for (;; block -= 32) {
      if (block < 64) return false;
      const size_t acc = acc_per_thread * block;
      if (acc >= budget) continue;
      S = (int)((budget - acc) / ((size_t)(block / 32) * F.stage_bytes));
      if (S >= 2) break;
    }
    S = std::min(S, want_S);
    if (S < 2) return false;
    F.n_stages = S;
    FP.block = block;
    // the end-of-kernel reduction stages [VM_REG_ACC][block] 16-byte partials in the idle rings
    size_t ring = std::max((size_t)(block / 32) * S * F.stage_bytes, (size_t)VM_REG_ACC * block * 16);
    ring = (ring + 127) & ~(size_t)127;
    F.acc_off = (uint32_t)ring;
    FP.smem = ring + acc_per_thread * block;
  }
  auto int_col = [&](const Operand& o, uint32_t* off, uint8_t* w, bool want_i128) -> bool {
    if (o.kind != OPD_COL) return false;
    const ColDesc& cd = P.cols[o.idx];
    if (cd.valid) return false;
    if (!(cd.phys == PH_I32 || cd.phys == PH_I64 || cd.phys == PH_DEC128)) return false;
    if (want_i128 && o.vk == VK_I128 && cd.phys != PH_DEC128) return false;
    // the width the kernel streams: a decimal (also its narrow view, the low word) is 16 bytes, or 4 with its image
    *off = fused_off[o.idx];
    *w = (uint8_t)F.cols[o.idx].width;
    return true;
  };
  int prod_reg[2] = {-1, -1};
  struct PackInfo { int reg; FusedKey k; };
  std::vector<PackInfo> packs;      // packed-string / biased-int key images by register
  int combined_reg = -1, comb_a = -1, comb_b = -1;
  for (int i = 0; i < P.n_instr; i++) {
    const VInstr& v = P.code[i];
    if (v.flags & IF_NULLCHK) return false;
    switch (v.op) {
      case OP_CMP_EQ: case OP_CMP_NE: case OP_CMP_LT: case OP_CMP_LE: case OP_CMP_GT: case OP_CMP_GE: {
        if (!(v.flags & IF_FILTER) || v.t != VK_I64 || v.aux == PH_U64) return false;
        if (F.n_filters >= FUSED_MAX_FILTERS) return false;
        FusedFilter& f = F.f[F.n_filters];
        Operand col = v.a, imm = v.b;
        uint8_t op = v.op;
        if (v.a.kind == OPD_IMM && v.b.kind == OPD_COL) {
          col = v.b;
          imm = v.a;
          op = v.op == OP_CMP_LT ? OP_CMP_GT : v.op == OP_CMP_LE ? OP_CMP_GE : v.op == OP_CMP_GT ? OP_CMP_LT : v.op == OP_CMP_GE ? OP_CMP_LE : v.op;
        }
        if (imm.kind != OPD_IMM || P.imms[imm.idx].is_null) return false;
        Operand c64 = col;
        c64.vk = VK_I64;
        if (!int_col(c64, &f.off, &f.w, false)) return false;
        f.op = op;
        f.imm = (int64_t)P.imms[imm.idx].lo;
        F.n_filters++;
        break;
      }
      case OP_DEC_MUL_LIT_MINUS: case OP_DEC_MUL_LIT_PLUS: case OP_MUL: {
        if (v.op == OP_MUL && v.t != VK_I128) return false;
        if (F.n_prod >= 2 || v.dst.kind != OPD_REG) return false;
        FusedProd& q = F.p[F.n_prod];
        q.kind = v.op == OP_DEC_MUL_LIT_MINUS ? 0 : v.op == OP_DEC_MUL_LIT_PLUS ? 1 : 2;
        if (v.a.kind == OPD_REG && F.n_prod == 1 && (int)v.a.idx == prod_reg[0]) {
          q.a_src = 1;
        } else if (!int_col(v.a, &q.a_off, &q.a_w, true)) {
          return false;
        }
        if (!int_col(v.b, &q.b_off, &q.b_w, true)) return false;
        if (q.kind != 2) {
          q.lit_lo = P.imms[v.imm].lo;
          q.lit_hi = P.imms[v.imm].hi;
        }
        prod_reg[F.n_prod++] = v.dst.idx;
        break;
      }
      case OP_STR_PACK8: {
        if (v.a.kind != OPD_COL || P.cols[v.a.idx].phys != PH_UTF8 || P.cols[v.a.idx].valid || v.dst.kind != OPD_REG) return false;
        PackInfo pi;
        pi.reg = v.dst.idx;
        memset(&pi.k, 0, sizeof pi.k);
        if (imaged[v.a.idx]) {  // the image is already in the tile: an integer key column of width 4
          pi.k.kind = 0;
          pi.k.off = fused_off[v.a.idx];
          pi.k.w = 4;
          packs.push_back(pi);
          break;
        }
        pi.k.kind = 1;
        pi.k.off = fused_off[v.a.idx];
        pi.k.chars = P.cols[v.a.idx].chars;
        pi.k.offsets = (const int32_t*)P.cols[v.a.idx].data;
        pi.k.max_len = v.aux;
        pi.k.shift = (uint8_t)v.imm;
        pi.k.w = (pi.k.shift == 24 && pi.k.max_len <= 3) ? 4 : 8;
        packs.push_back(pi);
        break;
      }
      case OP_MADD_I64: {
        if (v.a.kind != OPD_REG || v.b.kind != OPD_REG || v.dst.kind != OPD_REG || P.imms[v.imm].lo != 4294967296ull) return false;
        combined_reg = v.dst.idx;
        comb_a = v.a.idx;
        comb_b = v.b.idx;
        break;
      }
      default: return false;
    }
  }
  // keys
  F.n_keys = P.n_keys;
  if (P.n_keys > 2) return false;
  if (P.n_keys > 0 && !P.keys_all_i64) return false;
  auto key_from = [&](const Operand& o, FusedKey& k) -> bool {
    if (o.kind == OPD_REG) {
      for (auto& pi : packs)
        if (pi.reg == (int)o.idx) {
          k = pi.k;
          return true;
        }
      return false;
    }
    if (o.kind == OPD_COL) {
      memset(&k, 0, sizeof k);
      uint32_t off;
      uint8_t w;
      Operand c64 = o;
      c64.vk = VK_I64;
      if (!int_col(c64, &off, &w, false) || P.cols[o.idx].phys == PH_DEC128) return false;
      k.kind = 0;
      k.off = off;
      k.w = w;
      return true;
    }
    return false;
  };
  for (int k = 0; k < P.n_keys; k++)
    if (!key_from(P.keys[k], F.k[k])) return false;
  if (P.n_keys == 1) {
    if (!(P.key_hash.kind == P.keys[0].kind && P.key_hash.idx == P.keys[0].idx)) return false;
    F.combine = 0;
  } else if (P.n_keys == 2) {
    // only the all-packed-string form: the 32-bit images are the pack registers themselves
    if (P.key_hash.kind != OPD_REG || (int)P.key_hash.idx != combined_reg) return false;
    if (!(P.keys[0].kind == OPD_REG && P.keys[1].kind == OPD_REG && comb_a == (int)P.keys[0].idx && comb_b == (int)P.keys[1].idx)) return false;
    F.combine = 1;
  }
  if (combined_reg >= 0 && P.n_keys != 2) return false;
  // accumulators
  if (P.n_acc > VM_REG_ACC) return false;
  F.n_acc = P.n_acc;
  for (int a = 0; a < P.n_acc; a++) {
    const AccDesc& ad = P.acc[a];
    FusedAcc& fa = F.a[a];
    if (ad.kind == ACC_COUNT_STAR || (ad.kind == ACC_COUNT && !ad.nullable)) {
      fa.src = 3;
      continue;
    }
    if (ad.kind != ACC_SUM_I128 || ad.nullable) return false;
    if (ad.src.kind == OPD_REG) {
      if ((int)ad.src.idx == prod_reg[0]) fa.src = 1;
      else if ((int)ad.src.idx == prod_reg[1]) fa.src = 2;
      else return false;
    } else if (ad.src.kind == OPD_COL) {
      if (!int_col(ad.src, &fa.off, &fa.w, true)) return false;
      if (ad.src.vk != VK_I128 && P.cols[ad.src.idx].phys == PH_DEC128) return false;
      fa.src = 0;
    } else {
      return false;
    }
  }
  // every packed register must be a key (no stray uses)
  for (auto& pi : packs) {
    bool used = false;
    for (int k = 0; k < P.n_keys; k++) used |= P.keys[k].kind == OPD_REG && (int)P.keys[k].idx == pi.reg;
    if (!used) return false;
  }
  // the code-shaping part of the spec (program.h FusedShape)
  FusedShapeDesc d;
  memset(&d, 0, sizeof d);
  d.nf = F.n_filters;
  for (int i = 0; i < F.n_filters; i++) {
    d.fw[i] = F.f[i].w;
    d.fop[i] = (uint8_t)(F.f[i].op - OP_CMP_EQ);
  }
  d.nk = F.n_keys;
  for (int k = 0; k < F.n_keys; k++) {
    d.kkind[k] = F.k[k].kind;
    d.kw[k] = F.k[k].w;
  }
  d.combine = F.combine;
  d.np = F.n_prod;
  for (int j = 0; j < F.n_prod; j++) {
    d.pkind[j] = F.p[j].kind;
    d.pasrc[j] = F.p[j].a_src;
    d.paw[j] = F.p[j].a_w;
    d.pbw[j] = F.p[j].b_w;
  }
  d.na = F.n_acc;
  for (int a = 0; a < F.n_acc; a++) {
    d.asrc[a] = F.a[a].src;
    d.aw[a] = F.a[a].w;
  }
  FP.shape = fused_shape_encode(d);
  return true;
}

// Recognise scan -> integer/date/decimal compares against literals -> up to two decimal products -> one or two integer-like
// key COLUMNS -> COUNT / SUM accumulators in a lowered aggregate program: the shape the dedicated high-cardinality kernel
// (groupby.cu) runs without the tile VM.  Hash instructions of the general key path are ignored (the kernel hashes the
// key image itself).
bool match_groupby(const Program& P, GroupBySpec& S) {
  memset(&S, 0, sizeof S);
  if (getenv("B200_NO_GROUPBY")) return false;
  if (P.n_mom) return false;  // VAR / STDDEV / COVAR / CORR need the second pass of the VM sinks
  if (P.n_sets) return false;  // grouping sets run on the global sink's grouping-set variant only
  if (P.n_keys < 1 || P.n_keys > 2 || P.n_acc > GB_MAX_ACC || P.n_cols > FUSED_MAX_COLS || P.n_cols == 0) return false;
  for (int c = 0; c < P.n_cols; c++) {
    const ColDesc& cd = P.cols[c];
    if (cd.valid) return false;
    if (!(cd.phys == PH_I32 || cd.phys == PH_I64 || cd.phys == PH_U64 || cd.phys == PH_DEC128)) return false;
    S.cols[c].data = cd.data;
    S.cols[c].width = cd.width;
  }
  S.n_cols = P.n_cols;
  auto col_of = [&](const Operand& o, int* out) -> bool {
    if (o.kind != OPD_COL || o.idx >= (unsigned)P.n_cols) return false;
    *out = (int)o.idx;
    return true;
  };
  int prod_reg[2] = {-1, -1};
  for (int i = 0; i < P.n_instr; i++) {
    const VInstr& v = P.code[i];
    switch (v.op) {
      case OP_HASH:
      case OP_HASH_COMBINE: break;  // the general path's row hash: not needed
      case OP_CMP_EQ: case OP_CMP_NE: case OP_CMP_LT: case OP_CMP_LE: case OP_CMP_GT: case OP_CMP_GE: {
        if (!(v.flags & IF_FILTER) || (v.flags & IF_NULLCHK) || v.t != VK_I64 || v.aux == PH_U64) return false;
        if (S.n_filters >= FUSED_MAX_FILTERS) return false;
        Operand col = v.a, imm = v.b;
        uint8_t op = v.op;
        if (v.a.kind == OPD_IMM && v.b.kind == OPD_COL) {
          col = v.b;
          imm = v.a;
          op = v.op == OP_CMP_LT ? OP_CMP_GT : v.op == OP_CMP_LE ? OP_CMP_GE : v.op == OP_CMP_GT ? OP_CMP_LT : v.op == OP_CMP_GE ? OP_CMP_LE : v.op;
        }
        if (imm.kind != OPD_IMM || P.imms[imm.idx].is_null) return false;
        if (!col_of(col, &S.f_col[S.n_filters])) return false;
        S.f_op[S.n_filters] = (int)op - (int)OP_CMP_EQ;
        S.f_imm[S.n_filters] = (int64_t)P.imms[imm.idx].lo;
        S.n_filters++;
        break;
      }
      case OP_DEC_MUL_LIT_MINUS: case OP_DEC_MUL_LIT_PLUS: case OP_MUL: {
        if ((v.flags & IF_NULLCHK) || (v.op == OP_MUL && v.t != VK_I128)) return false;
        if (S.n_prod >= 2 || v.dst.kind != OPD_REG) return false;
        const int j = S.n_prod;
        S.p_kind[j] = v.op == OP_DEC_MUL_LIT_MINUS ? 0 : v.op == OP_DEC_MUL_LIT_PLUS ? 1 : 2;
        if (v.a.kind == OPD_REG && j == 1 && (int)v.a.idx == prod_reg[0]) S.p_a_src[j] = 1;
        else if (!col_of(v.a, &S.p_a_col[j])) return false;
        if (!col_of(v.b, &S.p_b_col[j])) return false;
        if (S.p_kind[j] != 2) {
          const uint64_t lo = P.imms[v.imm].lo, hi = P.imms[v.imm].hi;
          if (hi != (uint64_t)((int64_t)lo >> 63)) return false;
          S.p_lit[j] = (int64_t)lo;
        }
        prod_reg[S.n_prod++] = v.dst.idx;
        break;
      }
      default: return false;
    }
  }
  S.n_keys = P.n_keys;
  for (int k = 0; k < P.n_keys; k++) {
    if (!col_of(P.keys[k], &S.key_col[k])) return false;
    if (P.cols[S.key_col[k]].phys == PH_DEC128) return false;
  }
  S.n_acc = P.n_acc;
  for (int a = 0; a < P.n_acc; a++) {
    const AccDesc& ad = P.acc[a];
    if (ad.kind == ACC_COUNT_STAR || (ad.kind == ACC_COUNT && !ad.nullable)) {
      S.a_src[a] = 3;
      continue;
    }
    if (ad.kind != ACC_SUM_I128 || ad.nullable) return false;
    if (ad.src.kind == OPD_REG) {
      if ((int)ad.src.idx == prod_reg[0]) S.a_src[a] = 1;
      else if ((int)ad.src.idx == prod_reg[1]) S.a_src[a] = 2;
      else return false;
    } else if (col_of(ad.src, &S.a_col[a])) {
      S.a_src[a] = 0;
    } else {
      return false;
    }
  }
  S.n_rows = P.n_rows;
  S.table = P.table;
  return true;
}

// Recognise a materialising program that only FILTERS (comparisons of plain columns with literals or with each other,
// combined with AND / OR / NOT) and forwards plain columns: the shape the dedicated FilterExec kernel (filter.cu) runs
// without the tile VM.  LIKE, arithmetic, casts, NULL-aware compares or computed outputs keep the VM.
bool match_fast_filter(const Program& P, FastFilterSpec& S) {
  if (P.sink != SINK_MATERIALIZE || getenv("B200_NO_FASTFILTER")) return false;
  if (P.n_cols > FF_MAX_COLS || P.n_cols == 0 || P.n_instr > FF_MAX_OPS || P.n_instr == 0 || P.n_imms > FF_MAX_IMMS || P.n_out > FF_MAX_OUT || P.n_regs > 64) return false;
  memset(&S, 0, sizeof S);
  auto int_phys = [](uint8_t ph) { return ph == PH_I8 || ph == PH_I16 || ph == PH_I32 || ph == PH_I64 || ph == PH_U8 || ph == PH_U16 || ph == PH_U32 || ph == PH_U64; };
  for (int c = 0; c < P.n_cols; c++) {
    const ColDesc& cd = P.cols[c];
    if (cd.valid) return false;
    if (!(int_phys(cd.phys) || cd.phys == PH_DEC128 || cd.phys == PH_UTF8 || cd.phys == PH_STRVIEW || cd.phys == PH_F64 || cd.phys == PH_F32 || cd.phys == PH_BOOL8)) return false;
    S.cols[c].data = cd.data;
    S.cols[c].chars = cd.chars;
    S.cols[c].phys = cd.phys;
    S.cols[c].width = cd.width;
  }
  S.n_cols = P.n_cols;
  for (int i = 0; i < P.n_imms; i++) {
    S.imms[i].lo = P.imms[i].lo;
    S.imms[i].hi = P.imms[i].hi;
  }
  auto bool_reg = [&](const Operand& o, uint8_t* out) {
    if (o.kind != OPD_REG || o.vk != VK_BOOL || o.idx >= 64) return false;
    *out = (uint8_t)o.idx;
    return true;
  };
  bool any_filter = false;
  for (int i = 0; i < P.n_instr; i++) {
    const VInstr& v = P.code[i];
    FfOp& op = S.ops[S.n_ops];
    memset(&op, 0, sizeof op);
    if (v.flags & IF_NULLCHK) return false;
    switch (v.op) {
      case OP_CMP_EQ: case OP_CMP_NE: case OP_CMP_LT: case OP_CMP_LE: case OP_CMP_GT: case OP_CMP_GE: {
        op.kind = FF_CMP;
        op.cmp = (uint8_t)(v.op - OP_CMP_EQ);
        if (!(v.t == VK_I64 || v.t == VK_I128 || v.t == VK_STR)) return false;
        if (v.t == VK_STR && !(v.op == OP_CMP_EQ || v.op == OP_CMP_NE)) return false;
        bool wide = v.t == VK_I128;
        const Operand* ops2[2] = {&v.a, &v.b};
        uint8_t idx[2], is_imm[2];
        for (int k = 0; k < 2; k++) {
          const Operand& o = *ops2[k];
          if (o.kind == OPD_IMM) {
            if (o.idx >= (unsigned)P.n_imms || P.imms[o.idx].is_null) return false;
            idx[k] = (uint8_t)o.idx;
            is_imm[k] = 1;
          } else if (o.kind == OPD_COL) {
            if (o.idx >= (unsigned)P.n_cols) return false;
            const uint8_t ph = P.cols[o.idx].phys;
            if (v.t == VK_STR) {
              if (!(ph == PH_UTF8 || ph == PH_STRVIEW)) return false;
            } else {
              if (!(int_phys(ph) || ph == PH_DEC128)) return false;
              wide = wide || ph == PH_DEC128;
            }
            idx[k] = (uint8_t)o.idx;
            is_imm[k] = 0;
          } else {
            return false;
          }
        }
        op.a = idx[0];
        op.b = idx[1];
        op.a_imm = is_imm[0];
        op.b_imm = is_imm[1];
        op.vt = v.t == VK_STR ? 2 : (wide ? 1 : (v.aux == PH_U64 ? 3 : 0));
        if (wide && v.aux == PH_U64) return false;
        // a 64-bit immediate compared as 128 bits needs its sign extension in `hi`
        for (int k = 0; k < 2; k++)
          if (op.vt == 1 && is_imm[k] && v.t != VK_I128) S.imms[idx[k]].hi = (uint64_t)((int64_t)S.imms[idx[k]].lo >> 63);
        if (v.flags & IF_FILTER) op.filter = 1;
        else if (!bool_reg(v.dst, &op.dst)) return false;
        break;
      }
      case OP_AND:
      case OP_OR:
        op.kind = v.op == OP_AND ? FF_AND : FF_OR;
        if (!bool_reg(v.a, &op.a) || !bool_reg(v.b, &op.b) || !bool_reg(v.dst, &op.dst)) return false;
        break;
      case OP_NOT:
        op.kind = FF_NOT;
        if (!bool_reg(v.a, &op.a) || !bool_reg(v.dst, &op.dst)) return false;
        break;
      case OP_FILTER:
        op.kind = FF_FILTER_REG;
        op.filter = 1;
        if (!bool_reg(v.a, &op.a)) return false;
        break;
      default: return false;
    }
    any_filter = any_filter || op.filter;
    S.n_ops++;
  }
  if (!any_filter) return false;
  for (int j = 0; j < P.n_out; j++) {
    const OutCol& oc = P.out[j];
    if (oc.src.kind != OPD_COL || oc.src.idx >= (unsigned)P.n_cols || oc.valid) return false;
    const uint8_t ph = P.cols[oc.src.idx].phys;
    const bool str = ph == PH_UTF8 || ph == PH_STRVIEW;
    if (str ? oc.phys != PH_STRVIEW : (oc.phys != ph)) return false;
    S.out_col[j] = (uint8_t)oc.src.idx;
    S.out_data[j] = oc.data;
  }
  S.n_out = P.n_out;
  S.n_rows = P.n_rows;
  return true;
}

struct TableMem {
  AggTable T;
  std::vector<DevPtr> keep;
};

// zero_cols: f64 sum columns after the accumulators (the co-moments of VAR / STDDEV / COVAR / CORR), zero-initialised
TableMem alloc_table(const Exec& x, uint64_t cap, int n_keys, const std::vector<AccDesc>& accs, size_t zero_cols = 0) {
  TableMem tm;
  memset(&tm.T, 0, sizeof tm.T);
  auto A = [&](size_t bytes) {
    DevPtr p = dev_alloc(bytes, x.st());
    tm.keep.push_back(p);
    return p->ptr;
  };
  tm.T.cap = cap;
  tm.T.hash = (unsigned long long*)A(cap * 8);
  tm.T.state = (unsigned int*)A(cap * 4);
  tm.T.lock = (unsigned int*)A(cap * 4);
  tm.T.keys = (unsigned long long*)A(std::max<size_t>(1, (size_t)n_keys) * cap * 16);
  tm.T.key_valid = (unsigned char*)A(std::max<size_t>(1, (size_t)n_keys) * cap);
  tm.T.acc = (unsigned long long*)A(std::max<size_t>(1, accs.size() + zero_cols) * cap * 16);
  if (zero_cols) CUDA_CHECK(cudaMemsetAsync(tm.T.acc + accs.size() * cap * 2, 0, zero_cols * cap * 16, x.st()));
  tm.T.n_groups = (unsigned int*)A(16);
  AccKinds k;
  memset(&k, 0, sizeof k);
  k.n = (int)accs.size();
  for (size_t i = 0; i < accs.size(); i++) k.kind[i] = accs[i].kind;
  launch_agg_table_init(tm.T, k, x.st());
  return tm;
}

typedef std::function<std::unique_ptr<PipelineBuilder>()> BuilderFactory;

DevBatchPtr run_aggregate(const Exec& x, const BuilderFactory& make_pb, const PlanNode& node, const DevBatchPtr& src, OpMetrics* met) {
  const int n_keys = (int)node.group_by.size();
  if (n_keys > VM_MAX_KEYS) throw EngineError(B200_ERR_UNSUPPORTED, "too many group-by columns");
  // grouping sets: every row lands in up to n_sets groups, all on the global table's grouping-set sink (the register sink
  // holds 4 groups: a ROLLUP of two flags already has more)
  const int n_sets = (int)node.grouping_sets.size();
  static_assert(kMaxGroupingSetKeys + 1 <= (size_t)VM_MAX_KEYS && kMaxGroupingSets <= sizeof(Program::set_mask), "grouping-set limits");
  const int table_keys = n_keys + (n_sets ? 1 : 0);
  const int64_t max_groups = std::max<int64_t>(src->n, 1) * std::max(n_sets, 1);
  // initial optimism about the keys
  int pack_mode = 0;
  {
    bool any_str = false, all_narrow = n_keys > 0;
    for (auto& g : node.group_by) {
      any_str |= g.expr->type.id == TypeId::Utf8;
      all_narrow &= narrowable(g.expr->type);
    }
    if (n_keys == 2 && all_narrow && !n_sets) pack_mode = 2;
    else if (any_str) pack_mode = 1;
  }
  int node_idx = -1;
  if (x.s) {
    auto it = x.s->metric_index.find(&node);
    if (it != x.s->metric_index.end()) node_idx = it->second;
  }
  const std::string hint_key = (x.s ? x.s->fingerprint : std::string("?")) + "#" + std::to_string(node_idx);
  int level = 0;
  bool had_hint = false;
  uint64_t groups_hint = 0;
  {
    std::lock_guard<std::mutex> g(x.e->mu);
    auto it = x.e->agg_hint.find(hint_key);
    if (it != x.e->agg_hint.end()) {
      level = it->second / 4;
      pack_mode = std::min(pack_mode, it->second % 4);
      had_hint = true;
      auto ig = x.e->agg_groups.find(hint_key);
      if (ig != x.e->agg_groups.end()) groups_hint = ig->second;
    }
  }
  const int hinted_level = had_hint ? level : -1;
  bool sampled = false;
  // strategy ladder: register sink (<= 4 groups) -> global table of growing capacity; packed keys -> plain keys
  std::unique_ptr<PipelineBuilder> pbp;
  AggLowered L;
  TableMem tm;
  RunOutcome ro;
  unsigned int n_groups = 0;
  int reg_groups = 0;
  bool gb_bailed = false, pf_off = false, gs_grown = false;
  uint64_t arena_floor = 0;  // string builders: the character arena an earlier attempt needed
  for (;;) {
    x.check_cancel();
    ScopeTimer t_iter("  agg: lower+alloc+launch+sync");
    pbp = make_pb();
    PipelineBuilder& pb = *pbp;
    L = AggLowered();
    lower_aggregate(pb, node, L, pack_mode);
    pb.arena_floor = arena_floor;
    Program& P = pb.prog;
    P.n_keys = (uint8_t)n_keys;
    P.n_acc = (uint8_t)L.accs.size();
    for (int k = 0; k < n_keys; k++) P.keys[k] = pb.resolve(L.keys[(size_t)k]);
    for (size_t a = 0; a < L.accs.size(); a++) P.acc[a] = L.accs[a];
    P.n_mom = (uint8_t)L.moms.size();
    for (size_t m = 0; m < L.moms.size(); m++) P.mom[m] = L.moms[m];
    memset(&P.key_hash, 0, sizeof P.key_hash);
    P.keys_all_i64 = L.fast ? 1 : 0;
    P.n_sets = (uint8_t)n_sets;
    for (int s = 0; s < n_sets; s++) {
      P.set_mask[s] = (uint8_t)node.grouping_sets[(size_t)s];
      P.set_id[s] = grouping_id(node.grouping_sets[(size_t)s], (size_t)n_keys);
    }
    for (size_t k = 0; k < L.key_hashes.size(); k++) P.key_hashes[k] = pb.resolve(L.key_hashes[k]);
    if (n_keys && !n_sets) {
      if (L.fast) {
        P.key_hash = pb.resolve(L.combined);
      } else {
        ColRef h = pb.hash_of(L.keys);
        P.key_hash = h.op;
      }
    }
    const bool reg_ok = (int)L.accs.size() <= VM_REG_ACC && !n_sets;
    if (!reg_ok && level == 0) level = 1;
    // up to a few million input rows a table sized for "every row its own group" is cheap: no capacity ladder.  Grouping
    // sets first get that size too (the finest set holds at most one group per row and the coarser ones usually few);
    // the table for every row in every set only after that overflows
    const bool small_input = src->n <= ((int64_t)1 << 22);
    if (level > 0 && small_input) level = 8;
    const bool gs_rows_first = n_sets && small_input && !gs_grown;
    uint64_t cap;
    reg_groups = 0;
    if (level == 0) {
      P.sink = SINK_AGG_REG;
      reg_groups = n_keys ? VM_REG_GROUPS : 1;
      cap = n_keys ? 64 : 2;
    } else {
      P.sink = SINK_AGG_GLOBAL;
      if (!n_keys) cap = 2;
      else cap = std::min<uint64_t>(next_pow2((uint64_t)(gs_rows_first ? std::max<int64_t>(src->n, 1) : max_groups) * 2), (uint64_t)1 << std::min(40, 12 + 4 * level));
      // a plan shape seen before: size the table for the groups its tasks produced (x2.5: load factor <= 0.4 with room for a
      // somewhat larger sibling task) instead of the whole class -- the classes are 16x apart, and every slot costs ~80 bytes
      // of memset and of extraction scan.  An overflow falls back to the class size (level++ below leaves hinted_level).
      if (groups_hint && level == hinted_level && n_keys) cap = std::min(cap, std::max<uint64_t>(next_pow2(groups_hint * 5 / 2), 4096));
      if (cap < 16) cap = 16;
    }
    {
      ScopeTimer t_alloc("    agg: alloc_table");
      tm = alloc_table(x, cap, table_keys, L.accs, 3 * L.moms.size());
    }
    P.table = tm.T;
    pb.finalize_layout((size_t)VM_REG_ACC * 512 * 16 + 256);
    if (level == 0) {
      const size_t hi_bytes = (size_t)x.e->sm_count * 512 * VM_REG_GROUPS * VM_REG_ACC * 8;
      DevPtr hi = dev_alloc(hi_bytes, x.st());
      tm.keep.push_back(hi);
      P.acc_hi = (unsigned long long*)hi->ptr;
      // string / UInt64 MIN / MAX keep their per-thread values in a scratch of their own (initialised by the kernel)
      for (size_t a = 0; a < L.accs.size(); a++)
        P.has_side_acc |= (L.accs[a].kind == ACC_MIN_STR || L.accs[a].kind == ACC_MAX_STR || L.accs[a].zext) ? 1 : 0;
      if (P.has_side_acc) {
        DevPtr side = dev_alloc(hi_bytes, x.st());
        tm.keep.push_back(side);
        P.acc_side = (unsigned long long*)side->ptr;
      }
    }
    // First sight of a large integer-keyed aggregate: group the first 16 K rows on the hash kernel to learn whether the
    // 4-group register sink can apply at all and which table class to start with, instead of discovering it by running
    // (and abandoning) full passes up the capacity ladder.
    if (!sampled && !had_hint && level == 0 && n_keys > 0 && src->n > ((int64_t)1 << 20)) {
      sampled = true;
      GroupBySpec probe;
      const int64_t sample_rows = 16384;
      TableMem stm = alloc_table(x, 65536, n_keys, L.accs);
      P.table = stm.T;
      if (match_groupby(P, probe)) {
        probe.n_rows = sample_rows;
        probe.pf_K = -1;
        unsigned int seen = 0;
        RunOutcome so = launch_program(x, pb, 0, nullptr, true, nullptr, stm.T.n_groups, &seen, &probe);
        if (!so.status.pack_overflow && (so.status.overflow || seen > (unsigned)VM_REG_GROUPS)) {
          level = (so.status.overflow || (int64_t)seen * 2 > sample_rows) ? 3 : 2;  // (nearly) every row its own group: 16 M slots; else 1 M
          continue;
        }
      }
      P.table = tm.T;
    }
    FusedPlan fspec;
    const bool use_fused = level == 0 && match_fused(P, fspec);
    GroupBySpec gspec;
    const bool use_gb = level > 0 && !gb_bailed && match_groupby(P, gspec);
    gspec.pf_K = pf_off ? -1 : 0;
    {
      ScopeTimer t_l("    agg: launch_program (incl. sync)");
      ro = launch_program(x, pb, reg_groups, use_fused ? &fspec : nullptr, true, met, tm.T.n_groups, &n_groups, use_gb ? &gspec : nullptr);
    }
    if (P.arena && ro.status.arena_need > P.arena_cap) {
      arena_floor = ro.status.arena_need;  // the same table size again (re-allocated, so re-initialised) with that arena
      x.e->string_arena_retries++;
      continue;
    }
    if (ro.status.pack_overflow && use_gb) {
      gb_bailed = true;  // operands outside the dedicated kernel's ranges: same table size on the general sink
      continue;
    }
    if (ro.status.pack_overflow) {
      pack_mode = pack_mode == 2 ? 1 : 0;
      continue;
    }
    if (!ro.status.overflow) break;
    if (gs_rows_first) {
      gs_grown = true;  // more groups than input rows over all sets: the table for every row in every set
      continue;
    }
    if (level > 0 && cap >= next_pow2((uint64_t)max_groups * 2)) {
      if (use_gb && !pf_off) {
        pf_off = true;  // a bucket's region of the partitioned table filled up (skewed buckets): same table, unpartitioned
        continue;
      }
      throw EngineError(B200_ERR_EXECUTION, "aggregate hash table overflow");
    }
    level++;
  }
  if (!L.moms.empty()) {
    // pass 2 of VAR / STDDEV / COVAR / CORR: the same program over the same rows folds the centred co-moments into the
    // groups pass 1 published (an overflow of pass 1 has already restarted both passes above)
    x.check_cancel();
    Program& P = pbp->prog;
    P.mom_pass = 1;
    RunOutcome r2 = launch_program(x, *pbp, reg_groups, nullptr, true, met);
    P.mom_pass = 0;
    if (P.arena && r2.status.arena_need > P.arena_cap) throw EngineError(B200_ERR_EXECUTION, "aggregate: the second pass built more string bytes than the first");
    if (r2.status.overflow) throw EngineError(B200_ERR_EXECUTION, "aggregate: a group of the first pass was not found by the second");
  }
  {
    // remember the smallest table class that holds this many groups (not the level that happened to be used: a small
    // input jumps straight to a table sized for its row count)
    int learnt = level;
    if (level > 0) {
      learnt = 1;
      while (learnt < 7 && ((uint64_t)1 << (12 + 4 * learnt)) < (uint64_t)n_groups * 2) learnt++;
    }
    std::lock_guard<std::mutex> g(x.e->mu);
    x.e->agg_hint[hint_key] = learnt * 4 + pack_mode;
    uint64_t& gh = x.e->agg_groups[hint_key];
    gh = std::max<uint64_t>(gh, n_groups);
  }
  PipelineBuilder& pb = *pbp;
  // extraction
  ScopeTimer t_ex("  agg: extract");
  auto out = std::make_shared<DevBatch>();
  out->n = n_groups;
  AggExtractArgs A;
  memset(&A, 0, sizeof A);
  if (L.outs.size() > (size_t)VM_MAX_OUT) throw EngineError(B200_ERR_UNSUPPORTED, "too many aggregate output columns");
  A.n_out = (int)L.outs.size();
  A.n_keys = table_keys;
  DevPtr counter = dev_alloc(16, x.st());
  CUDA_CHECK(cudaMemsetAsync(counter->ptr, 0, 16, x.st()));
  A.counter = (unsigned long long*)counter->ptr;
  A.error = (unsigned int*)((uint8_t*)counter->ptr + 8);
  uint64_t wbytes = 0;
  for (size_t j = 0; j < L.outs.size(); j++) {
    const auto& r = L.outs[j];
    DevColumn oc = make_out_column(r.name, r.type, r.phys, n_groups, r.with_valid, x.st());
    oc.n = n_groups;
    if (r.key_idx >= 0) {
      for (auto& k : L.keys[(size_t)r.key_idx].keep) oc.keep.push_back(k);
      if (r.phys == PH_STRVIEW) {
        for (auto& sc : src->cols)
          for (auto& k : sc.keep) oc.keep.push_back(k);
        for (auto& k : pb.keep) oc.keep.push_back(k);
      }
    }
    AggOut& o = A.out[j];
    o.data = (void*)oc.data;
    o.valid = (uint8_t*)oc.valid;
    o.aux = nullptr;
    if (r.kind == AO_KEY_PACKED) {
      DevPtr ch = dev_alloc((size_t)std::max<unsigned int>(n_groups, 1) * 8, x.st());
      o.aux = ch->ptr;
      oc.keep.push_back(ch);
    }
    o.kind = r.kind;
    o.a = r.a;
    o.b = r.b;
    o.phys = r.phys;
    o.imm = r.imm;
    o.prec = r.type.precision;
    memcpy(o.st, r.st, sizeof o.st);
    wbytes += (uint64_t)oc.width() * n_groups;
    out->cols.push_back(oc);
  }
  launch_agg_extract(tm.T, A, x.st());
  // string MIN / MAX results are views of the input's characters (or of a literal of the pipeline): copy them into a
  // buffer of their own, so that the result outlives the input and a few strings do not pin a multi-GB character buffer.
  // The character total is not known on the host: each such column costs three launches and one read-back of it.
  for (size_t j = 0; j < L.outs.size(); j++)
    if (L.outs[j].kind == AO_MINMAX_STR) out->cols[j] = as_utf8(x, out->cols[j]);
  {
    // the extraction's overflow flag (decimal AVG / SUM precision) only has to be seen before the task returns
    const unsigned int* herr = x.fetch<unsigned int>(A.error);
    x.defer([herr, counter]() {
      if (*herr) throw EngineError(B200_ERR_EXECUTION, "Arithmetic overflow");
    });
  }
  for (size_t c = 0; c < out->cols.size() && c < node.schema.size(); c++) out->cols[c].name = node.schema[c].name;
  if (met) {
    met->bytes_read += source_bytes(pb);
    met->bytes_written += wbytes;
    met->input_rows += (uint64_t)src->n;
  }
  return out;
}

// ------------------------------------------------------------------------------------------------
// Operator tree execution
// ------------------------------------------------------------------------------------------------
struct Runner {
  Exec x;
  std::string job;

  int n_partitions(const PlanNode& n) {
    switch (n.op) {
      case PlanNode::Scan: {
        std::lock_guard<std::mutex> g(x.e->mu);
        auto it = x.e->tables.find(n.table);
        if (it == x.e->tables.end()) throw EngineError(B200_ERR_INVALID, "table not registered: " + n.table);
        return it->second.empty() ? 0 : it->second.rbegin()->first + 1;
      }
      case PlanNode::ShuffleReader: return x.e->shuffle.partitions(job, n.reader_stage_id);
      case PlanNode::SortPreservingMerge: return 1;
      case PlanNode::Passthrough:
        if (n.op_name == "CoalescePartitionsExec") return 1;
        return n_partitions(*n.children[0]);
      case PlanNode::HashJoin: return n_partitions(*n.children[1]);
      default: return n_partitions(*n.children[0]);
    }
  }

  DevBatchPtr empty_batch(const Schema& s) {
    auto out = std::make_shared<DevBatch>();
    for (auto& f : s) {
      Phys ph = f.type.id == TypeId::Utf8 ? PH_STRVIEW : phys_of(f.type);
      DevColumn c = make_out_column(f.name, f.type, ph, 0, false, x.st());
      c.n = 0;
      out->cols.push_back(c);
    }
    return out;
  }

  DevBatchPtr exec_all(const PlanNode& n) {
    int np = n_partitions(n);
    std::vector<DevBatchPtr> parts;
    for (int p = 0; p < np; p++) parts.push_back(exec(n, p));
    if (parts.empty()) return empty_batch(n.schema);
    return concat(x, parts, n.schema);
  }

  // Walk down a Filter/Projection chain; returns the base node and the chain (top-down order).
  const PlanNode* chain_base(const PlanNode& top, std::vector<const PlanNode*>& chain) {
    const PlanNode* cur = &top;
    while (cur->op == PlanNode::Filter || cur->op == PlanNode::Projection ||
           (cur->op == PlanNode::Passthrough && cur->op_name != "CoalescePartitionsExec")) {
      if (cur->op == PlanNode::Filter && cur->fetch >= 0) break;
      if (cur->op != PlanNode::Passthrough) chain.push_back(cur);
      cur = cur->children[0].get();
    }
    return cur;
  }

  void apply_chain(PipelineBuilder& pb, const std::vector<const PlanNode*>& chain) {
    for (size_t i = chain.size(); i-- > 0;) {
      const PlanNode* n = chain[i];
      if (n->op == PlanNode::Filter) {
        pb.apply_filter(*n->predicate);
        if (n->has_projection) pb.apply_select(n->projection);
      } else {
        pb.apply_projection(n->exprs);
      }
    }
  }

  // Executes `top` (a Filter/Projection chain over some base) fused into one pipeline whose sink is
  // decided by the caller through `finish`.
  // Executes `top` (a Filter/Projection chain over some base) fused into one pipeline whose sink is
  // decided by the caller through `finish(make_builder, src)`; make_builder() returns a fresh
  // builder over `src` with the chain applied (sinks that retry with another lowering call it again).
  template <class F>
  DevBatchPtr with_chain(const PlanNode& top, int part, bool all_parts, F&& finish) {
    std::vector<const PlanNode*> chain;
    const PlanNode* base = chain_base(top, chain);
    DevBatchPtr src = all_parts ? exec_all(*base) : exec(*base, part);
    for (auto* n : chain)
      if (OpMetrics* m = x.m(n)) m->input_rows += (uint64_t)src->n;
    BuilderFactory make_pb = [&]() {
      std::unique_ptr<PipelineBuilder> pb(new PipelineBuilder(*src, x.st(), &x.e->regex));
      apply_chain(*pb, chain);
      return pb;
    };
    return finish(make_pb, src);
  }

  std::vector<ColRef> named_cols(PipelineBuilder& pb, const Schema& schema) {
    std::vector<ColRef> outs = pb.cols;
    for (size_t i = 0; i < outs.size() && i < schema.size(); i++) outs[i].name = schema[i].name;
    return outs;
  }

  // Runs operator n and charges it (its kernel_launches metric) the kernels it launched itself: what this thread enqueued
  // meanwhile, less what the operators it ran through exec() enqueued -- they are charged their own.  Filter / projection
  // nodes fused into a parent's chain run inside the parent and are charged to it.  Returns the operator's own launches.
  uint64_t nested_launches = 0;  // kernels enqueued inside the charged calls of this Runner so far
  template <class F>
  uint64_t charge_launches(const PlanNode& n, F&& run) {
    const uint64_t l0 = launches_on_thread(), n0 = nested_launches;
    run();
    const uint64_t all = launches_on_thread() - l0, own = all - (nested_launches - n0);
    nested_launches = n0 + all;
    if (OpMetrics* m = x.m(&n)) m->launches += own;
    return own;
  }

  // B200_TIMING=1: inclusive host wall time per operator (launch + synchronisation overheads) and its own launches
  DevBatchPtr exec(const PlanNode& n, int part) {
    static const bool timing = getenv("B200_TIMING") != nullptr;
    const auto t0 = std::chrono::steady_clock::now();
    DevBatchPtr out;
    const uint64_t own = charge_launches(n, [&] { out = exec_impl(n, part); });
    if (timing) {
      cudaStreamSynchronize(x.st());
      const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      fprintf(stderr, "[b200-time] op=%d part=%d rows_out=%lld host_ms=%.3f launches=%llu\n", (int)n.op, part, (long long)(out ? out->n : -1), ms,
              (unsigned long long)own);
    }
    return out;
  }
  DevBatchPtr exec_impl(const PlanNode& n, int part) {
    x.check_cancel();
    OpMetrics* met = x.m(&n);
    DevBatchPtr out;
    switch (n.op) {
      case PlanNode::Scan: {
        std::lock_guard<std::mutex> g(x.e->mu);
        auto it = x.e->tables.find(n.table);
        if (it == x.e->tables.end()) throw EngineError(B200_ERR_INVALID, "table not registered: " + n.table);
        auto pit = it->second.find(part);
        if (pit == it->second.end()) {
          out = empty_batch(n.schema);
          break;
        }
        out = std::make_shared<DevBatch>();
        out->n = pit->second->n;
        for (size_t k = 0; k < n.scan_projection.size(); k++) {
          int idx = n.scan_projection[k];
          if ((size_t)idx >= pit->second->cols.size()) throw EngineError(B200_ERR_INVALID, "scan projection out of range for " + n.table);
          DevColumn c = pit->second->cols[(size_t)idx];
          if (c.type != n.schema[k].type)
            throw EngineError(B200_ERR_INVALID, "scan: column " + n.schema[k].name + " has type " + c.type.str() + ", plan says " + n.schema[k].type.str());
          c.name = n.schema[k].name;
          out->cols.push_back(c);
        }
        break;
      }
      case PlanNode::ShuffleReader: {
        std::vector<Piece> pieces;
        for (Piece& p : x.e->shuffle.pieces(ShuffleKey{job, n.reader_stage_id, n.broadcast ? 0 : part}))
          if (p.r1 > p.r0) pieces.push_back(std::move(p));
        if (pieces.empty()) out = empty_batch(n.schema);
        else out = concat_slices(x, pieces, n.schema);
        for (size_t c = 0; c < out->cols.size() && c < n.schema.size(); c++) {
          if (out->cols[c].type != n.schema[c].type)
            throw EngineError(B200_ERR_INVALID, "shuffle reader: column " + n.schema[c].name + " has type " + out->cols[c].type.str() + ", plan says " + n.schema[c].type.str());
          out->cols[c].name = n.schema[c].name;
        }
        break;
      }
      case PlanNode::Filter:
      case PlanNode::Projection: {
        if (n.op == PlanNode::Filter && n.fetch >= 0) {
          // FilterExec { fetch } (datafusion.proto:1027-1034): the first `fetch` rows that pass, in input order -- the
          // materialising sinks keep the input order, so the prefix of the filtered batch is exactly that
          std::vector<const PlanNode*> chain;
          chain.push_back(&n);
          const PlanNode* base = chain_base(*n.children[0], chain);
          DevBatchPtr src = exec(*base, part);
          for (auto* c : chain)
            if (OpMetrics* m = x.m(c)) m->input_rows += (uint64_t)src->n;
          PipelineBuilder pb(*src, x.st(), &x.e->regex);
          apply_chain(pb, chain);
          DevBatchPtr all = run_materialize(x, pb, named_cols(pb, n.schema), src, met);
          const int64_t keep = std::min<int64_t>(all->n, n.fetch);
          out = std::make_shared<DevBatch>();
          out->n = keep;
          for (auto& c : all->cols) out->cols.push_back(slice_column(c, 0, keep));
          break;
        }
        out = with_chain(n, part, false, [&](const BuilderFactory& mk, DevBatchPtr& src) {
          auto pb = mk();
          return run_materialize(x, *pb, named_cols(*pb, n.schema), src, met);
        });
        break;
      }
      case PlanNode::Aggregate: {
        const PlanNode& child = *n.children[0];
        bool all = (n.agg_mode == AggMode::Final || n.agg_mode == AggMode::Single) && part == 0 && n_partitions(child) > 1;
        out = with_chain(child, part, all, [&](const BuilderFactory& mk, DevBatchPtr& src) { return run_aggregate(x, mk, n, src, met); });
        break;
      }
      case PlanNode::HashJoin:
        out = n.nested_loop ? exec_nlj(n, part, met) : exec_join(n, part, met);
        if (!n.sort_keys.empty()) out = do_sort(n.sort_keys, -1, out, met);  // SortMergeJoinExec: ordered by the join keys
        break;
      case PlanNode::Sort: {
        DevBatchPtr in = exec(*n.children[0], part);
        out = do_sort(n.sort_keys, n.fetch, in, met);
        break;
      }
      case PlanNode::SortPreservingMerge: {
        DevBatchPtr in = exec_all(*n.children[0]);
        out = do_sort(n.sort_keys, n.fetch, in, met);
        break;
      }
      case PlanNode::Passthrough:
        out = (n.op_name == "CoalescePartitionsExec") ? exec_all(*n.children[0]) : exec(*n.children[0], part);
        break;
      case PlanNode::Limit: {
        DevBatchPtr in = (n.op_name == "GlobalLimitExec") ? exec_all(*n.children[0]) : exec(*n.children[0], part);
        int64_t r0 = std::min<int64_t>(std::max<int64_t>(0, n.skip), in->n);
        int64_t r1 = n.fetch >= 0 ? std::min<int64_t>(in->n, r0 + n.fetch) : in->n;
        out = std::make_shared<DevBatch>();
        out->n = r1 - r0;
        for (auto& c : in->cols) out->cols.push_back(slice_column(c, r0, r1));
        break;
      }
      case PlanNode::Window: out = exec_window(n, part, met); break;
      case PlanNode::ShuffleWriter: throw EngineError(B200_ERR_INVALID, "nested ShuffleWriterExec");
    }
    if (met) met->output_rows += (uint64_t)out->n;
    return out;
  }

  // ---- sort -----------------------------------------------------------------------------------
  DevBatchPtr do_sort(const std::vector<SortKey>& keys, int64_t fetch, DevBatchPtr in, OpMetrics* met) {
    const int64_t n = in->n;
    auto t0 = std::chrono::steady_clock::now();
    // key columns: plain column references are used in place, anything else is computed first
    std::vector<DevColumn> kcols;
    bool need_eval = false;
    for (auto& k : keys) need_eval |= k.expr->kind != Expr::Col;
    DevBatchPtr work = in;
    size_t n_in_cols = in->cols.size();
    if (need_eval && n > 0) {
      PipelineBuilder pb(*in, x.st(), &x.e->regex);
      std::vector<ColRef> outs = pb.cols;
      for (auto& k : keys) {
        ColRef c = pb.compile(*k.expr);
        pb.pin(c);
        outs.push_back(c);
      }
      work = run_materialize(x, pb, outs, in, met);
      for (size_t k = 0; k < keys.size(); k++) kcols.push_back(work->cols[n_in_cols + k]);
    } else {
      for (auto& k : keys) kcols.push_back(in->cols.at((size_t)(k.expr->kind == Expr::Col ? k.expr->col : 0)));
    }
    if (n <= 1 || keys.empty()) {
      auto out = std::make_shared<DevBatch>();
      int64_t m = fetch >= 0 ? std::min<int64_t>(fetch, n) : n;
      out->n = m;
      for (size_t c = 0; c < n_in_cols; c++) out->cols.push_back(slice_column(in->cols[c], 0, m));
      return out;
    }
    const int64_t m = fetch >= 0 ? std::min<int64_t>(fetch, n) : n;
    DevPtr idx = sort_permutation(keys, kcols, n, m);
    DevBatch proj;
    proj.n = n;
    for (size_t c = 0; c < n_in_cols; c++) proj.cols.push_back(in->cols[c]);
    DevBatchPtr out = gather_batch(x, proj, (const int64_t*)idx->ptr, m, false);
    if (n > SMALL_SORT_MAX_ROWS || keys.size() > (size_t)SMALL_SORT_MAX_KEYS) CUDA_CHECK(host_wait(x.e, x.st()));
    if (met) {
      met->elapsed_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
      met->input_rows += (uint64_t)n;
    }
    return out;
  }

  // ---- window functions (WindowAggExec / BoundedWindowAggExec) ---------------------------------------------------------
  // True when the input is a sort (through CoalesceBatchesExec) by the partition keys, in any order and direction, then
  // exactly the window's ORDER BY: its rows already are in the window's order and the operator sorts nothing.
  static bool window_input_sorted(const PlanNode& n) {
    const PlanNode* c = n.children[0].get();
    while (c->op == PlanNode::Passthrough && c->op_name == "CoalesceBatchesExec") c = c->children[0].get();
    if (c->op != PlanNode::Sort && c->op != PlanNode::SortPreservingMerge) return false;
    const size_t np = n.window_partition.size(), no = n.window_order.size();
    if (c->sort_keys.size() != np + no) return false;
    auto in_sort_prefix = [&](const ExprPtr& e) {
      for (size_t k = 0; k < np; k++)
        if (expr_equal(c->sort_keys[k].expr, e)) return true;
      return false;
    };
    for (size_t k = 0; k < np; k++) {
      bool found = false;
      for (auto& pk : n.window_partition) found = found || expr_equal(c->sort_keys[k].expr, pk);
      if (!found || !in_sort_prefix(n.window_partition[k])) return false;
    }
    for (size_t k = 0; k < no; k++) {
      const SortKey &a = c->sort_keys[np + k], &b = n.window_order[k];
      if (!expr_equal(a.expr, b.expr) || a.asc != b.asc || a.nulls_first != b.nulls_first) return false;
    }
    return true;
  }

  DevBatchPtr exec_window(const PlanNode& n, int part, OpMetrics* met) {
    DevBatchPtr in = exec(*n.children[0], part);
    const auto t0 = std::chrono::steady_clock::now();
    const int64_t N = in->n;
    if (N >= ((int64_t)1 << 32)) throw EngineError(B200_ERR_UNSUPPORTED, "window over " + std::to_string(N) + " rows (the sort takes at most 2^32)");
    const size_t np = n.window_partition.size(), no = n.window_order.size(), nw = n.window_exprs.size();
    if (np + no > (size_t)WIN_MAX_KEYS) throw EngineError(B200_ERR_UNSUPPORTED, "window with more than " + std::to_string(WIN_MAX_KEYS) + " partition and order keys");
    auto out = std::make_shared<DevBatch>();
    out->n = N;
    out->cols = in->cols;
    const size_t n_in = in->cols.size();
    if (met) met->input_rows += (uint64_t)N;
    if (N == 0) {
      for (size_t w = 0; w < nw; w++) {
        const Field& f = n.schema[n_in + w];
        DevColumn c = make_out_column(f.name, f.type, f.type.id == TypeId::Utf8 ? PH_STRVIEW : phys_of(f.type), 0, f.nullable, x.st());
        c.n = 0;
        out->cols.push_back(c);
      }
      return out;
    }
    // the columns the kernels read: partition keys, order keys, then the first argument of each function
    std::vector<ExprPtr> exprs(n.window_partition);
    for (auto& k : n.window_order) exprs.push_back(k.expr);
    std::vector<size_t> arg_at(nw, 0);
    for (size_t w = 0; w < nw; w++)
      if (!n.window_exprs[w].args.empty()) {
        arg_at[w] = exprs.size();
        exprs.push_back(n.window_exprs[w].args[0]);
      }
    std::vector<DevColumn> cols;
    bool need_eval = false;
    for (auto& e : exprs) need_eval |= e->kind != Expr::Col;
    if (need_eval) {
      PipelineBuilder pb(*in, x.st(), &x.e->regex);
      std::vector<ColRef> outs;
      for (auto& e : exprs) {
        ColRef c = pb.compile(*e);
        pb.pin(c);
        outs.push_back(c);
      }
      cols = run_materialize(x, pb, outs, in, met)->cols;
    } else {
      for (auto& e : exprs) cols.push_back(in->cols.at((size_t)e->col));
    }
    // the order: the input's own when a matching sort feeds the window, else the device sort's permutation
    DevPtr perm_buf;
    const int64_t* perm = nullptr;
    if (np + no > 0 && N > 1 && !window_input_sorted(n)) {
      x.check_cancel();
      std::vector<SortKey> keys;
      std::vector<DevColumn> kcols;
      for (size_t k = 0; k < np + no; k++) {
        SortKey sk;
        if (k < np) sk.expr = n.window_partition[k];  // any direction groups a partition's rows
        else sk = n.window_order[k - np];
        keys.push_back(sk);
        kcols.push_back(cols[k]);
      }
      KernelTimer kt(x, "window_sort", (uint64_t)N * 8 * 2 * (np + no));
      perm_buf = sort_permutation(keys, kcols, N, N);
      perm = (const int64_t*)perm_buf->ptr;
      x.e->n_window_sorts++;
    }
    // partition and peer-group boundaries
    x.check_cancel();
    WinKeys K;
    memset(&K, 0, sizeof K);
    K.n_part = (int)np;
    K.n_order = (int)no;
    std::vector<DevColumn> kviews;
    uint64_t key_bytes = 0;
    for (size_t k = 0; k < np + no; k++) kviews.push_back(as_views(x, cols[k]));
    for (size_t k = 0; k < np + no; k++) {
      const DevColumn& c = kviews[k];
      K.k[k] = KeyCol{c.data, c.valid, (uint8_t)c.phys, (uint8_t)c.width()};
      key_bytes += 2ull * ((uint64_t)c.width() + (c.valid ? 1 : 0));
    }
    const size_t N1 = (size_t)N + 1;
    DevPtr part_flag = dev_alloc((size_t)N * 4, x.st()), peer_flag = dev_alloc((size_t)N * 4, x.st());
    DevPtr part_ex = dev_alloc(N1 * 8, x.st()), peer_ex = dev_alloc(N1 * 8, x.st()), scan_scratch = dev_alloc(((size_t)N / 1024 + 4) * 8, x.st());
    DevPtr pid = dev_alloc((size_t)N * 4, x.st()), gid = dev_alloc((size_t)N * 4, x.st());
    DevPtr part_start = dev_alloc(N1 * 4, x.st()), peer_start = dev_alloc(N1 * 4, x.st()), first_peer = dev_alloc((size_t)N * 4, x.st());
    WinBounds B;
    B.pid = (uint32_t*)pid->ptr;
    B.gid = (uint32_t*)gid->ptr;
    B.part_start = (uint32_t*)part_start->ptr;
    B.peer_start = (uint32_t*)peer_start->ptr;
    B.part_first_peer = (uint32_t*)first_peer->ptr;
    {
      // flags (keys of two rows, two flags), two scans (flag in, offset out, and back), segments (flags, offsets, ids, starts)
      KernelTimer kt(x, "window_bounds", (uint64_t)N * (key_bytes + (perm ? 16 : 0) + 8 + 2 * (4 + 16) + (16 + 16 + 8 + 12)));
      launch_window_flags(K, perm, N, (uint32_t*)part_flag->ptr, (uint32_t*)peer_flag->ptr, x.st());
      launch_scan_u32_to_u64((const uint32_t*)part_flag->ptr, (uint64_t*)part_ex->ptr, N, (uint64_t*)scan_scratch->ptr, x.st());
      launch_scan_u32_to_u64((const uint32_t*)peer_flag->ptr, (uint64_t*)peer_ex->ptr, N, (uint64_t*)scan_scratch->ptr, x.st());
      launch_window_segments((const uint32_t*)part_flag->ptr, (const uint32_t*)peer_flag->ptr, (const uint64_t*)part_ex->ptr, (const uint64_t*)peer_ex->ptr, N, B,
                             x.st());
    }
    DevPtr error;
    for (size_t w = 0; w < nw; w++) {
      x.check_cancel();
      const WindowExpr& we = n.window_exprs[w];
      const Field& f = n.schema[n_in + w];
      WinEval E;
      memset(&E, 0, sizeof E);
      const int64_t kMaxOff = (int64_t)1 << 40;  // beyond any partition (< 2^32 rows): no overflow in the frame arithmetic
      E.units = we.frame.range ? WUNITS_RANGE : WUNITS_ROWS;
      E.s_kind = we.frame.start.kind;
      E.e_kind = we.frame.end.kind;
      E.s_off = (int64_t)std::min<uint64_t>(we.frame.start.n, (uint64_t)kMaxOff);
      E.e_off = (int64_t)std::min<uint64_t>(we.frame.end.n, (uint64_t)kMaxOff);
      E.arg = we.n;
      E.acc = WACC_I64;
      static const uint8_t fn_kind[] = {WF_ROW_NUMBER, WF_RANK, WF_DENSE_RANK, WF_PERCENT_RANK, WF_CUME_DIST, WF_NTILE, WF_OFFSET, WF_OFFSET,
                                        WF_FIRST,      WF_LAST, WF_NTH,        WF_AGG,          WF_AGG,       WF_AGG,   WF_AGG,    WF_AGG};
      E.fn = fn_kind[(int)we.fn];
      if (E.fn == WF_OFFSET || E.fn == WF_FIRST || E.fn == WF_LAST || E.fn == WF_NTH) {
        DevPtr idx = dev_alloc((size_t)N * 8, x.st());
        E.idx_out = (int64_t*)idx->ptr;
        {
          KernelTimer kt(x, "window_frames", (uint64_t)N * (8 + 8 + 16 + (perm ? 16 : 0)));
          launch_window_eval(E, B, perm, N, x.st());
        }
        DevBatch one;
        one.n = N;
        one.cols.push_back(cols[arg_at[w]]);
        DevColumn oc = gather_batch(x, one, (const int64_t*)idx->ptr, N, true)->cols[0];
        if (we.default_value) {
          const LitValue& l = we.default_value->lit;
          uint64_t lit[2] = {0, 0};
          switch (we.result_type.pk()) {
            case PK::F64:
              if (we.result_type.id == TypeId::Float32) {
                const float v = (float)l.f;
                memcpy(lit, &v, 4);
              } else {
                memcpy(lit, &l.f, 8);
              }
              break;
            case PK::I128: memcpy(lit, &l.d, 16); break;
            case PK::Str: {
              DevPtr chars = dev_alloc(l.s.size() + 1, x.st());
              if (!l.s.empty()) CUDA_CHECK(cudaMemcpyAsync(chars->ptr, l.s.data(), l.s.size(), cudaMemcpyHostToDevice, x.st()));
              lit[0] = (uint64_t)(uintptr_t)chars->ptr;
              lit[1] = (uint64_t)l.s.size();
              oc.keep.push_back(chars);
              break;
            }
            default: memcpy(lit, &l.i, 8); break;  // little-endian: the low bytes are the narrower integer
          }
          launch_window_fill((const int64_t*)idx->ptr, N, (void*)oc.data, (uint8_t*)oc.valid, oc.width(), lit, x.st());
        }
        oc.name = f.name;
        out->cols.push_back(oc);
        continue;
      }
      const Phys out_phys = phys_of(f.type);
      // only the aggregates write a validity (ntile is typed nullable but never NULL)
      DevColumn oc = make_out_column(f.name, f.type, out_phys, N, f.nullable && E.fn == WF_AGG, x.st());
      oc.n = N;
      E.out = (void*)oc.data;
      E.out_valid = (uint8_t*)oc.valid;
      E.out_phys = out_phys;
      if (E.fn != WF_AGG) {
        KernelTimer kt(x, "window_frames", (uint64_t)N * (8 + 16 + (perm ? 8 : 0)));
        launch_window_eval(E, B, perm, N, x.st());
        out->cols.push_back(oc);
        continue;
      }
      // framed aggregates: the argument in sorted order, then forward / backward segmented scans by frame kind
      const DevColumn* arg = we.args.empty() ? nullptr : &cols[arg_at[w]];
      const DataType at = arg ? arg->type : DataType(TypeId::Int64);
      WinLoad L;
      memset(&L, 0, sizeof L);
      if (arg) {
        L.data = arg->data;
        L.valid = arg->valid;
        L.phys = (uint8_t)arg->phys;
      }
      E.op = WOP_SUM;
      E.fin = WFIN_VALUE;
      switch (we.fn) {
        case WinFn::Count:
          L.conv = arg ? WCV_VALID : WCV_ONE;
          E.fin = WFIN_COUNT;
          break;
        case WinFn::Sum:
        case WinFn::Avg:
          if (at.is_decimal()) {
            E.acc = WACC_I128;
            L.conv = WCV_I128;
          } else if (we.fn == WinFn::Avg || at.is_float()) {
            E.acc = WACC_F64;
            L.conv = WCV_F64;
          } else {
            L.conv = WCV_I64;
          }
          if (we.fn == WinFn::Avg) {
            E.fin = WFIN_AVG;
            E.imm = we.result_type.scale - at.scale;
            E.prec = we.result_type.precision;
          }
          break;
        default:  // Min, Max
          E.op = we.fn == WinFn::Min ? WOP_MIN : WOP_MAX;
          if (at.is_decimal()) {
            E.acc = WACC_I128;
            L.conv = WCV_I128;
          } else if (at.is_float()) {
            L.conv = WCV_F64_KEY;
            E.fin = WFIN_MINMAX_F64;
          } else if (at.id == TypeId::UInt64) {
            L.conv = WCV_U64_KEY;
            E.fin = WFIN_MINMAX_U64;
          } else {
            L.conv = WCV_I64;
          }
      }
      if (arg && arg->phys == PH_UTF8 && L.conv != WCV_VALID) throw EngineError(B200_ERR_UNSUPPORTED, "window " + we.fn_name + " over Utf8");
      const size_t vw = E.acc == WACC_I128 ? 16 : 8;
      DevPtr vals = dev_alloc((size_t)N * vw, x.st()), valid = dev_alloc((size_t)N, x.st());
      L.out = vals->ptr;
      L.out_valid = (uint8_t*)valid->ptr;
      // which scans the frame needs (the frame kinds of DESIGN.md §4.8)
      const uint8_t sk = we.frame.start.kind, ek = we.frame.end.kind;
      bool fwd = false, bwd = false;
      uint8_t seg = WSEG_PART;
      if (sk == WB_UNBOUNDED_PRECEDING) {
        fwd = true;
        E.read = WRD_FWD;
      } else if (ek == WB_UNBOUNDED_FOLLOWING) {
        bwd = true;
        E.read = WRD_BWD;
      } else if (we.frame.range) {  // RANGE CURRENT ROW .. CURRENT ROW: the peer group
        fwd = true;
        seg = WSEG_PEER;
        E.read = WRD_FWD;
      } else {  // ROWS bounded on both sides: a fixed width
        const int64_t so = sk == WB_PRECEDING ? -E.s_off : sk == WB_CURRENT_ROW ? 0 : E.s_off;
        const int64_t eo = ek == WB_PRECEDING ? -E.e_off : ek == WB_CURRENT_ROW ? 0 : E.e_off;
        E.w = std::min<int64_t>(eo - so + 1, N);
        fwd = bwd = E.w > 0;  // w <= 0: every frame is empty, nothing to scan
        seg = WSEG_BLOCK;
        E.read = WRD_BLOCKS;
      }
      DevPtr fv, fc, bv, bc, tiles;
      {
        KernelTimer kt(x, "window_scan", (uint64_t)N * ((arg ? (uint64_t)arg->width() + 1 : 0) + (perm ? 8 : 0) + vw + 1) +
                                             (uint64_t)N * (fwd + bwd) * 2 * (vw + 1 + 8 + vw + 4));
        launch_window_load(L, perm, N, x.st());
        WinScan S;
        memset(&S, 0, sizeof S);
        S.vals = vals->ptr;
        S.valid = (const uint8_t*)valid->ptr;
        S.n = N;
        S.w = std::max<int64_t>(E.w, 1);
        S.acc = E.acc;
        S.op = E.op;
        S.seg = seg;
        if (fwd || bwd) tiles = dev_alloc((size_t)window_scan_tile_bytes(N), x.st());
        S.tiles = tiles ? tiles->ptr : nullptr;
        if (fwd) {
          fv = dev_alloc((size_t)N * vw, x.st());
          fc = dev_alloc((size_t)N * 4, x.st());
          S.out_v = fv->ptr;
          S.out_c = (uint32_t*)fc->ptr;
          S.dir = 0;
          launch_window_scan(S, B, x.st());
          E.fwd_v = fv->ptr;
          E.fwd_c = (const uint32_t*)fc->ptr;
        }
        x.check_cancel();
        if (bwd) {
          bv = dev_alloc((size_t)N * vw, x.st());
          bc = dev_alloc((size_t)N * 4, x.st());
          S.out_v = bv->ptr;
          S.out_c = (uint32_t*)bc->ptr;
          S.dir = 1;
          launch_window_scan(S, B, x.st());
          E.bwd_v = bv->ptr;
          E.bwd_c = (const uint32_t*)bc->ptr;
        }
      }
      if (E.fin == WFIN_AVG && E.acc == WACC_I128) {
        if (!error) {
          error = dev_alloc(16, x.st());
          CUDA_CHECK(cudaMemsetAsync(error->ptr, 0, 16, x.st()));
        }
        E.error = (unsigned int*)error->ptr;
      }
      {
        KernelTimer kt(x, "window_frames", (uint64_t)N * (32 + 2 * (vw + 4) + (perm ? 8 : 0) + (uint64_t)oc.width() + 1));
        launch_window_eval(E, B, perm, N, x.st());
      }
      out->cols.push_back(oc);
    }
    if (error && x.get<unsigned int>(error->ptr)) throw EngineError(B200_ERR_EXECUTION, "Arithmetic overflow in a window AVG over Decimal128");
    CUDA_CHECK(host_wait(x.e, x.st()));  // the temporaries above are freed stream-ordered; the metrics take the device time
    if (met) met->elapsed_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
    return out;
  }

  // The stable sort permutation of n >= 2 rows by `keys`, evaluated in `kcols`: the input rows of sorted positions
  // [0, m) as int64 indices.  Rows with equal keys keep their input order.  SortExec and the window operator share it.
  DevPtr sort_permutation(const std::vector<SortKey>& keys, const std::vector<DevColumn>& kcols, int64_t n, int64_t m) {
    if (n >= ((int64_t)1 << 32)) throw EngineError(B200_ERR_UNSUPPORTED, "sort of more than 2^32 rows");
    if (n <= SMALL_SORT_MAX_ROWS && keys.size() <= (size_t)SMALL_SORT_MAX_KEYS) {
      // the tail of a query (ORDER BY over a few groups): one comparison-sort launch, no length read-backs
      SmallSortKeys K;
      K.n_keys = (int)keys.size();
      std::vector<DevColumn> kv;  // keeps the view buffers alive until the launch is enqueued
      for (size_t ki = 0; ki < keys.size(); ki++) {
        kv.push_back(as_views(x, kcols[ki]));
        const DevColumn& kc = kv.back();
        SortWordArgs& A = K.k[ki];
        A.data = kc.data;
        A.valid = kc.valid;
        A.phys = kc.phys;
        A.asc = keys[ki].asc;
        A.nulls_first = keys[ki].nulls_first;
        A.word = 0;
      }
      DevPtr idx = dev_alloc((size_t)n * 8, x.st());
      launch_small_sort(K, (int64_t*)idx->ptr, n, x.st());
      return idx;
    }
    const uint32_t n_blocks = (uint32_t)((n + 2047) / 2048);
    DevPtr ka = dev_alloc((size_t)n * 8, x.st()), kb = dev_alloc((size_t)n * 8, x.st());
    DevPtr va = dev_alloc((size_t)n * 4, x.st()), vb = dev_alloc((size_t)n * 4, x.st());
    DevPtr hist = dev_alloc((size_t)256 * n_blocks * 4 + 64, x.st());
    DevPtr scan = dev_alloc(((size_t)256 * n_blocks + 1 + (size_t)(256 * n_blocks) / 1024 + 8) * 8, x.st());
    uint32_t* perm = (uint32_t*)va->ptr;
    launch_iota_u32(perm, n, x.st());
    for (size_t ki = keys.size(); ki-- > 0;) {
      DevColumn kc = as_views(x, kcols[ki]);
      int n_words = 1;
      if (kc.phys == PH_DEC128) n_words = 2;
      if (kc.phys == PH_STRVIEW) {
        DevPtr mx = dev_alloc(16, x.st());
        CUDA_CHECK(cudaMemsetAsync(mx->ptr, 0, 16, x.st()));
        launch_max_view_len((const unsigned long long*)kc.data, kc.valid, n, (unsigned int*)mx->ptr, x.st());
        unsigned int maxlen = x.get<unsigned int>(mx->ptr);
        n_words = (int)(maxlen / 7) + 1;
      }
      // least significant word first; the NULL-rank word is the most significant
      for (int w = n_words - 1; w >= (kc.valid ? -1 : 0); w--) {
        x.check_cancel();
        SortWordArgs A;
        A.data = kc.data;
        A.valid = kc.valid;
        A.phys = kc.phys;
        A.asc = keys[ki].asc;
        A.nulls_first = keys[ki].nulls_first;
        A.word = w;
        uint64_t* kin = (uint64_t*)ka->ptr;
        launch_sort_word(A, perm, kin, n, x.st());
        bool in_a;
        if (perm == (uint32_t*)va->ptr) {
          radix_sort_pairs_u64((uint64_t*)ka->ptr, (uint32_t*)va->ptr, (uint64_t*)kb->ptr, (uint32_t*)vb->ptr, n, (uint32_t*)hist->ptr, (uint64_t*)scan->ptr, x.st(), &in_a);
          perm = in_a ? (uint32_t*)va->ptr : (uint32_t*)vb->ptr;
        } else {
          // current permutation lives in vb: sort with roles swapped (keys were written to ka)
          radix_sort_pairs_u64((uint64_t*)ka->ptr, (uint32_t*)vb->ptr, (uint64_t*)kb->ptr, (uint32_t*)va->ptr, n, (uint32_t*)hist->ptr, (uint64_t*)scan->ptr, x.st(), &in_a);
          perm = in_a ? (uint32_t*)vb->ptr : (uint32_t*)va->ptr;
        }
      }
    }
    DevPtr idx = dev_alloc((size_t)std::max<int64_t>(m, 1) * 8, x.st());
    launch_u32_to_i64(perm, (int64_t*)idx->ptr, m, x.st());
    return idx;
  }

  // ---- hash join --------------------------------------------------------------------------------
  // Evaluates `outs` of a pipeline: columns the chain forwards untouched (and that no filter compacts) are taken
  // from the source batch as they are, only computed columns go through the materialising kernel.
  struct Mixed {
    std::vector<DevColumn> cols;  // one per entry of `outs`
    int64_t n = 0;
  };
  Mixed materialize_mixed(PipelineBuilder& pb, const std::vector<ColRef>& outs, const DevBatchPtr& src, OpMetrics* met) {
    Mixed m;
    const bool filters = program_filters(pb.prog);
    std::vector<int> direct(outs.size(), -1);
    std::vector<ColRef> mouts;
    for (size_t c = 0; c < outs.size(); c++) {
      if (!filters) direct[c] = pb.source_index(outs[c]);
      if (direct[c] < 0) mouts.push_back(outs[c]);
    }
    DevBatchPtr mat;
    m.n = src->n;
    if (!mouts.empty()) {
      mat = run_materialize(x, pb, mouts, src, met);
      m.n = mat->n;
    }
    size_t mi = 0;
    for (size_t c = 0; c < outs.size(); c++) {
      DevColumn col = direct[c] >= 0 ? src->cols[(size_t)direct[c]] : mat->cols[mi++];
      col.name = outs[c].name;
      m.cols.push_back(col);
    }
    return m;
  }

  struct JoinSide {
    DevBatch payload;              // output columns of the side
    std::vector<DevColumn> keys;   // evaluated join keys (strings as views)
    const uint64_t* hash = nullptr;
    DevColumn hash_col;
    int64_t n = 0;
  };
  JoinSide prepare_side(const PlanNode& child, int part, bool all, const std::vector<ExprPtr>& key_exprs, bool need_hash, OpMetrics* met) {
    JoinSide js;
    with_chain(child, part, all, [&](const BuilderFactory& mk, DevBatchPtr& src) {
      auto pbp = mk();
      PipelineBuilder& pb = *pbp;
      std::vector<ColRef> outs = named_cols(pb, child.schema);
      const size_t n_payload = outs.size();
      std::vector<ColRef> keys;
      for (auto& ke : key_exprs) {
        ColRef k = pb.compile(*ke);
        pb.pin(k);
        keys.push_back(k);
      }
      for (auto& k : keys) outs.push_back(k);
      if (need_hash) {
        ColRef h = pb.hash_of(keys);
        h.name = "__hash";
        outs.push_back(h);
      }
      Mixed m = materialize_mixed(pb, outs, src, met);
      js.n = m.n;
      js.payload.n = m.n;
      for (size_t c = 0; c < n_payload; c++) js.payload.cols.push_back(m.cols[c]);
      for (size_t k = 0; k < keys.size(); k++) js.keys.push_back(as_views(x, m.cols[n_payload + k]));
      if (need_hash) {
        js.hash_col = m.cols.back();
        js.hash = (const uint64_t*)js.hash_col.data;
      }
      return src;
    });
    return js;
  }

  static bool exact_key(const DataType& t) {
    switch (t.id) {
      case TypeId::Int8: case TypeId::Int16: case TypeId::Int32: case TypeId::Int64: case TypeId::UInt8: case TypeId::UInt16: case TypeId::UInt32:
      case TypeId::UInt64: case TypeId::Date32: case TypeId::Timestamp: return true;
      default: return false;
    }
  }

  // unmatched or semi / anti build rows: a join whose whole build side is read by every task (CollectLeft, nested loop)
  // emits those rows once per task
  static bool emits_build_rows(JoinType jt) {
    return jt == JoinType::Left || jt == JoinType::Full || jt == JoinType::LeftSemi || jt == JoinType::LeftAnti;
  }

  DevBatchPtr exec_join(const PlanNode& n, int part, OpMetrics* met) {
    const bool collect_left = n.partition_mode == "CollectLeft";
    std::vector<ExprPtr> lk, rk;
    for (auto& on : n.on) {
      lk.push_back(on.first);
      rk.push_back(on.second);
    }
    const size_t nk = lk.size();
    if (nk > (size_t)VM_MAX_KEYS) throw EngineError(B200_ERR_UNSUPPORTED, "too many join keys");
    // CollectLeft replays the whole build side in every probe task; a join type that also EMITS build rows
    // (unmatched or semi/anti) would then emit them once per task.  DataFusion shares a visited bitmap across
    // the probe partitions of one process; tasks here are independent, so those shapes are only legal with a
    // single probe partition.
    if (collect_left && emits_build_rows(n.join_type) && n_partitions(*n.children[1]) > 1)
      throw EngineError(B200_ERR_UNSUPPORTED, "CollectLeft hash join that emits build-side rows over more than one probe partition: plan it as Partitioned");
    // one integer-like key: the table is keyed by the key itself (no hash column, no second look at the keys).  That
    // table keeps NULL keys out, so a join where NULL matches NULL takes the hash-tagged table, whose key check
    // (join_keys_equal) pairs two NULLs.
    const bool exact = nk == 1 && exact_key(lk[0]->type) && lk[0]->type.id == rk[0]->type.id && !n.null_equals_null;
    JoinSide L = prepare_side(*n.children[0], part, collect_left, lk, !exact, met);
    JoinSide R = prepare_side(*n.children[1], part, false, rk, !exact, met);
    const int64_t nb = L.n, np = R.n;
    if (nb >= ((int64_t)1 << 31)) throw EngineError(B200_ERR_UNSUPPORTED, "hash join build side exceeds 2^31 rows");
    auto t0 = std::chrono::steady_clock::now();
    JoinKeys K;
    memset(&K, 0, sizeof K);
    K.n_keys = (int)nk;
    K.null_equals_null = n.null_equals_null ? 1 : 0;
    uint64_t key_bytes_b = 0, key_bytes_p = 0;
    for (size_t k = 0; k < nk; k++) {
      const DevColumn& b = L.keys[k];
      const DevColumn& p = R.keys[k];
      // the exact-key table compares 64-bit images of the values (jkey_image widens each side by its own width), so a key
      // whose cast to the other side's type left its source column as it was (CAST(i32 AS i64)) still matches; the
      // hash-tagged table compares key bytes and needs one physical type
      if (!exact && b.phys != p.phys) throw EngineError(B200_ERR_UNSUPPORTED, "join key physical types differ (" + b.type.str() + " vs " + p.type.str() + "): add casts");
      K.build[k] = KeyCol{b.data, b.valid, (uint8_t)b.phys, (uint8_t)b.width()};
      K.probe[k] = KeyCol{p.data, p.valid, (uint8_t)p.phys, (uint8_t)p.width()};
      key_bytes_b += (uint64_t)b.width();
      key_bytes_p += (uint64_t)p.width();
    }
    x.check_cancel();
    const uint64_t n_buckets = next_pow2((uint64_t)std::max<int64_t>(nb, 1) * 2);
    DevPtr heads = dev_alloc((size_t)n_buckets * 4, x.st());
    DevPtr nodes = dev_alloc((size_t)std::max<int64_t>(nb, 1) * sizeof(JoinNode), x.st());
    {
      KernelTimer kt(x, "join_build", (uint64_t)nb * (key_bytes_b + sizeof(JoinNode)) + n_buckets * 4);
      CUDA_CHECK(cudaMemsetAsync(heads->ptr, 0xFF, (size_t)n_buckets * 4, x.st()));
      launch_join_build2(K, exact, L.hash, nb, (int32_t*)heads->ptr, n_buckets, (JoinNode*)nodes->ptr, x.st());
    }
    x.check_cancel();
    const bool has_filter = n.join_filter != nullptr;
    const JoinType jt = n.join_type;
    const bool semi_anti = jt == JoinType::LeftSemi || jt == JoinType::LeftAnti || jt == JoinType::RightSemi || jt == JoinType::RightAnti;
    const bool left_outer = jt == JoinType::Left || jt == JoinType::Full, right_outer = jt == JoinType::Right || jt == JoinType::Full;
    const bool want_bmark = jt == JoinType::LeftSemi || jt == JoinType::LeftAnti || left_outer;
    const bool want_pmark = jt == JoinType::RightSemi || jt == JoinType::RightAnti || right_outer;
    // with a residual filter the marks must come from the pairs that survive it
    const bool need_pairs = has_filter || !semi_anti;
    int mode = need_pairs ? 1 : 0;
    DevPtr bmark, pmark;
    if (!has_filter && want_bmark) {
      bmark = dev_alloc((size_t)std::max<int64_t>(nb, 1), x.st());
      CUDA_CHECK(cudaMemsetAsync(bmark->ptr, 0, (size_t)std::max<int64_t>(nb, 1), x.st()));
      mode |= 4;
    }
    if (!has_filter && want_pmark) {
      pmark = dev_alloc((size_t)std::max<int64_t>(np, 1), x.st());
      CUDA_CHECK(cudaMemsetAsync(pmark->ptr, 0, (size_t)std::max<int64_t>(np, 1), x.st()));
      mode |= 2;
    }
    int64_t n_pairs = 0;
    DevPtr bi, pi;
    if (mode) {
      DevPtr counter = dev_alloc(16, x.st());
      uint64_t cap = need_pairs ? (uint64_t)std::max<int64_t>(np + nb / 8 + 1024, 1) : 0;
      for (int attempt = 0;; attempt++) {
        if (need_pairs) {
          bi = dev_alloc((size_t)std::max<uint64_t>(cap, 1) * 8, x.st());
          pi = dev_alloc((size_t)std::max<uint64_t>(cap, 1) * 8, x.st());
        }
        CUDA_CHECK(cudaMemsetAsync(counter->ptr, 0, 16, x.st()));
        {
          KernelTimer kt(x, "join_probe", (uint64_t)np * (key_bytes_p + 4 + sizeof(JoinNode)));
          launch_join_probe2(K, exact, mode, (const JoinNode*)nodes->ptr, (const int32_t*)heads->ptr, n_buckets, R.hash, np, (unsigned long long*)counter->ptr, cap,
                             need_pairs ? (int64_t*)bi->ptr : nullptr, need_pairs ? (int64_t*)pi->ptr : nullptr, pmark ? (uint8_t*)pmark->ptr : nullptr,
                             bmark ? (uint8_t*)bmark->ptr : nullptr, x.st());
        }
        if (!need_pairs) break;
        n_pairs = (int64_t)x.get<unsigned long long>(counter->ptr);
        if ((uint64_t)n_pairs <= cap) break;
        if (attempt) throw EngineError(B200_ERR_EXECUTION, "hash join: pair count changed between passes");
        cap = (uint64_t)n_pairs;  // many-to-many join: run again with the exact size
      }
    }
    x.check_cancel();
    const int64_t* bidx = need_pairs ? (const int64_t*)bi->ptr : nullptr;
    const int64_t* pidx = need_pairs ? (const int64_t*)pi->ptr : nullptr;
    const DevBatch& Lp = L.payload;
    const DevBatch& Rp = R.payload;
    DevPtr fbi, fpi;  // filtered pair lists
    if (has_filter && n_pairs > 0) {
      // evaluate the residual filter on the candidate pairs, carrying the pair indices through
      DevBatchPtr lg = gather_batch(x, Lp, bidx, n_pairs, false), rg = gather_batch(x, Rp, pidx, n_pairs, false);
      auto cat = std::make_shared<DevBatch>();
      cat->n = n_pairs;
      for (auto& c : lg->cols) cat->cols.push_back(c);
      for (auto& c : rg->cols) cat->cols.push_back(c);
      DevColumn ib, ip;
      ib.type = ip.type = DataType(TypeId::Int64);
      ib.phys = ip.phys = PH_I64;
      ib.n = ip.n = n_pairs;
      ib.data = (const uint8_t*)bi->ptr;
      ip.data = (const uint8_t*)pi->ptr;
      ib.keep.push_back(bi);
      ip.keep.push_back(pi);
      ib.name = "__bi";
      ip.name = "__pi";
      cat->cols.push_back(ib);
      cat->cols.push_back(ip);
      PipelineBuilder pb(*cat, x.st(), &x.e->regex);
      pb.apply_filter(*n.join_filter);
      std::vector<ColRef> outs = {pb.cols[cat->cols.size() - 2], pb.cols[cat->cols.size() - 1]};
      DevBatchPtr kept = run_materialize(x, pb, outs, cat, met);
      n_pairs = kept->n;
      fbi = kept->cols[0].keep[0];
      fpi = kept->cols[1].keep[0];
      bidx = (const int64_t*)kept->cols[0].data;
      pidx = (const int64_t*)kept->cols[1].data;
    }
    return join_output(n, Lp, Rp, bidx, pidx, n_pairs, bmark, pmark, t0, met);
  }

  // The join's output from its matching pairs (bidx[k], pidx[k]), k < n_pairs, shared by the hash join and the nested-loop
  // join: semi / anti selection, outer rows (unmatched build rows, then unmatched probe rows, after the pairs) and the
  // gather of the columns the projection keeps.  bmark / pmark: "has a pair" marks of build / probe rows when the caller
  // already has them; otherwise they are derived from the pairs.
  DevBatchPtr join_output(const PlanNode& n, const DevBatch& Lp, const DevBatch& Rp, const int64_t* bidx, const int64_t* pidx, int64_t n_pairs,
                          const DevPtr& bmark, const DevPtr& pmark, std::chrono::steady_clock::time_point t0, OpMetrics* met) {
    const JoinType jt = n.join_type;
    const int64_t nb = Lp.n, np = Rp.n;
    const bool left_outer = jt == JoinType::Left || jt == JoinType::Full, right_outer = jt == JoinType::Right || jt == JoinType::Full;
    auto flags_to_indices = [&](const uint8_t* marks, int64_t nrows, bool want, int64_t* n_sel) {
      DevPtr f = dev_alloc((size_t)(nrows + 1) * 4, x.st());
      DevPtr o = dev_alloc((size_t)(nrows + 2) * 8, x.st());
      DevPtr sc = dev_alloc((size_t)(nrows / 1024 + 4) * 8, x.st());
      launch_flag_to_u32(marks, want ? 1 : 0, (uint32_t*)f->ptr, nrows, x.st());
      launch_scan_u32_to_u64((const uint32_t*)f->ptr, (uint64_t*)o->ptr, nrows, (uint64_t*)sc->ptr, x.st());
      *n_sel = (int64_t)x.get<uint64_t>((const uint64_t*)o->ptr + nrows);
      DevPtr idx = dev_alloc((size_t)std::max<int64_t>(*n_sel, 1) * 8, x.st());
      launch_select_indices((const uint32_t*)f->ptr, (const uint64_t*)o->ptr, (int64_t*)idx->ptr, nrows, x.st());
      return idx;
    };
    auto marks_of = [&](const int64_t* idx, int64_t nrows, const DevPtr& from_probe) {
      if (from_probe) return from_probe;  // the probe pass already marked them
      DevPtr m = dev_alloc((size_t)std::max<int64_t>(nrows, 1), x.st());
      CUDA_CHECK(cudaMemsetAsync(m->ptr, 0, (size_t)std::max<int64_t>(nrows, 1), x.st()));
      if (n_pairs > 0) {
        launch_mark_from_idx(idx, n_pairs, (uint8_t*)m->ptr, x.st());
      }
      return m;
    };
    DevBatchPtr out;
    switch (jt) {
      case JoinType::LeftSemi:
      case JoinType::LeftAnti: {
        DevPtr m = marks_of(bidx, nb, bmark);
        int64_t ns = 0;
        DevPtr idx = flags_to_indices((const uint8_t*)m->ptr, nb, jt == JoinType::LeftSemi, &ns);
        out = gather_batch(x, Lp, (const int64_t*)idx->ptr, ns, false);
        break;
      }
      case JoinType::RightSemi:
      case JoinType::RightAnti: {
        DevPtr m = marks_of(pidx, np, pmark);
        int64_t ns = 0;
        DevPtr idx = flags_to_indices((const uint8_t*)m->ptr, np, jt == JoinType::RightSemi, &ns);
        out = gather_batch(x, Rp, (const int64_t*)idx->ptr, ns, false);
        break;
      }
      default: {
        // inner pairs (+ unmatched rows for outer joins, index -1 on the missing side)
        int64_t extra_l = 0, extra_r = 0;
        DevPtr ul, ur;
        if (left_outer) {
          DevPtr m = marks_of(bidx, nb, bmark);
          ul = flags_to_indices((const uint8_t*)m->ptr, nb, false, &extra_l);
        }
        if (right_outer) {
          DevPtr m = marks_of(pidx, np, pmark);
          ur = flags_to_indices((const uint8_t*)m->ptr, np, false, &extra_r);
        }
        const int64_t total = n_pairs + extra_l + extra_r;
        const int64_t* li_p = bidx;
        const int64_t* ri_p = pidx;
        DevPtr li, ri;
        if (extra_l || extra_r) {
          li = dev_alloc((size_t)std::max<int64_t>(total, 1) * 8, x.st());
          ri = dev_alloc((size_t)std::max<int64_t>(total, 1) * 8, x.st());
          if (n_pairs) {
            CUDA_CHECK(cudaMemcpyAsync(li->ptr, bidx, (size_t)n_pairs * 8, cudaMemcpyDeviceToDevice, x.st()));
            CUDA_CHECK(cudaMemcpyAsync(ri->ptr, pidx, (size_t)n_pairs * 8, cudaMemcpyDeviceToDevice, x.st()));
          }
          if (extra_l) {
            CUDA_CHECK(cudaMemcpyAsync((int64_t*)li->ptr + n_pairs, ul->ptr, (size_t)extra_l * 8, cudaMemcpyDeviceToDevice, x.st()));
            CUDA_CHECK(cudaMemsetAsync((int64_t*)ri->ptr + n_pairs, 0xFF, (size_t)extra_l * 8, x.st()));
          }
          if (extra_r) {
            CUDA_CHECK(cudaMemsetAsync((int64_t*)li->ptr + n_pairs + extra_l, 0xFF, (size_t)extra_r * 8, x.st()));
            CUDA_CHECK(cudaMemcpyAsync((int64_t*)ri->ptr + n_pairs + extra_l, ur->ptr, (size_t)extra_r * 8, cudaMemcpyDeviceToDevice, x.st()));
          }
          li_p = (const int64_t*)li->ptr;
          ri_p = (const int64_t*)ri->ptr;
        }
        // only the columns the join's projection keeps are gathered
        std::vector<int> want;
        const size_t nl = Lp.cols.size(), nr = Rp.cols.size();
        if (n.has_projection) want = n.projection;
        else
          for (size_t c = 0; c < nl + nr; c++) want.push_back((int)c);
        DevBatch Ls, Rs;
        Ls.n = nb;
        Rs.n = np;
        std::vector<std::pair<int, size_t>> where;  // per wanted column: (side, index inside the side's gathered batch)
        for (int idx : want) {
          if ((size_t)idx < nl) {
            where.push_back({0, Ls.cols.size()});
            Ls.cols.push_back(Lp.cols[(size_t)idx]);
          } else {
            where.push_back({1, Rs.cols.size()});
            Rs.cols.push_back(Rp.cols.at((size_t)idx - nl));
          }
        }
        KernelTimer kt(x, "join_gather", 0);
        DevBatchPtr lg = gather_batch(x, Ls, li_p, total, right_outer);
        DevBatchPtr rg = gather_batch(x, Rs, ri_p, total, left_outer);
        out = std::make_shared<DevBatch>();
        out->n = total;
        for (auto& w : where) out->cols.push_back(w.first == 0 ? lg->cols[w.second] : rg->cols[w.second]);
        for (size_t c = 0; c < out->cols.size() && c < n.schema.size(); c++) out->cols[c].name = n.schema[c].name;
        if (met) {
          met->elapsed_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
          met->input_rows += (uint64_t)(nb + np);
        }
        return out;
      }
    }
    if (n.has_projection) {
      auto p = std::make_shared<DevBatch>();
      p->n = out->n;
      for (int idx : n.projection) p->cols.push_back(out->cols.at((size_t)idx));
      out = p;
    }
    for (size_t c = 0; c < out->cols.size() && c < n.schema.size(); c++) out->cols[c].name = n.schema[c].name;
    if (met) {
      met->elapsed_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
      met->input_rows += (uint64_t)(nb + np);
    }
    return out;
  }

  // ---- nested-loop join -------------------------------------------------------------------------
  // The join filter (over left ++ right) split into NljSpec's boolean program: AND / OR / NOT become steps, every other
  // node is an atom -- a Bool expression over one side, or a comparison between an expression over the build side and
  // one over the probe side.  The VM evaluates the atoms' side expressions as columns of their side.
  struct NljLowered {
    NljSpec S;
    std::vector<ExprPtr> build_exprs, probe_exprs;  // probe expressions index the probe side's own schema
    int build_at[NLJ_MAX_ATOMS], probe_at[NLJ_MAX_ATOMS];
    int n_left = 0;
  };
  static int expr_sides(const Expr& e, int n_left) {  // bit 0: reads build columns, bit 1: reads probe columns
    if (e.kind == Expr::Col) return e.col < n_left ? 1 : 2;
    int s = 0;
    for (auto& a : e.args) s |= expr_sides(*a, n_left);
    return s;
  }
  static uint8_t nlj_value_kind(const DataType& b, const DataType& p, const Expr& e) {
    auto refuse = [&](const std::string& why) {
      return EngineError(B200_ERR_UNSUPPORTED, "nested-loop join filter " + dump_expr(std::make_shared<Expr>(e)) + ": " + why);
    };
    if (b.is_string() && p.is_string()) return NLJ_V_STR;
    if (b.is_decimal() && p.is_decimal()) {
      if (b.scale != p.scale) throw refuse("decimal operands of different scales (" + b.str() + " vs " + p.str() + "): the plan must cast one of them");
      return NLJ_V_I128;
    }
    if (b.is_float() && p.is_float()) return NLJ_V_F64;
    if (b.id == TypeId::UInt64 || p.id == TypeId::UInt64) {
      if (b.id == p.id) return NLJ_V_U64;
    } else if (b.pk() == p.pk() && (b.pk() == PK::I64 || b.pk() == PK::Bool)) {
      return NLJ_V_I64;
    }
    throw refuse("cannot compare " + b.str() + " with " + p.str() + " without a cast");
  }
  int nlj_step(NljLowered& L, uint8_t kind, int a, int b) {
    NljSpec& S = L.S;
    if (S.n_steps == NLJ_MAX_STEPS) throw EngineError(B200_ERR_UNSUPPORTED, "nested-loop join filter has more than " + std::to_string(NLJ_MAX_STEPS) + " AND / OR / NOT nodes");
    NljStep& s = S.steps[S.n_steps];
    s.kind = kind;
    s.a = (uint8_t)a;
    s.b = (uint8_t)b;
    s.dst = (uint8_t)(NLJ_MAX_ATOMS + S.n_steps);
    return NLJ_MAX_ATOMS + S.n_steps++;
  }
  int nlj_lower(const ExprPtr& e, NljLowered& L) {
    if (e->kind == Expr::Bin && is_logic(e->op)) {
      const int a = nlj_lower(e->args[0], L), b = nlj_lower(e->args[1], L);
      return nlj_step(L, e->op == BinOp::And ? NLJ_AND : NLJ_OR, a, b);
    }
    if (e->kind == Expr::Not) {
      const int a = nlj_lower(e->args[0], L);
      return nlj_step(L, NLJ_NOT, a, a);
    }
    NljSpec& S = L.S;
    if (S.n_atoms == NLJ_MAX_ATOMS)
      throw EngineError(B200_ERR_UNSUPPORTED, "nested-loop join filter has more than " + std::to_string(NLJ_MAX_ATOMS) + " comparisons or one-side conditions");
    const int k = S.n_atoms++;
    NljAtom& a = S.atoms[k];
    L.build_at[k] = L.probe_at[k] = -1;
    const int sides = expr_sides(*e, L.n_left);
    if (sides != 3) {  // one side (or none: a constant, evaluated on the build side)
      if (e->type.id != TypeId::Bool) throw EngineError(B200_ERR_UNSUPPORTED, "nested-loop join filter term is not boolean: " + dump_expr(e));
      if (sides == 2) {
        a.kind = NLJ_PROBE_BOOL;
        L.probe_at[k] = (int)L.probe_exprs.size();
        L.probe_exprs.push_back(shift_cols(e, -L.n_left));
      } else {
        a.kind = NLJ_BUILD_BOOL;
        L.build_at[k] = (int)L.build_exprs.size();
        L.build_exprs.push_back(e);
      }
      return k;
    }
    const int sl = e->kind == Expr::Bin && is_compare(e->op) ? expr_sides(*e->args[0], L.n_left) : 0;
    const int sr = e->kind == Expr::Bin && is_compare(e->op) ? expr_sides(*e->args[1], L.n_left) : 0;
    if (!((sl == 1 && sr == 2) || (sl == 2 && sr == 1)))
      throw EngineError(B200_ERR_UNSUPPORTED, "nested-loop join filter term mixes both sides inside one operand, which the device does not evaluate: " + dump_expr(e));
    static const uint8_t swapped[] = {0, 1, 4, 5, 2, 3};  // p op b == b op' p (codes 0 EQ 1 NE 2 LT 3 LE 4 GT 5 GE)
    const int c = (int)e->op - (int)BinOp::Eq;
    const ExprPtr& be = sl == 1 ? e->args[0] : e->args[1];
    const ExprPtr& pe = sl == 1 ? e->args[1] : e->args[0];
    a.kind = NLJ_CMP;
    a.cmp = (uint8_t)(sl == 1 ? c : swapped[c]);
    a.vk = nlj_value_kind(be->type, pe->type, *e);
    L.build_at[k] = (int)L.build_exprs.size();
    L.build_exprs.push_back(be);
    L.probe_at[k] = (int)L.probe_exprs.size();
    L.probe_exprs.push_back(shift_cols(pe, -L.n_left));
    return k;
  }
  static KeyCol nlj_operand(const DevColumn& c, const NljAtom& a) {
    bool ok;
    if (a.kind != NLJ_CMP) ok = c.phys == PH_BOOL8;
    else switch (a.vk) {
      case NLJ_V_STR: ok = c.phys == PH_STRVIEW; break;
      case NLJ_V_I128: ok = c.phys == PH_DEC128; break;
      case NLJ_V_F64: ok = c.phys == PH_F64 || c.phys == PH_F32; break;
      case NLJ_V_U64: ok = c.phys == PH_U64; break;
      default: ok = c.phys <= PH_U32 || c.phys == PH_BOOL8;
    }
    if (!ok) throw EngineError(B200_ERR_EXECUTION, "nested-loop join: operand column " + c.name + " has an unexpected encoding");
    return KeyCol{c.data, c.valid, (uint8_t)c.phys, (uint8_t)c.width()};
  }

  DevBatchPtr exec_nlj(const PlanNode& n, int part, OpMetrics* met) {
    const JoinType jt = n.join_type;
    // the build side is read whole by every task, as a CollectLeft hash join's
    if (emits_build_rows(jt) && n_partitions(*n.children[1]) > 1)
      throw EngineError(B200_ERR_UNSUPPORTED, "nested-loop join that emits build-side rows over more than one probe partition");
    NljLowered L;
    memset(&L.S, 0, sizeof L.S);
    L.n_left = (int)n.children[0]->schema.size();
    L.S.result = n.join_filter ? nlj_lower(n.join_filter, L) : -1;
    JoinSide B = prepare_side(*n.children[0], part, true, L.build_exprs, false, met);
    JoinSide P = prepare_side(*n.children[1], part, false, L.probe_exprs, false, met);
    const int64_t nb = B.n, np = P.n;
    if (nb >= ((int64_t)1 << 31)) throw EngineError(B200_ERR_UNSUPPORTED, "nested-loop join build side exceeds 2^31 rows");
    auto t0 = std::chrono::steady_clock::now();
    uint64_t w_b = 0, w_p = 0;
    for (int k = 0; k < L.S.n_atoms; k++) {
      NljAtom& a = L.S.atoms[k];
      if (L.build_at[k] >= 0) {
        a.build = nlj_operand(B.keys[(size_t)L.build_at[k]], a);
        w_b += a.build.width;
      }
      if (L.probe_at[k] >= 0) {
        a.probe = nlj_operand(P.keys[(size_t)L.probe_at[k]], a);
        w_p += a.probe.width;
      }
    }
    const bool want_bmark = emits_build_rows(jt);
    const bool want_pmark = jt == JoinType::RightSemi || jt == JoinType::RightAnti || jt == JoinType::Right || jt == JoinType::Full;
    DevPtr bmark, pmark;
    if (want_bmark) {
      bmark = dev_alloc((size_t)std::max<int64_t>(nb, 1), x.st());
      CUDA_CHECK(cudaMemsetAsync(bmark->ptr, 0, (size_t)std::max<int64_t>(nb, 1), x.st()));
    }
    if (want_pmark) {
      pmark = dev_alloc((size_t)std::max<int64_t>(np, 1), x.st());
      CUDA_CHECK(cudaMemsetAsync(pmark->ptr, 0, (size_t)std::max<int64_t>(np, 1), x.st()));
    }
    x.check_cancel();
    // algorithmic bytes: probe operands once, build operands once per 256-row probe tile
    const uint64_t tiles = (uint64_t)(np + 255) / 256;
    const uint64_t operand_bytes = (uint64_t)np * w_p + (uint64_t)nb * w_b * tiles;
    DevPtr counts = dev_alloc((size_t)std::max<int64_t>(np, 1) * 4, x.st());
    {
      KernelTimer kt(x, "nlj_count", operand_bytes);
      launch_nlj_count(L.S, nb, np, (uint32_t*)counts->ptr, bmark ? (uint8_t*)bmark->ptr : nullptr, pmark ? (uint8_t*)pmark->ptr : nullptr, x.st());
    }
    x.e->nlj_pairs += (uint64_t)nb * (uint64_t)np;
    x.check_cancel();
    const bool semi_anti = jt == JoinType::LeftSemi || jt == JoinType::LeftAnti || jt == JoinType::RightSemi || jt == JoinType::RightAnti;
    int64_t n_pairs = 0;
    DevPtr bi, pi;
    if (!semi_anti) {
      DevPtr offs = dev_alloc((size_t)(np + 1) * 8, x.st());
      DevPtr scratch = dev_alloc((size_t)(np / 1024 + 4) * 8, x.st());
      if (np > 0) {
        launch_scan_u32_to_u64((const uint32_t*)counts->ptr, (uint64_t*)offs->ptr, np, (uint64_t*)scratch->ptr, x.st());
        n_pairs = (int64_t)x.get<uint64_t>((const uint64_t*)offs->ptr + np);
        x.check_cancel();
      }
      bi = dev_alloc((size_t)std::max<int64_t>(n_pairs, 1) * 8, x.st());
      pi = dev_alloc((size_t)std::max<int64_t>(n_pairs, 1) * 8, x.st());
      if (n_pairs > 0) {
        KernelTimer kt(x, "nlj_write", operand_bytes + 16 * (uint64_t)n_pairs);
        launch_nlj_write(L.S, nb, np, (const uint32_t*)counts->ptr, (const uint64_t*)offs->ptr, (int64_t*)bi->ptr, (int64_t*)pi->ptr, x.st());
      }
      x.check_cancel();
    }
    return join_output(n, B.payload, P.payload, bi ? (const int64_t*)bi->ptr : nullptr, pi ? (const int64_t*)pi->ptr : nullptr, n_pairs, bmark, pmark, t0, met);
  }

  // ---- shuffle writer -----------------------------------------------------------------------------
  uint64_t slice_bytes(const DevBatch& b, int64_t rows, const std::vector<int64_t>& chars_bytes) {
    uint64_t t = 0;
    size_t si = 0;
    for (auto& c : b.cols) {
      if (c.type.id == TypeId::Bool) t += (uint64_t)(rows + 7) / 8;
      else if (c.type.id == TypeId::Utf8) t += 4ull * (uint64_t)(rows + 1) + (uint64_t)chars_bytes[si++];
      else t += (uint64_t)c.width() * (uint64_t)rows;
    }
    return t;
  }

  // what the writer reports for one output partition (ShuffleWritePartition, ballista.proto:481-492)
  b200_shuffle_write_partition written(uint64_t part, uint64_t rows, uint64_t bytes, int64_t file_id, bool sort_shuffle) const {
    const uint64_t bs = (uint64_t)x.e->batch_size;
    b200_shuffle_write_partition w{};
    w.partition_id = part;
    w.num_rows = rows;
    w.num_batches = (rows + bs - 1) / bs;
    w.num_bytes = bytes;
    w.file_id = file_id;
    w.is_sort_shuffle = sort_shuffle ? 1 : 0;
    return w;
  }
  // the writer's metrics: a repartitioning writer read the bytes it wrote (the scatter moved them); one that stores its
  // input as it is counts that input's rows
  static void count_written(OpMetrics* met, uint64_t rows, uint64_t bytes, bool repartitioned) {
    if (!met) return;
    met->output_rows += rows;
    met->bytes_written += bytes;
    if (repartitioned) met->bytes_read += bytes;
    else met->input_rows += rows;
  }

  struct FusedExchange {
    bool done = false;  // the rows were scattered into their owners' windows (nothing left to exchange)
    uint64_t sent = 0, recvd = 0;
  };

  // ------------------------------------------------------------------------------------------------
  // Fused shuffle writer + exchange (gang collective; ShuffleWriterExec's repartition, shuffle_writer.rs:214-330, and
  // the readers' remote fetch, shuffle_reader.rs:522-602, as ONE kernel pass).  After the histogram every executor
  // knows how many rows every map task holds for every output partition (one small NCCL all-gather), so every row has a
  // known final address in the window of the executor that owns its partition: the scatter kernel stores it there
  // directly -- local partitions through HBM, remote ones as peer stores over NVLink.  The reduce side finds its input
  // already laid out partition by partition, map task by map task (the order sort_shuffle and the NCCL exchange produce).
  // Returns false (nothing written) when some window cannot hold this exchange: the caller then takes the two-step path;
  // the decision is taken from the all-gathered matrix, i.e. identically on every executor.
  // ------------------------------------------------------------------------------------------------
  bool scatter_to_owners(const PlanNode& root, int input_partition, const std::vector<DevColumn>& pay, const PidSrc& pid, int64_t n, uint32_t P,
                         uint32_t n_tiles, const DevPtr& mat, const DevPtr& tile_hist, uint64_t row_bytes, FusedExchange* fx,
                         std::vector<b200_shuffle_write_partition>& res, OpMetrics* met) {
    b200_engine* e = x.e;
    NcclApi& N = NcclApi::get();
    const int W = e->world, me = e->rank;
    const size_t mrow = (size_t)P + 3;
    const size_t ncols = pay.size();
    auto al = [](uint64_t v) { return (v + 255) & ~255ull; };
    std::lock_guard<std::mutex> cg(e->comm_mu);
    // my row of the matrix: the counts are already there (histogram); add validity mask, window fill, map task id
    uint64_t* extra = (uint64_t*)x.stage_bytes(24);
    extra[0] = 0;
    for (size_t c = 0; c < ncols; c++)
      if (pay[c].valid) extra[0] |= 1ull << c;
    extra[1] = al(e->win_used);
    extra[2] = (uint64_t)(int64_t)input_partition;
    unsigned long long* mrows = (unsigned long long*)mat->ptr;
    CUDA_CHECK(cudaMemcpyAsync(mrows + mrow * (size_t)me + P, extra, 24, cudaMemcpyHostToDevice, x.st()));
    NCCL_CHECK(N.GroupStart());
    for (int d = 0; d < W; d++) {
      if (d == me) continue;
      NCCL_CHECK(N.Send(mrows + mrow * (size_t)me, mrow * 8, kNcclUint8, d, e->comm, x.st()));
      NCCL_CHECK(N.Recv(mrows + mrow * (size_t)d, mrow * 8, kNcclUint8, d, e->comm, x.st()));
    }
    NCCL_CHECK(N.GroupEnd());
    count_launches();
    // (the matrix and the base table below can exceed the task's pinned arena at large fan-outs: plain host vectors)
    std::vector<unsigned long long> Mv(mrow * (size_t)W);
    CUDA_CHECK(cudaMemcpyAsync(Mv.data(), mat->ptr, Mv.size() * 8, cudaMemcpyDeviceToHost, x.st()));
    const unsigned long long* M = Mv.data();
    x.sync();
    auto cnt = [&](int s, uint32_t p) { return (uint64_t)M[mrow * (size_t)s + p]; };
    uint64_t any_valid = 0;
    for (int s = 0; s < W; s++) any_valid |= M[mrow * (size_t)s + P];
    // layout of every owner's window for this exchange: per owned partition, per column, all map tasks back to back
    std::vector<uint64_t> tot(P, 0), before(P, 0);
    for (uint32_t p = 0; p < P; p++)
      for (int s = 0; s < W; s++) {
        if (s < me) before[p] += cnt(s, p);
        tot[p] += cnt(s, p);
      }
    const size_t nslots = ncols * 2;  // [c] data, [ncols + c] validity
    std::vector<uint64_t> region(nslots * P, 0);
    std::vector<uint64_t> cursor((size_t)W);
    for (int r = 0; r < W; r++) cursor[(size_t)r] = M[mrow * (size_t)r + P + 1];
    for (uint32_t p = 0; p < P; p++) {
      uint64_t& cur = cursor[(size_t)(p % (uint32_t)W)];
      for (size_t c = 0; c < ncols; c++) {
        region[c * P + p] = cur;
        cur += al(tot[p] * (uint64_t)pay[c].width());
        if (any_valid >> c & 1) {
          region[(ncols + c) * P + p] = cur;
          cur += al(tot[p]);
        }
      }
    }
    for (int r = 0; r < W; r++)
      if (cursor[(size_t)r] > e->win_bytes) return false;  // same verdict everywhere; nothing was written
    // destination bases: byte address of row 0 of (column, partition) as the scatter kernel numbers the rows, i.e.
    // shifted back by this task's prefix of the partition-contiguous order
    std::vector<int64_t> bounds(P + 1, 0);
    for (uint32_t p = 0; p < P; p++) bounds[p + 1] = bounds[p] + (int64_t)cnt(me, p);
    std::vector<uint64_t> hbv(nslots * P);
    uint64_t* hb = hbv.data();
    for (size_t sl = 0; sl < nslots; sl++) {
      const size_t c = sl % ncols;
      const int64_t w = sl < ncols ? (int64_t)pay[c].width() : 1;
      for (uint32_t p = 0; p < P; p++) {
        const uint8_t* base = e->win_peer[(size_t)(p % (uint32_t)W)] + region[sl * P + p];
        hb[sl * P + p] = (uint64_t)(base + ((int64_t)before[p] - bounds[p]) * w);
      }
    }
    DevPtr bases = dev_alloc(nslots * P * 8 + 64, x.st());
    CUDA_CHECK(cudaMemcpyAsync(bases->ptr, hb, nslots * P * 8, cudaMemcpyHostToDevice, x.st()));
    std::vector<DevPtr> ones_keep;
    std::vector<ScatterCol> cols;
    const unsigned long long* part_base = (const unsigned long long*)bases->ptr;
    for (size_t c = 0; c < ncols; c++) {
      cols.push_back(ScatterCol{pay[c].data, nullptr, part_base + c * P, pay[c].width()});
      if (any_valid >> c & 1) {
        const uint8_t* v = pay[c].valid;
        if (!v && n > 0) {  // another map task has nulls in this column: this one contributes all-valid bytes
          DevPtr ones = dev_alloc((size_t)n + 64, x.st());
          CUDA_CHECK(cudaMemsetAsync(ones->ptr, 1, (size_t)n, x.st()));
          ones_keep.push_back(ones);
          v = (const uint8_t*)ones->ptr;
        }
        cols.push_back(ScatterCol{v, nullptr, part_base + (ncols + c) * P, 1});
      }
    }
    partition_scatter(x, "partition_scatter_peer", pid, n, P, n_tiles, tile_hist, cols);
    // every executor's stores must have landed before anyone reads its window: a zero-payload all-to-all on the same
    // stream completes only after every peer's scatter kernel did
    {
      DevPtr bar = dev_alloc((size_t)W * 16 + 64, x.st());
      NCCL_CHECK(N.GroupStart());
      for (int d = 0; d < W; d++) {
        if (d == me) continue;
        NCCL_CHECK(N.Send((const uint8_t*)bar->ptr + 8 * (size_t)W, 8, kNcclUint8, d, e->comm, x.st()));
        NCCL_CHECK(N.Recv((uint8_t*)bar->ptr + 8 * (size_t)d, 8, kNcclUint8, d, e->comm, x.st()));
      }
      NCCL_CHECK(N.GroupEnd());
      count_launches();
    }
    e->win_used = cursor[(size_t)me];
    // the reduce side's view: one batch per owned partition, one piece per map task
    uint64_t total_bytes = 0;
    std::map<int64_t, std::vector<Piece>> arrivals;
    for (uint32_t p = 0; p < P; p++) {
      const uint64_t rows = cnt(me, p);
      if (rows) {
        res.push_back(written(p, rows, rows * row_bytes, input_partition, root.sort_shuffle));
        total_bytes += res.back().num_bytes;
        if ((int)(p % (uint32_t)W) != me) fx->sent += res.back().num_bytes;
      }
      if ((int)(p % (uint32_t)W) != me || tot[p] == 0) continue;
      auto b = std::make_shared<DevBatch>();
      b->n = (int64_t)tot[p];
      for (size_t c = 0; c < ncols; c++) {
        DevColumn col;
        col.name = root.schema[c].name;
        col.type = pay[c].type;
        col.phys = pay[c].phys;
        col.n = b->n;
        col.data = e->win_local + region[c * P + p];
        col.nullable = (any_valid >> c & 1) != 0;
        if (col.nullable) col.valid = e->win_local + region[(ncols + c) * P + p];
        b->cols.push_back(col);
      }
      int64_t at = 0;
      for (int s = 0; s < W; s++) {
        const int64_t rs = (int64_t)cnt(s, p);
        if (rs) {
          arrivals[p].push_back(Piece{(int64_t)M[mrow * (size_t)s + P + 2], b, at, at + rs, s, {}});
          if (s != me) fx->recvd += (uint64_t)rs * row_bytes;
        }
        at += rs;
      }
    }
    e->shuffle.install(job, root.stage_id, arrivals);
    x.sync();
    count_written(met, (uint64_t)n, total_bytes, true);
    e->fused_exchanges++;
    fx->done = true;
    return true;
  }

  std::vector<b200_shuffle_write_partition> execute_stage(const PlanNode& root, int input_partition, FusedExchange* fx = nullptr) {
    std::vector<b200_shuffle_write_partition> res;
    charge_launches(root, [&] { res = write_stage(root, input_partition, fx); });
    return res;
  }
  std::vector<b200_shuffle_write_partition> write_stage(const PlanNode& root, int input_partition, FusedExchange* fx) {
    if (root.op != PlanNode::ShuffleWriter) throw EngineError(B200_ERR_INVALID, "stage plan root must be a ShuffleWriterExec");
    OpMetrics* met = x.m(&root);
    const PlanNode& child = *root.children[0];
    const int32_t my_rank = x.e->rank;
    std::vector<b200_shuffle_write_partition> res;
    // no repartitioning; also hash partitioning into ONE partition (hash % 1 == 0 for every row), which
    // keeps the rows of this task together as output partition 0
    const bool single = root.n_out_partitions == 1;
    if (root.n_out_partitions == 0 || single) {
      DevBatchPtr in = exec(child, input_partition);
      // stored as produced: strings stay views into kept-alive character buffers; they are laid out as Arrow
      // Utf8 only when the partition leaves the device (export) or the GPU (exchange)
      auto st = std::make_shared<DevBatch>();
      st->n = in->n;
      for (size_t c = 0; c < in->cols.size(); c++) {
        DevColumn col = in->cols[c];
        col.name = root.schema[c].name;
        st->cols.push_back(col);
      }
      std::vector<int64_t> cb;
      {
        ScopeTimer t2("writer: string bytes + final sync");
        cb = string_bytes(x, *st);
        x.sync();  // deferred status checks of this task's kernels
      }
      const int64_t fid = single ? (int64_t)input_partition : -1;
      const ShuffleKey key{job, root.stage_id, single ? 0 : input_partition};
      if (single) x.e->shuffle.store(key, Piece{fid, st, 0, st->n, my_rank, cb}, false);
      else x.e->shuffle.replace_partition(key, Piece{fid, st, 0, st->n, my_rank, cb});
      const b200_shuffle_write_partition w = written((uint64_t)key.part, (uint64_t)st->n, slice_bytes(*st, st->n, cb), fid, single && root.sort_shuffle);
      count_written(met, w.num_rows, w.num_bytes, false);
      if (!(single && st->n == 0)) res.push_back(w);  // only partitions with rows are reported
      return res;
    }
    // hash repartition: pid = hash(keys) % P computed by the child's pipeline kernel, then ONE stable radix
    // partition pass (per-tile histogram -> scan -> ranked scatter of every column)
    const uint32_t P = (uint32_t)root.n_out_partitions;
    if (P > PART_MAX_FANOUT) throw EngineError(B200_ERR_UNSUPPORTED, "more than 4096 output partitions in one shuffle");
    size_t n_payload = 0;
    std::vector<DevColumn> pay;   // payload columns (strings as views)
    PidSrc ps;
    memset(&ps, 0, sizeof ps);
    std::vector<DevColumn> key_keep;
    DevBatchPtr mat_keep;
    int64_t n = 0;
    with_chain(child, input_partition, false, [&](const BuilderFactory& mk, DevBatchPtr& src) {
      auto pbp = mk();
      PipelineBuilder& pb = *pbp;
      std::vector<ColRef> outs = named_cols(pb, root.schema);
      n_payload = outs.size();
      std::vector<ColRef> keys;
      for (auto& e : root.part_exprs) {
        ColRef k = pb.compile(*e);
        pb.pin(k);
        keys.push_back(k);
      }
      // shuffle keys that are plain integer-like columns of an unfiltered input: the partition kernels hash them on
      // the fly; otherwise the pipeline kernel materialises the partition id next to the computed payload columns
      // integer-like shuffle keys travel as columns (forwarded untouched, or compacted with the payload when the chain
      // filters) and the partition kernels hash them on the fly; other key types get a materialised partition id
      bool direct_keys = !keys.empty() && keys.size() <= (size_t)VM_MAX_KEYS;
      for (auto& k : keys) direct_keys = direct_keys && exact_key(k.type) && (k.op.kind == OPD_NONE || k.op.kind == OPD_COL);
      if (direct_keys) {
        for (auto& k : keys) outs.push_back(k);
      } else {
        ColRef h = pb.hash_of(keys);
        ColRef pid = pb.mod_u64(h, P);
        pid.name = "__pid";
        outs.push_back(pid);
      }
      Mixed m = materialize_mixed(pb, outs, src, met);
      n = m.n;
      for (size_t c = 0; c < n_payload; c++) {
        DevColumn col = as_views(x, m.cols[c]);
        col.name = root.schema[c].name;
        pay.push_back(col);
      }
      if (direct_keys) {
        for (size_t k = 0; k < keys.size(); k++) {
          const DevColumn& kc = m.cols[n_payload + k];
          ps.keys[ps.n_keys++] = KeyCol{kc.data, kc.valid, (uint8_t)kc.phys, (uint8_t)kc.width()};
          key_keep.push_back(kc);
        }
      } else {
        key_keep.push_back(m.cols.back());
        ps.pid = (const uint32_t*)m.cols.back().data;
      }
      return src;
    });
    if (n >= ((int64_t)1 << 32)) throw EngineError(B200_ERR_UNSUPPORTED, "more than 2^32 rows in one shuffle-writer task");
    const PidSrc& pid = ps;
    // histogram (+ string bytes per partition for ShuffleWritePartition.num_bytes)
    PartStrCols sc;
    sc.n = 0;
    for (auto& c : pay)
      if (c.type.id == TypeId::Utf8) {
        if (sc.n == PART_MAX_STR_COLS) throw EngineError(B200_ERR_UNSUPPORTED, "more than 16 string columns in one shuffle output");
        sc.c[sc.n++] = PartStrCol{c.data, c.valid, c.phys == PH_STRVIEW ? 1 : 0, 0};
      }
    if ((size_t)P * (1 + sc.n) * 4 > 200 * 1024) throw EngineError(B200_ERR_UNSUPPORTED, "shuffle fan-out x string columns exceeds the histogram's shared memory");
    const uint32_t n_tiles = partition_n_tiles(n);
    const size_t acc_words = (size_t)P * (1 + sc.n);
    // fused shuffle: decided from the schema and the engine's configuration only, so that every executor of the gang
    // takes the same branch
    const int W = x.e->world, me = x.e->rank;
    const bool fuse = fx && W > 1 && x.e->comm && x.e->win_local && sc.n == 0 && n_payload <= 60;
    const size_t mrow = (size_t)P + 3;  // per executor: P row counts, validity mask, window fill, map task id
    DevPtr acc = dev_alloc((fuse ? mrow * (size_t)W : acc_words) * 8, x.st());
    CUDA_CHECK(cudaMemsetAsync(acc->ptr, 0, (fuse ? mrow * (size_t)W : acc_words) * 8, x.st()));
    unsigned long long* const acc_ptr = (unsigned long long*)acc->ptr + (fuse ? mrow * (size_t)me : 0);
    DevPtr tile_hist = dev_alloc((size_t)std::max<uint64_t>((uint64_t)P * n_tiles, 1) * 4 + 64, x.st());
    uint64_t row_bytes = 0;
    for (auto& c : pay) row_bytes += (uint64_t)c.width() + (c.valid ? 1 : 0);
    {
      uint64_t kb = pid.pid ? 4 : 0;
      for (int k = 0; k < pid.n_keys; k++) kb += pid.keys[k].width;
      KernelTimer kt(x, "partition_hist", (uint64_t)n * kb);
      CUDA_CHECK(launch_partition_hist(pid, n, P, (uint32_t*)tile_hist->ptr, acc_ptr, sc, acc_ptr + P, x.st()));
    }
    if (fuse) {
      std::vector<b200_shuffle_write_partition> fr;
      if (scatter_to_owners(root, input_partition, pay, pid, n, P, n_tiles, acc, tile_hist, row_bytes, fx, fr, met)) return fr;
    }
    const unsigned long long* hc = (const unsigned long long*)x.fetch_bytes(acc_ptr, acc_words * 8);
    // while the counts travel: scan the per-tile histogram and scatter
    auto st = std::make_shared<DevBatch>();
    st->n = n;
    std::vector<ScatterCol> cols;
    for (size_t c = 0; c < n_payload; c++) {
      const DevColumn& scn = pay[c];
      DevColumn oc = make_out_column(root.schema[c].name, scn.type, scn.phys, n, scn.valid != nullptr, x.st());
      oc.n = n;
      cols.push_back(ScatterCol{scn.data, (void*)oc.data, nullptr, scn.width()});
      if (scn.valid) cols.push_back(ScatterCol{scn.valid, (void*)oc.valid, nullptr, 1});
      for (auto& k : scn.keep) oc.keep.push_back(k);
      st->cols.push_back(oc);
    }
    partition_scatter(x, "partition_scatter", pid, n, P, n_tiles, tile_hist, cols);
    x.sync();
    std::vector<int64_t> bounds(P + 1, 0);
    for (uint32_t p = 0; p < P; p++) bounds[p + 1] = bounds[p] + (int64_t)hc[p];
    std::vector<std::vector<int64_t>> chars_per_part((size_t)sc.n, std::vector<int64_t>(P));  // [string col][p]
    for (int c = 0; c < sc.n; c++)
      for (uint32_t p = 0; p < P; p++) chars_per_part[(size_t)c][p] = (int64_t)hc[(size_t)P * (1 + c) + p];
    uint64_t total_bytes = 0;
    for (uint32_t p = 0; p < P; p++) {
      const int64_t rows = bounds[p + 1] - bounds[p];
      std::vector<int64_t> cb;
      for (auto& cp : chars_per_part) cb.push_back(cp[p]);
      x.e->shuffle.store(ShuffleKey{job, root.stage_id, (int64_t)p}, Piece{input_partition, st, bounds[p], bounds[p + 1], my_rank, cb}, false);
      if (rows == 0) continue;  // only partitions with rows are reported (sort_shuffle/writer.rs:357-369)
      res.push_back(written(p, (uint64_t)rows, slice_bytes(*st, rows, cb), input_partition, root.sort_shuffle));
      total_bytes += res.back().num_bytes;
    }
    count_written(met, (uint64_t)n, total_bytes, true);
    return res;
  }
};

// ------------------------------------------------------------------------------------------------
// Exchange between the box's GPU executors (ShuffleReaderExec's remote fetch, shuffle_reader.rs:522-602 /
// client.rs:143-220, as an all-to-all-v over NVLink).  Gang collective: every executor of the communicator calls
// it for the same (job, stage) after its map tasks finished.
//
// Round 1: every pair exchanges one fixed-size slot = [header | inline payload].  The header lists, per piece,
// (partition, file id, rows, byte size of every column buffer) -- the ShuffleWritePartition / PartitionLocation
// metadata the reference sends through the scheduler -- so no separate size collective is needed, and messages
// of up to EXCH_INLINE bytes (the partial-aggregate states of q1: a few hundred bytes) are complete after it.
// Round 2 (only for pairs whose payload is larger): grouped ncclSend/ncclRecv straight from the stored column
// slices into the receiver's final column buffers -- no packing copy on either side.
// ------------------------------------------------------------------------------------------------
static const uint64_t EXCH_MAGIC = 0xB200E8C4A11ull;
static const size_t EXCH_INLINE = 16 << 10;
enum ExchangeMode { EXCH_HASH = 0, EXCH_GATHER = 1, EXCH_BROADCAST = 2 };

struct ExchEntry {
  int64_t partition, file_id, rows;
  std::vector<uint64_t> sizes;  // 3 per column: validity bytes, data bytes, chars bytes
};

struct Exchange {
  Exec x;
  b200_engine* e;
  std::string job;
  int64_t stage;
  int P, mode, root;
  Schema schema;
  size_t ncols;

  bool goes_to(int p, int d) const {
    if (mode == EXCH_BROADCAST) return true;
    if (mode == EXCH_GATHER) return d == root;
    return p % e->world == d;
  }
  int n_owned(int d) const {
    int k = 0;
    for (int p = 0; p < P; p++) k += goes_to(p, d) ? 1 : 0;
    return k;
  }
  size_t entry_bytes() const { return (3 + 3 * ncols) * 8; }
  size_t hdr_bytes(int d) const { return (32 + (size_t)n_owned(d) * entry_bytes() + 255) & ~(size_t)255; }
  size_t slot_bytes() const {
    size_t h = 0;
    for (int d = 0; d < e->world; d++) h = std::max(h, hdr_bytes(d));
    return h + EXCH_INLINE;
  }
  static uint64_t al16(uint64_t v) { return (v + 15) & ~15ull; }

  void run(uint64_t* sent_out, uint64_t* recv_out) {
    NcclApi& N = NcclApi::get();
    const int W = e->world, me = e->rank;
    // ---- local pieces: one (coalesced) piece per partition ------------------------------------------------
    std::vector<StoredPiece> locals;
    {
      std::map<int64_t, std::vector<Piece>> snap;
      for (auto& sp : e->shuffle.of_rank(job, stage, me))
        if (sp.part >= 0 && sp.part < P && sp.piece.r1 > sp.piece.r0) snap[sp.part].push_back(sp.piece);
      for (auto& kv : snap) {
        if (kv.second.size() == 1) {
          locals.push_back(StoredPiece{kv.first, kv.second[0]});
          continue;
        }
        Piece c;
        c.file_id = kv.second[0].file_id;
        c.batch = concat_slices(x, kv.second, schema);
        c.r0 = 0;
        c.r1 = c.batch->n;
        c.src_rank = me;
        bool known = true;
        for (auto& pc : kv.second) known &= !pc.str_bytes.empty() || pc.batch->cols.empty();
        if (known && !kv.second[0].str_bytes.empty()) {
          c.str_bytes.assign(kv.second[0].str_bytes.size(), 0);
          for (auto& pc : kv.second)
            for (size_t k = 0; k < c.str_bytes.size(); k++) c.str_bytes[k] += pc.str_bytes[k];
        }
        locals.push_back(StoredPiece{kv.first, c});
      }
    }
    // string bytes of every outgoing slice must be known on the host (they normally are: the writer recorded them)
    for (auto& L : locals) {
      size_t n_str = 0;
      for (auto& c : L.piece.batch->cols) n_str += c.type.id == TypeId::Utf8 ? 1 : 0;
      if (L.piece.batch->cols.size() != ncols) throw EngineError(B200_ERR_INVALID, "exchange: stored partition does not match the given schema");
      if (n_str && L.piece.str_bytes.size() != n_str) {
        DevBatch sl;
        sl.n = L.piece.r1 - L.piece.r0;
        for (auto& c : L.piece.batch->cols) sl.cols.push_back(slice_column(c, L.piece.r0, L.piece.r1));
        L.piece.str_bytes = string_bytes(x, sl);
      }
    }
    if (W <= 1) {
      *sent_out = *recv_out = 0;
      return;
    }
    if (!e->comm) throw EngineError(B200_ERR_INVALID, "exchange: communicator not initialised (b200_engine_comm_init)");
    const size_t slot = slot_bytes();
    DevPtr sendbuf = dev_alloc(slot * W, x.st()), recvbuf = dev_alloc(slot * W, x.st());
    // ---- compose headers and the payload layout per destination -----------------------------------------------
    struct Out {
      std::vector<ExchEntry> entries;
      std::vector<const StoredPiece*> src;
      uint64_t payload = 0;
      bool inl = true;
    };
    std::vector<Out> outs((size_t)W);
    for (int d = 0; d < W; d++) {
      if (d == me) continue;
      Out& o = outs[(size_t)d];
      for (auto& L : locals) {
        if (!goes_to((int)L.part, d)) continue;
        ExchEntry en;
        en.partition = L.part;
        en.file_id = L.piece.file_id;
        en.rows = L.piece.r1 - L.piece.r0;
        size_t si = 0;
        for (auto& c : L.piece.batch->cols) {
          en.sizes.push_back(c.valid ? (uint64_t)en.rows : 0);
          if (c.type.id == TypeId::Utf8) {
            en.sizes.push_back((uint64_t)(en.rows + 1) * 4);
            en.sizes.push_back((uint64_t)L.piece.str_bytes[si++]);
          } else {
            en.sizes.push_back((uint64_t)en.rows * c.width());
            en.sizes.push_back(0);
          }
        }
        for (uint64_t b : en.sizes) o.payload += al16(b);
        o.entries.push_back(en);
        o.src.push_back(&L);
      }
      o.inl = o.payload <= EXCH_INLINE;
    }
    // headers -> one staging block -> device; inline payloads packed by the same kernel that places the headers
    size_t hdr_total = 0;
    std::vector<size_t> hdr_at((size_t)W, 0);
    for (int d = 0; d < W; d++) {
      hdr_at[(size_t)d] = hdr_total;
      hdr_total += d == me ? 0 : hdr_bytes(d);
    }
    uint8_t* hstage = (uint8_t*)x.stage_bytes(hdr_total ? hdr_total : 16);
    memset(hstage, 0, hdr_total);
    for (int d = 0; d < W; d++) {
      if (d == me) continue;
      const Out& o = outs[(size_t)d];
      uint64_t* h = (uint64_t*)(hstage + hdr_at[(size_t)d]);
      h[0] = EXCH_MAGIC;
      h[1] = o.entries.size();
      h[2] = o.inl ? 1 : 0;
      h[3] = o.payload;
      uint64_t* q = h + 4;
      for (auto& en : o.entries) {
        *q++ = (uint64_t)en.partition;
        *q++ = (uint64_t)en.file_id;
        *q++ = (uint64_t)en.rows;
        for (uint64_t b : en.sizes) *q++ = b;
      }
    }
    DevPtr hdev = dev_alloc(hdr_total + 16, x.st());
    if (hdr_total) CUDA_CHECK(cudaMemcpyAsync(hdev->ptr, hstage, hdr_total, cudaMemcpyHostToDevice, x.st()));
    PackList pl;
    std::vector<DevColumn> keep_cols;  // converted string columns of large messages, alive until the sends are enqueued
    struct SendOp { const void* ptr; uint64_t bytes; int peer; };
    std::vector<SendOp> sends;
    uint64_t sent = 0;
    for (int d = 0; d < W; d++) {
      if (d == me) continue;
      const Out& o = outs[(size_t)d];
      uint8_t* sl = (uint8_t*)sendbuf->ptr + (size_t)d * slot;
      pl.copy((const uint8_t*)hdev->ptr + hdr_at[(size_t)d], sl, hdr_bytes(d));
      uint8_t* cur = sl + hdr_bytes(d);
      sent += o.payload;
      for (size_t k = 0; k < o.entries.size(); k++) {
        const Piece& pc = o.src[k]->piece;
        const ExchEntry& en = o.entries[k];
        size_t si = 0;
        for (size_t c = 0; c < ncols; c++) {
          DevColumn col = slice_column(pc.batch->cols[c], pc.r0, pc.r1);
          const uint64_t bv = en.sizes[3 * c], bd = en.sizes[3 * c + 1], bc = en.sizes[3 * c + 2];
          if (o.inl) {
            if (bv) pl.copy(col.valid, cur, bv);
            cur += al16(bv);
            if (col.type.id == TypeId::Utf8) {
              pl.strings(col, cur, cur + al16(bd), bc);
            } else if (bd) {
              pl.copy(col.data, cur, bd);
            }
            cur += al16(bd) + al16(bc);
          } else {
            if (bv) sends.push_back(SendOp{col.valid, bv, d});
            if (col.type.id == TypeId::Utf8) {
              DevColumn u = col.phys == PH_STRVIEW ? as_utf8(x, col, (int64_t)pc.str_bytes[si]) : col;
              const uint8_t* chars = u.chars;
              if (col.phys != PH_STRVIEW) {
                // Arrow slice: the receiver wants offsets that start at 0
                DevPtr ro = dev_alloc((size_t)(u.n + 1) * 4 + 64, x.st());
                DevPtr fl = dev_alloc(16, x.st());
                launch_rebase_offsets((const int32_t*)u.data, u.n + 1, (int32_t*)ro->ptr, (int32_t*)fl->ptr, x.st());
                // first offset of the slice: needed on the host to position the chars pointer
                const int32_t first = x.get<int32_t>(fl->ptr);
                chars = u.chars + first;
                u.data = (const uint8_t*)ro->ptr;
                u.keep.push_back(ro);
              }
              keep_cols.push_back(u);
              sends.push_back(SendOp{u.data, bd, d});
              if (bc) sends.push_back(SendOp{chars, bc, d});
            } else if (bd) {
              sends.push_back(SendOp{col.data, bd, d});
            }
          }
          if (col.type.id == TypeId::Utf8) si++;
        }
      }
    }
    pl.run(x);
    // ---- round 1: fixed-size slots ---------------------------------------------------------------------------
    std::lock_guard<std::mutex> cg(e->comm_mu);
    NCCL_CHECK(N.GroupStart());
    for (int d = 0; d < W; d++) {
      if (d == me) continue;
      NCCL_CHECK(N.Send((const uint8_t*)sendbuf->ptr + (size_t)d * slot, slot, kNcclUint8, d, e->comm, x.st()));
      NCCL_CHECK(N.Recv((uint8_t*)recvbuf->ptr + (size_t)d * slot, slot, kNcclUint8, d, e->comm, x.st()));
    }
    NCCL_CHECK(N.GroupEnd());
    count_launches();
    // incoming headers: every peer used hdr_bytes(me)
    const size_t hb = hdr_bytes(me);
    std::vector<const uint64_t*> rh((size_t)W, nullptr);
    for (int d = 0; d < W; d++)
      if (d != me) rh[(size_t)d] = (const uint64_t*)x.fetch_bytes((const uint8_t*)recvbuf->ptr + (size_t)d * slot, hb);
    x.sync();
    // ---- parse, allocate, round 2 ------------------------------------------------------------------------------
    struct RecvOp { void* ptr; uint64_t bytes; int peer; };
    std::vector<RecvOp> recvs;
    std::map<int64_t, std::vector<Piece>> incoming;
    uint64_t recvd = 0;
    for (int d = 0; d < W; d++) {
      if (d == me) continue;
      const uint64_t* h = rh[(size_t)d];
      if (h[0] != EXCH_MAGIC) throw EngineError(B200_ERR_CUDA, "exchange: bad header from rank " + std::to_string(d));
      const uint64_t n_ent = h[1];
      const bool inl = h[2] != 0;
      recvd += h[3];
      if (32 + n_ent * entry_bytes() > hb) throw EngineError(B200_ERR_INVALID, "exchange: header overflow");
      const uint64_t* q = h + 4;
      const uint8_t* cur = (const uint8_t*)recvbuf->ptr + (size_t)d * slot + hb;
      for (uint64_t k = 0; k < n_ent; k++) {
        const int64_t part = (int64_t)*q++, fid = (int64_t)*q++, rows = (int64_t)*q++;
        auto b = std::make_shared<DevBatch>();
        b->n = rows;
        std::vector<int64_t> sb;
        for (size_t c = 0; c < ncols; c++) {
          const uint64_t bv = *q++, bd = *q++, bc = *q++;
          DevColumn col;
          col.name = schema[c].name;
          col.type = schema[c].type;
          col.phys = phys_of(col.type);
          col.n = rows;
          col.nullable = bv != 0;
          auto place = [&](uint64_t bytes) -> const uint8_t* {
            if (inl) {
              const uint8_t* ptr = cur;
              cur += al16(bytes);
              col.keep.push_back(recvbuf);
              return ptr;
            }
            DevPtr dp = dev_alloc((size_t)bytes + 64, x.st());
            col.keep.push_back(dp);
            if (bytes) recvs.push_back(RecvOp{dp->ptr, bytes, d});
            return (const uint8_t*)dp->ptr;
          };
          const uint8_t* pv = place(bv);
          if (bv) col.valid = pv;
          col.data = place(bd);
          if (col.type.id == TypeId::Utf8) {
            col.chars = place(bc);
            col.chars_bytes = (int64_t)bc;
            sb.push_back((int64_t)bc);
          } else if (inl) {
            cur += al16(bc);
          }
          b->cols.push_back(col);
        }
        incoming[part].push_back(Piece{fid, b, 0, rows, d, sb});
      }
    }
    if (!sends.empty() || !recvs.empty()) {
      NCCL_CHECK(N.GroupStart());
      for (auto& so : sends) NCCL_CHECK(N.Send(so.ptr, so.bytes, kNcclUint8, so.peer, e->comm, x.st()));
      for (auto& ro : recvs) NCCL_CHECK(N.Recv(ro.ptr, ro.bytes, kNcclUint8, ro.peer, e->comm, x.st()));
      NCCL_CHECK(N.GroupEnd());
      count_launches();
    }
    // ---- install ---------------------------------------------------------------------------------------------
    std::vector<int64_t> handed_over;
    for (int p = 0; p < P; p++)
      if (!goes_to(p, me)) handed_over.push_back(p);
    e->shuffle.remove_parts(job, stage, handed_over);
    e->shuffle.install(job, stage, incoming);
    *sent_out = sent;
    *recv_out = recvd;
  }
};

// ------------------------------------------------------------------------------------------------
// Parquet scan: DataSourceExec + ParquetSource with the page decode on the device
// (ballista/core/proto/datafusion.proto:1058-1077; registration path benchmarks/src/bin/tpch.rs:684-693).
// The host parses the footer and the page headers (parquet_meta.hpp), ships the raw bytes of the REQUESTED column chunks
// to HBM (projection push-down: other columns never cross the bus) and csrc/device/parquet.cu decodes them.
// ------------------------------------------------------------------------------------------------
struct PqHostColumn {
  pq::SchemaElement se;
  int leaf = -1;
  bool optional = false;
  std::vector<PqPage> pages, dicts;
  int64_t rows = 0, dict_entries = 0;
  DevPtr raw;  // the column's chunks, back to back (as stored in the file: possibly compressed)
  DevPtr dec;  // compressed chunks: the pages' payloads rebuilt uncompressed
  std::vector<PqDecompJob> jobs;
  std::map<int32_t, uint64_t> codec_bytes;  // per compressed codec: its chunks' stored bytes + their rebuilt payload bytes
  std::vector<uint8_t> page_in_dec, dict_in_dec;  // per page: its payload pointer is an offset into `dec` until `dec` exists
  size_t dec_bytes = 0;
  int64_t delta_pages = 0, dba_pages = 0;  // data pages in PQ_ENC_DBP and above; of those, DELTA_BYTE_ARRAY
  uint64_t delta_bytes = 0;                // their payload bytes
};

static DataType pq_arrow_type(const pq::SchemaElement& se, int* out_kind) {
  const bool is_decimal = se.logical == 5 || se.converted == 5;
  const bool is_date = se.logical == 6 || se.converted == 6;
  switch (se.type) {
    case pq::T_BOOLEAN: *out_kind = PQ_OUT_BOOL8; return DataType(TypeId::Bool);
    case pq::T_INT32:
      if (is_decimal) { *out_kind = PQ_OUT_DEC128; return DataType::decimal(se.precision, se.scale); }
      *out_kind = PQ_OUT_I32;
      return DataType(is_date ? TypeId::Date32 : TypeId::Int32);
    case pq::T_INT64:
      if (is_decimal) { *out_kind = PQ_OUT_DEC128; return DataType::decimal(se.precision, se.scale); }
      *out_kind = PQ_OUT_I64;
      return DataType(TypeId::Int64);
    case pq::T_DOUBLE: *out_kind = PQ_OUT_F64; return DataType(TypeId::Float64);
    case pq::T_BYTE_ARRAY: *out_kind = PQ_OUT_STRVIEW; return DataType(TypeId::Utf8);
    case pq::T_FLBA:
      if (is_decimal && se.type_length >= 1 && se.type_length <= 16) { *out_kind = PQ_OUT_DEC128; return DataType::decimal(se.precision, se.scale); }
      break;
    default: break;
  }
  throw EngineError(B200_ERR_UNSUPPORTED, "parquet column '" + se.name + "': physical/logical type not supported by the device scan");
}

DevBatchPtr scan_parquet(const Exec& x, const std::string& path, const std::vector<std::string>& want) {
  ScopeTimer tm("parquet_scan");
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) throw EngineError(B200_ERR_NOT_FOUND, "cannot open " + path);
  fseek(f, 0, SEEK_END);
  const size_t fsize = (size_t)ftell(f);
  fseek(f, 0, SEEK_SET);
  struct Pinned {
    uint8_t* p = nullptr;
    ~Pinned() {
      if (p) cudaFreeHost(p);
    }
  } file;
  if (cudaHostAlloc((void**)&file.p, fsize + 64, cudaHostAllocDefault) != cudaSuccess) {
    fclose(f);
    throw EngineError(B200_ERR_OOM, "pinned staging for the parquet file");
  }
  const size_t got = fread(file.p, 1, fsize, f);
  fclose(f);
  if (got != fsize) throw EngineError(B200_ERR_INVALID, "short read on " + path);
  pq::FileMeta fm;
  try {
    fm = pq::read_file_meta(file.p, fsize);
  } catch (const std::runtime_error& ex) {
    throw EngineError(B200_ERR_INVALID, ex.what());
  }
  if (fm.schema.empty()) throw EngineError(B200_ERR_INVALID, "parquet: empty schema");
  const size_t n_leaves = fm.schema.size() - 1;
  if ((size_t)fm.schema[0].num_children != n_leaves) throw EngineError(B200_ERR_UNSUPPORTED, "parquet: nested schemas are not supported by the device scan");
  std::vector<PqHostColumn> cols;
  std::vector<std::string> names = want;
  if (names.empty())
    for (size_t i = 1; i < fm.schema.size(); i++) names.push_back(fm.schema[i].name);
  for (auto& nm : names) {
    PqHostColumn c;
    for (size_t i = 1; i < fm.schema.size(); i++)
      if (fm.schema[i].name == nm) c.leaf = (int)i - 1;
    if (c.leaf < 0) throw EngineError(B200_ERR_INVALID, "parquet: no column named " + nm);
    c.se = fm.schema[(size_t)c.leaf + 1];
    if (c.se.num_children) throw EngineError(B200_ERR_UNSUPPORTED, "parquet: nested column " + nm);
    if (c.se.repetition == 2) throw EngineError(B200_ERR_UNSUPPORTED, "parquet: repeated column " + nm);
    c.optional = c.se.repetition == 1;
    cols.push_back(c);
  }
  cudaStream_t st = x.st();
  int64_t n_rows = 0;
  for (auto& rg : fm.row_groups) n_rows += rg.num_rows;
  // ---- raw bytes to HBM + page tables ---------------------------------------------------------------------------------
  for (auto& c : cols) {
    size_t total = 0;
    for (auto& rg : fm.row_groups) {
      if ((size_t)c.leaf >= rg.columns.size()) throw EngineError(B200_ERR_INVALID, "parquet: row group without column " + c.se.name);
      total += (size_t)rg.columns[(size_t)c.leaf].total_compressed;
    }
    c.raw = dev_alloc(total + 64, st);
    size_t dpos = 0;
    for (auto& rg : fm.row_groups) {
      const pq::ColumnChunkMeta& cm = rg.columns[(size_t)c.leaf];
      if (cm.codec != pq::C_UNCOMPRESSED && cm.codec != pq::C_SNAPPY && cm.codec != pq::C_GZIP && cm.codec != pq::C_LZ4_RAW)
        throw EngineError(B200_ERR_UNSUPPORTED, "parquet: column " + c.se.name + " uses compression codec " + std::to_string(cm.codec) +
                                                    " (the device scan reads UNCOMPRESSED, SNAPPY, GZIP and LZ4_RAW pages)");
      const bool compressed = cm.codec != pq::C_UNCOMPRESSED;
      const size_t dec_before = c.dec_bytes;
      int64_t start = cm.data_page_offset;
      if (cm.dictionary_page_offset > 0 && cm.dictionary_page_offset < start) start = cm.dictionary_page_offset;
      if (start < 0 || (size_t)start + (size_t)cm.total_compressed > fsize) throw EngineError(B200_ERR_INVALID, "parquet: column chunk outside the file");
      CUDA_CHECK(cudaMemcpyAsync((uint8_t*)c.raw->ptr + dpos, file.p + start, (size_t)cm.total_compressed, cudaMemcpyHostToDevice, st));
      const uint8_t* hp = file.p + start;
      const uint8_t* hend = hp + cm.total_compressed;
      const uint8_t* dbase = (const uint8_t*)c.raw->ptr + dpos;
      int64_t chunk_dict_base = c.dict_entries, chunk_values = 0;
      while (hp < hend && chunk_values < cm.num_values) {
        pq::PageHeader h;
        try {
          h = pq::read_page_header(hp, hend);
        } catch (const std::runtime_error& ex) {
          throw EngineError(B200_ERR_INVALID, ex.what());
        }
        const uint8_t* payload = hp + h.header_bytes;
        if (payload + h.compressed_size > hend) throw EngineError(B200_ERR_INVALID, "parquet: page overruns its chunk");
        const uint8_t* dev_payload = dbase + (payload - (file.p + start));
        PqPage pg;
        memset(&pg, 0, sizeof pg);
        pg.n_values = (uint32_t)h.num_values;
        uint32_t plen = (uint32_t)h.compressed_size;   // bytes of the payload the decode kernels will see
        const bool is_data = h.type == pq::P_DATA || h.type == pq::P_DATA_V2;
        const uint32_t v2_levels = h.type == pq::P_DATA_V2 ? (uint32_t)(h.rep_bytes + h.def_bytes) : 0;
        const bool in_dec = compressed && (h.type == pq::P_DICTIONARY || is_data);
        if (in_dec) {
          // the page payload is rebuilt, uncompressed, at c.dec + dec_bytes (the addresses are patched in once c.dec exists)
          plen = (uint32_t)h.uncompressed_size;
          if (v2_levels > (uint32_t)h.compressed_size || v2_levels > plen) throw EngineError(B200_ERR_INVALID, "parquet: level section overruns the page");
          PqDecompJob lv, vj;
          memset(&lv, 0, sizeof lv);
          memset(&vj, 0, sizeof vj);
          if (v2_levels) {  // V2: the levels are never compressed
            lv.src = dev_payload;
            lv.dst = (uint8_t*)c.dec_bytes;
            lv.src_len = lv.dst_len = v2_levels;
            lv.raw_copy = 1;
            lv.codec = (uint32_t)cm.codec;
            c.jobs.push_back(lv);
          }
          vj.src = dev_payload + v2_levels;
          vj.dst = (uint8_t*)(c.dec_bytes + v2_levels);
          vj.src_len = (uint32_t)h.compressed_size - v2_levels;
          vj.dst_len = plen - v2_levels;
          vj.raw_copy = (h.type == pq::P_DATA_V2 && !h.v2_compressed) ? 1 : 0;
          // a stored section is copied byte for byte: its two sizes must agree, or the copy would overrun the payload
          if (vj.raw_copy && vj.src_len != vj.dst_len)
            throw EngineError(B200_ERR_INVALID, "parquet: column " + c.se.name + ": uncompressed V2 page whose compressed and uncompressed sizes differ");
          vj.codec = (uint32_t)cm.codec;
          c.jobs.push_back(vj);
          pg.data = (const uint8_t*)c.dec_bytes;   // offset for now
          c.dec_bytes += ((size_t)plen + 15) & ~(size_t)15;
        } else {
          pg.data = dev_payload;
        }
        if (h.type == pq::P_DICTIONARY) {
          if (h.encoding != pq::E_PLAIN && h.encoding != pq::E_PLAIN_DICTIONARY) throw EngineError(B200_ERR_UNSUPPORTED, "parquet: dictionary page encoding");
          pg.val_off = 0;
          pg.val_len = plen;
          pg.row0 = c.dict_entries;
          chunk_dict_base = c.dict_entries;
          c.dict_entries += h.num_values;
          c.dicts.push_back(pg);
          c.dict_in_dec.push_back(in_dec ? 1 : 0);
        } else if (is_data) {
          if (h.type == pq::P_DATA) {
            if (c.optional) {
              if (h.def_encoding != pq::E_RLE) throw EngineError(B200_ERR_UNSUPPORTED, "parquet: definition levels not RLE encoded");
              if (plen < 4) throw EngineError(B200_ERR_INVALID, "parquet: page too short for its level section");
              pg.v1_levels = 1;   // [u32 length][levels][values]: resolved on the device
            }
            pg.val_off = 0;
            pg.val_len = plen;
          } else {
            if (v2_levels > plen) throw EngineError(B200_ERR_INVALID, "parquet: level section overruns the page");
            pg.def_off = (uint32_t)h.rep_bytes;
            pg.def_len = c.optional ? (uint32_t)h.def_bytes : 0;
            pg.val_off = v2_levels;
            pg.val_len = plen - v2_levels;
          }
          const int32_t ty = c.se.type;
          const bool ints = ty == pq::T_INT32 || ty == pq::T_INT64;
          if (h.encoding == pq::E_PLAIN) pg.encoding = PQ_ENC_PLAIN;
          else if (h.encoding == pq::E_PLAIN_DICTIONARY || h.encoding == pq::E_RLE_DICTIONARY) pg.encoding = PQ_ENC_DICT;
          else if (h.encoding == pq::E_RLE && ty == pq::T_BOOLEAN) pg.encoding = PQ_ENC_RLE_BOOL;
          else if (h.encoding == pq::E_DELTA_BINARY_PACKED && ints) pg.encoding = PQ_ENC_DBP;
          else if (h.encoding == pq::E_DELTA_LENGTH_BYTE_ARRAY && ty == pq::T_BYTE_ARRAY) pg.encoding = PQ_ENC_DLBA;
          else if (h.encoding == pq::E_DELTA_BYTE_ARRAY && (ty == pq::T_BYTE_ARRAY || ty == pq::T_FLBA)) pg.encoding = PQ_ENC_DBA;
          else if (h.encoding == pq::E_BYTE_STREAM_SPLIT && (ints || ty == pq::T_DOUBLE || ty == pq::T_FLBA)) pg.encoding = PQ_ENC_BSS;
          else
            throw EngineError(B200_ERR_UNSUPPORTED, "parquet: column " + c.se.name + " uses encoding " + std::to_string(h.encoding) +
                                                        " (supported: PLAIN, RLE_DICTIONARY, DELTA_BINARY_PACKED for integers, DELTA_LENGTH_BYTE_ARRAY and "
                                                        "DELTA_BYTE_ARRAY for byte arrays, BYTE_STREAM_SPLIT for integers, doubles and fixed-length decimals)");
          if (pg.encoding >= PQ_ENC_DBP) {
            c.delta_pages++;
            c.delta_bytes += plen;
            if (pg.encoding == PQ_ENC_DBA) c.dba_pages++;
          }
          pg.row0 = c.rows;
          pg.dict_base = chunk_dict_base;
          c.rows += h.num_values;
          chunk_values += h.num_values;
          c.pages.push_back(pg);
          c.page_in_dec.push_back(in_dec ? 1 : 0);
        }  // index pages etc.: skipped
        hp = payload + h.compressed_size;
      }
      if (compressed) c.codec_bytes[cm.codec] += (uint64_t)cm.total_compressed + (uint64_t)(c.dec_bytes - dec_before);
      dpos += (size_t)cm.total_compressed;
    }
    if (c.rows != n_rows) throw EngineError(B200_ERR_INVALID, "parquet: column " + c.se.name + " has " + std::to_string(c.rows) + " values, the file " + std::to_string(n_rows) + " rows");
    if (c.dec_bytes) {
      // compressed chunks: rebuild every page payload uncompressed in HBM (one warp per job, each codec's jobs by its own
      // kernel), then decode as usual
      // The order matters for the error word: pq_snappy_kernel sets it with atomicExch(1), the other kernels OR in their
      // bits, so Snappy (codec 1) must run before GZIP (2) and LZ4_RAW (7) on the stream or it would erase their bits.
      std::stable_sort(c.jobs.begin(), c.jobs.end(), [](const PqDecompJob& a, const PqDecompJob& b) { return a.codec < b.codec; });
      c.dec = dev_alloc(c.dec_bytes + 64, st);
      uint8_t* base = (uint8_t*)c.dec->ptr;
      for (auto& j : c.jobs) j.dst = base + (size_t)j.dst;
      for (size_t i = 0; i < c.pages.size(); i++)
        if (c.page_in_dec[i]) c.pages[i].data = base + (size_t)c.pages[i].data;
      for (size_t i = 0; i < c.dicts.size(); i++)
        if (c.dict_in_dec[i]) c.dicts[i].data = base + (size_t)c.dicts[i].data;
      DevPtr dj = dev_alloc(c.jobs.size() * sizeof(PqDecompJob), st);
      CUDA_CHECK(cudaMemcpyAsync(dj->ptr, c.jobs.data(), c.jobs.size() * sizeof(PqDecompJob), cudaMemcpyHostToDevice, st));
      DevPtr err = dev_alloc(16, st);
      CUDA_CHECK(cudaMemsetAsync(err->ptr, 0, 16, st));
      // a column of one codec keeps the Snappy kernel's historical byte count (the column's allocation + rebuilt bytes)
      const bool one_codec = c.codec_bytes.size() == 1;
      for (size_t j0 = 0; j0 < c.jobs.size();) {
        size_t j1 = j0;
        while (j1 < c.jobs.size() && c.jobs[j1].codec == c.jobs[j0].codec) j1++;
        const int32_t codec = (int32_t)c.jobs[j0].codec;
        const PqDecompJob* jobs = (const PqDecompJob*)dj->ptr + j0;
        const uint64_t bytes = one_codec ? (uint64_t)c.raw->bytes + (uint64_t)c.dec_bytes : c.codec_bytes[codec];
        unsigned int* e = (unsigned int*)err->ptr;
        if (codec == pq::C_SNAPPY) {
          KernelTimer kt(x, "parquet_snappy", bytes);
          launch_pq_snappy(jobs, (int)(j1 - j0), e, st);
        } else if (codec == pq::C_GZIP) {
          KernelTimer kt(x, "parquet_gzip", bytes);
          launch_pq_inflate(jobs, (int)(j1 - j0), e, st);
        } else {
          KernelTimer kt(x, "parquet_lz4", bytes);
          launch_pq_lz4(jobs, (int)(j1 - j0), e, st);
        }
        j0 = j1;
      }
      const unsigned int* herr = x.fetch<unsigned int>(err->ptr);
      const std::string cname = c.se.name;
      x.defer([herr, cname, dj, err]() {
        if (!*herr) return;
        std::string what;
        const char* names[3] = {"Snappy", "GZIP", "LZ4_RAW"};
        for (int k = 0; k < 3; k++)
          if (*herr & (1u << k)) what += (what.empty() ? "" : "/") + std::string(names[k]);
        throw EngineError(B200_ERR_INVALID, "parquet: corrupt " + what + " data in column " + cname);
      });
    }
  }
  // ---- decode ------------------------------------------------------------------------------------------------------------
  struct ColWork {
    PqColumn pc;
    DataType type;
    DevPtr d_pages, d_dicts, valid, nonnull, dense_base, total, dict, out;
    const unsigned long long* h_total = nullptr;
    int width = 0;
    // DELTA / BYTE_STREAM_SPLIT pages (launch_pq_delta_prepare, launch_pq_values_delta)
    PqDeltaAux aux;
    DevPtr d_err, pre, sfx, page_bytes, char_base, char_total, chars;
    const unsigned int* h_err = nullptr;
    const unsigned long long* h_chars = nullptr;
  };
  std::vector<ColWork> work(cols.size());
  auto upload = [&](const std::vector<PqPage>& v) {
    DevPtr d = dev_alloc(std::max<size_t>(v.size(), 1) * sizeof(PqPage), st);
    if (!v.empty()) CUDA_CHECK(cudaMemcpyAsync(d->ptr, v.data(), v.size() * sizeof(PqPage), cudaMemcpyHostToDevice, st));  // pageable: staged before returning
    return d;
  };
  for (size_t ci = 0; ci < cols.size(); ci++) {
    PqHostColumn& c = cols[ci];
    ColWork& w = work[ci];
    memset(&w.pc, 0, sizeof w.pc);
    int kind = 0;
    w.type = pq_arrow_type(c.se, &kind);
    w.pc.phys = c.se.type;
    w.pc.type_length = c.se.type_length;
    w.pc.out_kind = kind;
    w.width = kind == PQ_OUT_I32 ? 4 : (kind == PQ_OUT_I64 || kind == PQ_OUT_F64) ? 8 : kind == PQ_OUT_BOOL8 ? 1 : 16;
    w.d_pages = upload(c.pages);
    w.d_dicts = upload(c.dicts);
    if (c.dict_entries) {
      w.dict = dev_alloc((size_t)c.dict_entries * (size_t)w.width + 64, st);
      w.pc.dict = w.dict->ptr;
      launch_pq_dict(w.pc, (const PqPage*)w.d_dicts->ptr, (int)c.dicts.size(), st);
    }
    if (c.optional) {
      w.valid = dev_alloc((size_t)std::max<int64_t>(n_rows, 1) + 64, st);
      w.nonnull = dev_alloc(std::max<size_t>(c.pages.size(), 1) * 4, st);
      w.dense_base = dev_alloc(std::max<size_t>(c.pages.size(), 1) * 8, st);
      w.total = dev_alloc(16, st);
      CUDA_CHECK(cudaMemsetAsync(w.total->ptr, 0, 16, st));
      launch_pq_levels((const PqPage*)w.d_pages->ptr, (int)c.pages.size(), (uint8_t*)w.valid->ptr, (uint32_t*)w.nonnull->ptr, (unsigned long long*)w.total->ptr, st);
      launch_pq_page_scan((const uint32_t*)w.nonnull->ptr, (int)c.pages.size(), (unsigned long long*)w.dense_base->ptr, st);
      w.h_total = x.fetch<unsigned long long>(w.total->ptr);
    }
    if (c.delta_pages) {
      // validate the DELTA / BYTE_STREAM_SPLIT pages and size the DELTA_BYTE_ARRAY strings before anything is decoded
      memset(&w.aux, 0, sizeof w.aux);
      w.d_err = dev_alloc(16, st);
      CUDA_CHECK(cudaMemsetAsync(w.d_err->ptr, 0, 16, st));
      w.aux.error = (unsigned int*)w.d_err->ptr;
      const bool dba_strings = c.dba_pages && c.se.type == pq::T_BYTE_ARRAY;
      if (c.dba_pages) {
        w.pre = dev_alloc((size_t)std::max<int64_t>(n_rows, 1) * 4 + 64, st);
        w.sfx = dev_alloc((size_t)std::max<int64_t>(n_rows, 1) * 4 + 64, st);
        w.aux.pre = (uint32_t*)w.pre->ptr;
        w.aux.sfx = (uint32_t*)w.sfx->ptr;
      }
      if (dba_strings) {
        w.page_bytes = dev_alloc(c.pages.size() * 4, st);
        w.char_base = dev_alloc(c.pages.size() * 8, st);
        w.char_total = dev_alloc(16, st);
        CUDA_CHECK(cudaMemsetAsync(w.char_total->ptr, 0, 16, st));
        w.aux.page_bytes = (uint32_t*)w.page_bytes->ptr;
        w.aux.char_total = (unsigned long long*)w.char_total->ptr;
        w.aux.char_base = (const unsigned long long*)w.char_base->ptr;
      }
      {
        KernelTimer kt(x, "parquet_delta_prepare", c.delta_bytes + (c.dba_pages ? (uint64_t)n_rows * 8 : 0));
        launch_pq_delta_prepare(w.pc, (const PqPage*)w.d_pages->ptr, (int)c.pages.size(), c.optional ? (const unsigned long long*)w.dense_base->ptr : nullptr,
                                c.optional ? (const uint32_t*)w.nonnull->ptr : nullptr, w.aux, st);
        if (dba_strings) {
          launch_pq_page_scan((const uint32_t*)w.page_bytes->ptr, (int)c.pages.size(), (unsigned long long*)w.char_base->ptr, st);
        }
      }
      w.h_err = x.fetch<unsigned int>(w.d_err->ptr);
      if (dba_strings) w.h_chars = x.fetch<unsigned long long>(w.char_total->ptr);
    }
  }
  x.sync();  // one read-back for all nullable columns (which of them really contain NULLs) and all DELTA / BYTE_STREAM_SPLIT checks
  for (size_t ci = 0; ci < cols.size(); ci++) {
    ColWork& w = work[ci];
    if (w.h_err && *w.h_err)
      throw EngineError(B200_ERR_INVALID, "parquet: column " + cols[ci].se.name + " has a malformed DELTA_BINARY_PACKED, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY or BYTE_STREAM_SPLIT page");
    if (w.h_chars) {
      w.chars = dev_alloc((size_t)*w.h_chars + 64, st);
      w.aux.chars = (uint8_t*)w.chars->ptr;
    }
  }
  auto out = std::make_shared<DevBatch>();
  out->n = n_rows;
  for (size_t ci = 0; ci < cols.size(); ci++) {
    PqHostColumn& c = cols[ci];
    ColWork& w = work[ci];
    const bool has_nulls = c.optional && (int64_t)*w.h_total != n_rows;
    w.out = dev_alloc((size_t)std::max<int64_t>(n_rows, 1) * (size_t)w.width + 64, st);
    {
      KernelTimer kt(x, "parquet_decode_values", (uint64_t)n_rows * (uint64_t)w.width);
      if (!has_nulls) {
        launch_pq_values(w.pc, (const PqPage*)w.d_pages->ptr, (int)c.pages.size(), nullptr, nullptr, w.out->ptr, st);
        if (c.delta_pages) {
          launch_pq_values_delta(w.pc, (const PqPage*)w.d_pages->ptr, (int)c.pages.size(), nullptr, nullptr, w.out->ptr, w.aux, st);
        }
      } else {
        DevPtr dense = dev_alloc((size_t)std::max<int64_t>(n_rows, 1) * (size_t)w.width + 64, st);
        launch_pq_values(w.pc, (const PqPage*)w.d_pages->ptr, (int)c.pages.size(), (const unsigned long long*)w.dense_base->ptr, (const uint32_t*)w.nonnull->ptr, dense->ptr, st);
        if (c.delta_pages) {
          launch_pq_values_delta(w.pc, (const PqPage*)w.d_pages->ptr, (int)c.pages.size(), (const unsigned long long*)w.dense_base->ptr, (const uint32_t*)w.nonnull->ptr,
                                 dense->ptr, w.aux, st);
        }
        launch_pq_expand((const PqPage*)w.d_pages->ptr, (int)c.pages.size(), (const unsigned long long*)w.dense_base->ptr, (const uint8_t*)w.valid->ptr, dense->ptr,
                         w.out->ptr, w.width, st);
      }
    }
    DevColumn col;
    col.name = c.se.name;
    col.type = w.type;
    col.n = n_rows;
    col.nullable = has_nulls;
    col.phys = w.pc.out_kind == PQ_OUT_STRVIEW ? PH_STRVIEW : phys_of(w.type);
    col.data = (const uint8_t*)w.out->ptr;
    col.keep.push_back(w.out);
    if (has_nulls) {
      col.valid = (const uint8_t*)w.valid->ptr;
      col.keep.push_back(w.valid);
    }
    if (col.phys == PH_STRVIEW) {
      // registered tables use the canonical Arrow layout (offsets + contiguous characters): the views into the raw pages
      // are compacted once, here, and the raw pages are released
      col.keep.push_back(c.raw);
      if (c.dec) col.keep.push_back(c.dec);
      if (w.dict) col.keep.push_back(w.dict);
      if (w.chars) col.keep.push_back(w.chars);  // DELTA_BYTE_ARRAY strings rebuilt on the device
      col = as_utf8(x, col);
    }
    out->cols.push_back(col);
  }
  build_column_images(x, *out);
  x.sync();
  return out;
}

// ------------------------------------------------------------------------------------------------
// CSV scan: DataSourceExec + CsvSource (CsvScanExecNode, ballista/core/proto/datafusion.proto:1088-1101; TPC-H .tbl files,
// benchmarks/src/bin/tpch.rs:653-683).  The host finds the byte span of each file (range rule below), streams it to HBM
// through two bounded pinned chunks and csrc/device/csv.cu does everything else.  Rules: DESIGN.md §6 (ix).
// ------------------------------------------------------------------------------------------------
struct CsvFileSpec {
  std::string path;
  int64_t start = 0, end = -1;  // end < 0: the whole file
};
struct CsvScanSpec {
  std::vector<CsvFileSpec> files;
  Schema schema;
  std::vector<std::string> columns;
  bool all_columns = true;  // no "columns" key; an empty list materialises no column (the rows are still counted)
  bool has_header = false, newlines_in_values = false;
  CsvDialect d{',', '"', 0, 0};
};

static uint8_t csv_option_byte(const Json& j, const char* key, uint8_t dflt) {
  const Json* v = j.find(key);
  if (!v || v->is_null()) return dflt;
  if (!v->is_str() || v->str().size() != 1)
    throw EngineError(B200_ERR_INVALID, std::string("csv: option '") + key + "' must be exactly one byte");
  return (uint8_t)v->str()[0];
}

static CsvScanSpec parse_csv_scan(const std::string& text) {
  Json j;
  try {
    j = parse_json(text);
  } catch (const std::exception& ex) {
    throw EngineError(B200_ERR_INVALID, std::string("csv: malformed scan description: ") + ex.what());
  }
  if (!j.is_obj()) throw EngineError(B200_ERR_INVALID, "csv: the scan description must be a JSON object");
  CsvScanSpec s;
  try {
    const Json* c = j.find("comment");
    if (c && !c->is_null()) throw EngineError(B200_ERR_UNSUPPORTED, "csv: option 'comment' is not supported");
    if (j.get_bool("truncate_rows", false)) throw EngineError(B200_ERR_UNSUPPORTED, "csv: option 'truncate_rows' is not supported");
    s.has_header = j.get_bool("has_header", false);
    s.newlines_in_values = j.get_bool("newlines_in_values", false);
    s.d.delim = csv_option_byte(j, "delimiter", ',');
    s.d.quote = csv_option_byte(j, "quote", '"');
    const Json* esc = j.find("escape");
    if (esc && !esc->is_null()) {
      s.d.escape = csv_option_byte(j, "escape", 0);
      s.d.has_escape = s.d.escape != s.d.quote;  // an escape equal to the quote is the doubled-quote rule
    }
    for (uint8_t b : {s.d.delim, s.d.quote})
      if (b == '\n' || b == '\r') throw EngineError(B200_ERR_INVALID, "csv: delimiter and quote cannot be line terminators");
    if (s.d.delim == s.d.quote || (s.d.has_escape && (s.d.escape == s.d.delim || s.d.escape == '\n' || s.d.escape == '\r')))
      throw EngineError(B200_ERR_INVALID, "csv: delimiter, quote and escape must be distinct bytes");
    s.schema = parse_schema(j.at("schema"));
    if (s.schema.empty()) throw EngineError(B200_ERR_INVALID, "csv: empty schema");
    const Json* cols = j.find("columns");
    if (cols && !cols->is_null()) {
      if (!cols->is_arr()) throw EngineError(B200_ERR_INVALID, "csv: 'columns' must be a list of names");
      s.all_columns = false;
      for (size_t i = 0; i < cols->size(); i++) s.columns.push_back(cols->at(i).str());
    }
    const Json& files = j.at("files");
    if (!files.is_arr() || files.size() == 0) throw EngineError(B200_ERR_INVALID, "csv: 'files' must be a non-empty list");
    for (size_t i = 0; i < files.size(); i++) {
      const Json& f = files.at(i);
      CsvFileSpec fs;
      if (f.is_str()) {
        fs.path = f.str();
      } else {
        fs.path = f.at("path").str();
        const Json* r = f.find("range");
        if (r && !r->is_null()) {
          if (r->size() != 2) throw EngineError(B200_ERR_INVALID, "csv: a range is [start, end]");
          fs.start = r->at(0).as_int();
          fs.end = r->at(1).as_int();
          if (fs.start < 0 || fs.end < fs.start) throw EngineError(B200_ERR_INVALID, "csv: bad byte range of " + fs.path);
          if (s.newlines_in_values)
            throw EngineError(B200_ERR_UNSUPPORTED, "csv: byte ranges together with 'newlines_in_values' are not supported");
        }
      }
      s.files.push_back(fs);
    }
  } catch (const EngineError&) {
    throw;
  } catch (const std::exception& ex) {
    throw EngineError(B200_ERR_INVALID, std::string("csv: ") + ex.what());
  }
  return s;
}

static int csv_family(const Field& f) {
  const DataType& t = f.type;
  if (t.is_integer()) return CSV_FAM_INT;
  if (t.is_decimal()) {
    if (t.precision < 1 || t.precision > 38 || t.scale < 0 || t.scale > t.precision)
      throw EngineError(B200_ERR_UNSUPPORTED, "csv: column '" + f.name + "' has type " + t.str() + ", which the CSV scan does not read");
    return CSV_FAM_DEC;
  }
  if (t.id == TypeId::Float64) return CSV_FAM_F64;
  if (t.id == TypeId::Float32) return CSV_FAM_F32;
  if (t.id == TypeId::Date32) return CSV_FAM_DATE;
  if (t.id == TypeId::Bool) return CSV_FAM_BOOL;
  if (t.id == TypeId::Utf8) return CSV_FAM_UTF8;
  throw EngineError(B200_ERR_UNSUPPORTED, "csv: column '" + f.name + "' has type " + t.str() + ", which the CSV scan does not read");
}

static const char* csv_reason(int r) {
  switch (r) {
    case CSV_E_FIELDS: return "wrong number of fields";
    case CSV_E_NULL: return "NULL in a non-nullable column";
    case CSV_E_INT: return "not an integer";
    case CSV_E_INT_RANGE: return "integer out of range";
    case CSV_E_DEC: return "not a decimal";
    case CSV_E_DEC_RANGE: return "decimal does not fit the precision";
    case CSV_E_DEC_SCALE: return "decimal has more fractional digits than the scale";
    case CSV_E_DEC_EXP: return "decimal with an exponent";
    case CSV_E_FLOAT: return "not a floating-point number";
    case CSV_E_DATE: return "not a valid YYYY-MM-DD date";
    case CSV_E_BOOL: return "not a boolean";
    case CSV_E_UTF8: return "invalid UTF-8";
    default: return "malformed value";
  }
}

// one file's byte span [s0, e0) on the device and where its records are
struct CsvSpan {
  std::string path;
  int64_t s0 = 0, e0 = 0, skip = 0, n_records = 0, rows = 0, row_base = 0;
  DevPtr data, tiles, blocks, blk_state, blk_base, counts, rec_start, side;
  const unsigned long long* h_n = nullptr;
  const unsigned int* h_quote = nullptr;
};

// first line terminator at or after `pos` (the file's size when there is none)
static int64_t csv_find_term(FILE* f, int64_t pos, int64_t size) {
  char buf[4096];
  while (pos < size) {
    if (fseeko(f, (off_t)pos, SEEK_SET) != 0) throw EngineError(B200_ERR_INVALID, "csv: seek failed");
    const size_t n = fread(buf, 1, sizeof buf, f);
    if (n == 0) break;
    for (size_t i = 0; i < n; i++)
      if (buf[i] == '\n' || buf[i] == '\r') return pos + (int64_t)i;
    pos += (int64_t)n;
  }
  return size;
}

DevBatchPtr scan_csv(const Exec& x, const CsvScanSpec& spec) {
  ScopeTimer tm("csv_scan");
  cudaStream_t st = x.st();
  const Schema& sch = spec.schema;
  // materialised columns, in the requested order
  std::vector<int> mat;
  if (spec.all_columns) {
    for (size_t i = 0; i < sch.size(); i++) mat.push_back((int)i);
  } else {
    for (auto& nm : spec.columns) {
      int at = -1;
      for (size_t i = 0; i < sch.size(); i++)
        if (sch[i].name == nm) at = (int)i;
      if (at < 0) throw EngineError(B200_ERR_INVALID, "csv: no column named " + nm);
      // every schema column feeds at most one output slot (csv_fields_kernel writes one view per field)
      if (std::find(mat.begin(), mat.end(), at) != mat.end()) throw EngineError(B200_ERR_INVALID, "csv: column " + nm + " is requested twice");
      mat.push_back(at);
    }
  }
  std::vector<int> fam;
  for (int c : mat) fam.push_back(csv_family(sch[(size_t)c]));
  std::vector<int32_t> slot_of_field(sch.size(), -1);
  for (size_t k = 0; k < mat.size(); k++) slot_of_field[(size_t)mat[k]] = (int32_t)k;

  // ---- bytes to HBM: two pinned chunks in flight, whatever the file size --------------------------------------------------
  static const size_t kChunk = 16u << 20;
  struct Staging {
    uint8_t* buf[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    ~Staging() {
      for (int b = 0; b < 2; b++) {
        if (ev[b]) {
          cudaEventSynchronize(ev[b]);
          cudaEventDestroy(ev[b]);
        }
        if (buf[b]) cudaFreeHost(buf[b]);
      }
    }
  } stg;
  for (int b = 0; b < 2; b++) {
    if (cudaHostAlloc((void**)&stg.buf[b], kChunk, cudaHostAllocDefault) != cudaSuccess) throw EngineError(B200_ERR_OOM, "pinned staging for the CSV scan");
    CUDA_CHECK(cudaEventCreateWithFlags(&stg.ev[b], cudaEventDisableTiming));
  }
  std::vector<CsvSpan> spans(spec.files.size());
  int64_t chunk_no = 0;
  for (size_t fi = 0; fi < spec.files.size(); fi++) {
    const CsvFileSpec& fs = spec.files[fi];
    CsvSpan& sp = spans[fi];
    sp.path = fs.path;
    FILE* f = fopen(fs.path.c_str(), "rb");
    if (!f) throw EngineError(B200_ERR_NOT_FOUND, "csv: cannot open " + fs.path);
    std::unique_ptr<FILE, int (*)(FILE*)> closer(f, fclose);
    const int64_t size = fseeko(f, 0, SEEK_END) == 0 ? (int64_t)ftello(f) : -1;
    if (size < 0) throw EngineError(B200_ERR_INVALID, "csv: cannot size " + fs.path);
    const int64_t start = std::min<int64_t>(fs.start, size);
    const int64_t end = fs.end < 0 ? size : std::min<int64_t>(fs.end, size);
    // a range holds the records whose first byte lies in [start, end): from after the first terminator at or after
    // start - 1, through the first terminator at or after end - 1
    sp.s0 = start == 0 ? 0 : std::min(size, csv_find_term(f, start - 1, size) + 1);
    sp.e0 = end == 0 ? 0 : end >= size ? size : std::min(size, csv_find_term(f, end - 1, size) + 1);
    if (sp.e0 < sp.s0) sp.e0 = sp.s0;
    sp.skip = (spec.has_header && start == 0) ? 1 : 0;
    const int64_t bytes = sp.e0 - sp.s0;
    sp.data = dev_alloc((size_t)bytes + 64, st);
    for (int64_t off = 0; off < bytes; chunk_no++) {
      const int b = (int)(chunk_no & 1);
      const size_t n = (size_t)std::min<int64_t>((int64_t)kChunk, bytes - off);
      CUDA_CHECK(cudaEventSynchronize(stg.ev[b]));  // the copy out of this chunk two steps ago is done
      if (fseeko(f, (off_t)(sp.s0 + off), SEEK_SET) != 0 || fread(stg.buf[b], 1, n, f) != n) throw EngineError(B200_ERR_INVALID, "csv: short read on " + fs.path);
      CUDA_CHECK(cudaMemcpyAsync((uint8_t*)sp.data->ptr + off, stg.buf[b], n, cudaMemcpyHostToDevice, st));
      CUDA_CHECK(cudaEventRecord(stg.ev[b], st));
      off += (int64_t)n;
    }
    if (bytes == 0) continue;
    const int64_t nt = csv_tile_count(bytes), nb = csv_block_count(bytes);
    sp.tiles = dev_alloc((size_t)nt * sizeof(CsvTrans), st);
    sp.blocks = dev_alloc((size_t)nb * sizeof(CsvTrans), st);
    sp.blk_state = dev_alloc((size_t)nb, st);
    sp.blk_base = dev_alloc((size_t)nb * 8, st);
    sp.counts = dev_alloc(16, st);
    CUDA_CHECK(cudaMemsetAsync(sp.counts->ptr, 0, 16, st));
    unsigned long long* n_rec = (unsigned long long*)sp.counts->ptr;
    unsigned int* quote = (unsigned int*)(n_rec + 1);
    {
      KernelTimer kt(x, "csv_records", (uint64_t)bytes + (uint64_t)nt * sizeof(CsvTrans));
      launch_csv_records_count((const uint8_t*)sp.data->ptr, bytes, spec.d, (CsvTrans*)sp.tiles->ptr, (CsvTrans*)sp.blocks->ptr, (uint8_t*)sp.blk_state->ptr,
                               (unsigned long long*)sp.blk_base->ptr, quote, n_rec, st);
    }
    sp.h_n = x.fetch<unsigned long long>(n_rec);
    sp.h_quote = x.fetch<unsigned int>(quote);
  }
  x.sync();  // one read-back for every file: record counts and whether any quote byte occurs
  int64_t n_total = 0;
  for (auto& sp : spans) {
    sp.n_records = sp.h_n ? (int64_t)*sp.h_n : 0;
    sp.rows = std::max<int64_t>(sp.n_records - sp.skip, 0);
    sp.row_base = n_total;
    n_total += sp.rows;
  }
  const size_t n_mat = mat.size();
  DevPtr views = dev_alloc(std::max<size_t>(n_mat * (size_t)n_total, 1) * 16 + 64, st);
  DevPtr d_slots = dev_alloc(slot_of_field.size() * 4, st);
  CUDA_CHECK(cudaMemcpyAsync(d_slots->ptr, slot_of_field.data(), slot_of_field.size() * 4, cudaMemcpyHostToDevice, st));  // pageable: staged before returning
  // error words: [0] field counts, [1 + k] column k; then the null count of every column
  DevPtr words = dev_alloc((1 + 2 * n_mat) * 8, st);
  CUDA_CHECK(cudaMemsetAsync(words->ptr, 0xFF, (1 + n_mat) * 8, st));
  CUDA_CHECK(cudaMemsetAsync((unsigned long long*)words->ptr + 1 + n_mat, 0, n_mat * 8, st));
  unsigned long long* w = (unsigned long long*)words->ptr;
  for (auto& sp : spans) {
    const int64_t bytes = sp.e0 - sp.s0;
    if (!sp.n_records) continue;
    sp.rec_start = dev_alloc((size_t)sp.n_records * 8, st);
    {
      KernelTimer kt(x, "csv_records", (uint64_t)bytes + (uint64_t)sp.n_records * 8);
      launch_csv_record_starts((const uint8_t*)sp.data->ptr, bytes, spec.d, (const CsvTrans*)sp.tiles->ptr, (const uint8_t*)sp.blk_state->ptr,
                               (const unsigned long long*)sp.blk_base->ptr, (uint64_t*)sp.rec_start->ptr, st);
    }
    sp.tiles.reset();
    sp.blocks.reset();
    if (*sp.h_quote) sp.side = dev_alloc((size_t)bytes + 64, st);
    CsvFieldArgs A;
    memset(&A, 0, sizeof A);
    A.data = (const uint8_t*)sp.data->ptr;
    A.bytes = bytes;
    A.rec_start = (const uint64_t*)sp.rec_start->ptr;
    A.n_records = sp.n_records;
    A.skip = sp.skip;
    A.d = spec.d;
    A.n_fields = (int)sch.size();
    A.slot_of_field = (const int32_t*)d_slots->ptr;
    A.views = (unsigned long long*)views->ptr;
    A.n_total = n_total;
    A.row_base = sp.row_base;
    A.side = sp.side ? (uint8_t*)sp.side->ptr : nullptr;
    A.err = w;
    KernelTimer kt(x, "csv_fields", (uint64_t)bytes + (uint64_t)sp.n_records * 8 + (uint64_t)sp.rows * n_mat * 16);
    launch_csv_fields(A, st);
  }
  std::vector<DevPtr> outs(n_mat), valids(n_mat);
  for (size_t k = 0; k < n_mat; k++) {
    const Field& f = sch[(size_t)mat[k]];
    CsvConvertArgs C;
    memset(&C, 0, sizeof C);
    C.views = (const unsigned long long*)views->ptr + 2 * k * (size_t)n_total;
    C.n = n_total;
    C.width = fam[k] == CSV_FAM_UTF8 ? 16 : f.type.is_decimal() ? 16 : f.type.id == TypeId::Bool ? 1 : f.type.width();
    // Utf8 views are validated in place
    outs[k] = fam[k] == CSV_FAM_UTF8 ? views : dev_alloc((size_t)std::max<int64_t>(n_total, 1) * (size_t)C.width + 64, st);
    C.out = fam[k] == CSV_FAM_UTF8 ? (void*)C.views : outs[k]->ptr;
    valids[k] = dev_alloc((size_t)std::max<int64_t>(n_total, 1) + 64, st);
    C.valid = (uint8_t*)valids[k]->ptr;
    C.err = w + 1 + k;
    C.null_count = w + 1 + n_mat + k;
    C.is_signed = f.type.is_signed_int();
    if (fam[k] == CSV_FAM_INT) {
      const int bits = 8 * f.type.width();
      C.lo = C.is_signed ? -((__int128)1 << (bits - 1)) : 0;
      C.hi = C.is_signed ? ((__int128)1 << (bits - 1)) - 1 : ((__int128)1 << bits) - 1;
    }
    C.precision = f.type.precision;
    C.scale = f.type.scale;
    C.nullable = f.nullable ? 1 : 0;
    KernelTimer kt(x, "csv_convert", (uint64_t)n_total * (16 + (uint64_t)C.width + 1));
    launch_csv_convert(C, fam[k], st);
  }
  const unsigned long long* hw = (const unsigned long long*)x.fetch_bytes(w, (1 + 2 * n_mat) * 8);
  x.sync();
  // the first failing record of the scan, a field-count error first among equals
  int which = -1;
  unsigned long long best = ~0ull;
  for (size_t k = 0; k <= n_mat; k++)
    if (hw[k] != ~0ull && (hw[k] >> 24) < (best >> 24)) {
      best = hw[k];
      which = (int)k - 1;
    }
  if (best != ~0ull) {
    const int64_t row = (int64_t)(best >> 24);
    const int reason = (int)((best >> 16) & 0xFF), detail = (int)(best & 0xFFFF);
    size_t fi = 0;
    while (fi + 1 < spans.size() && !(row >= spans[fi].row_base && row < spans[fi].row_base + spans[fi].rows)) fi++;
    const CsvSpan& sp = spans[fi];
    const int64_t rec = row - sp.row_base + sp.skip;
    const uint64_t rel = x.get<uint64_t>((const uint64_t*)sp.rec_start->ptr + rec);
    std::string value;
    if (which >= 0) {
      const unsigned long long* v = (const unsigned long long*)views->ptr + 2 * ((size_t)which * (size_t)n_total + (size_t)row);
      const unsigned long long* hv = (const unsigned long long*)x.fetch_bytes(v, 16);
      x.sync();
      const uint64_t len = std::min<uint64_t>(hv[1], 64);
      if (len) {
        const char* hb = (const char*)x.fetch_bytes((const void*)hv[0], (size_t)len);
        x.sync();
        value.assign(hb, (size_t)len);
      }
      if (hv[1] > 64) value += "...";
    } else {
      const uint64_t len = std::min<uint64_t>(64, (uint64_t)(sp.e0 - sp.s0) - rel);
      const char* hb = (const char*)x.fetch_bytes((const uint8_t*)sp.data->ptr + rel, (size_t)len);
      x.sync();
      value.assign(hb, (size_t)len);
      const size_t nl = value.find_first_of("\r\n");
      if (nl != std::string::npos) value.resize(nl);
      else if (len == 64) value += "...";
    }
    std::string what = csv_reason(reason);
    if (reason == CSV_E_FIELDS) what = "record has " + std::to_string(detail) + " fields, the schema " + std::to_string(sch.size());
    const std::string col = which >= 0 ? "column '" + sch[(size_t)mat[(size_t)which]].name + "', " : "";
    throw EngineError(B200_ERR_INVALID, "csv: " + sp.path + ": " + col + "record " + std::to_string(row - sp.row_base + 1) + " (byte offset " +
                                            std::to_string((uint64_t)sp.s0 + rel) + "): " + what + ": '" + value + "'");
  }
  auto out = std::make_shared<DevBatch>();
  out->n = n_total;
  for (size_t k = 0; k < n_mat; k++) {
    const Field& f = sch[(size_t)mat[k]];
    const bool has_nulls = hw[1 + n_mat + k] != 0;
    DevColumn col;
    col.name = f.name;
    col.type = f.type;
    col.n = n_total;
    col.nullable = has_nulls;
    if (has_nulls) {
      col.valid = (const uint8_t*)valids[k]->ptr;
      col.keep.push_back(valids[k]);
    }
    if (fam[k] == CSV_FAM_UTF8) {
      col.phys = PH_STRVIEW;
      col.data = (const uint8_t*)views->ptr + 16 * k * (size_t)n_total;
      col.keep.push_back(views);
      for (auto& sp : spans) {
        col.keep.push_back(sp.data);
        if (sp.side) col.keep.push_back(sp.side);
      }
      KernelTimer kt(x, "csv_strings", (uint64_t)n_total * 16 * 2);
      col = as_utf8(x, col);
    } else {
      col.phys = phys_of(f.type);
      col.data = (const uint8_t*)outs[k]->ptr;
      col.keep.push_back(outs[k]);
    }
    out->cols.push_back(col);
  }
  build_column_images(x, *out);
  x.sync();
  return out;
}

void collect_nodes(const PlanNode& n, b200_stage* s) {
  s->metric_index[&n] = (int)s->metrics.size();
  OpMetrics m;
  m.name = n.op_name;
  s->metrics.push_back(m);
  for (auto& c : n.children) collect_nodes(*c, s);
}

int table_id(const std::string& name) {
  static const char* names[] = {"lineitem", "orders", "customer", "supplier", "part", "partsupp", "nation", "region"};
  for (int i = 0; i < 8; i++)
    if (name == names[i]) return i;
  return -1;
}

template <class F>
int guard(F&& f) {
  try {
    f();
    return B200_OK;
  } catch (const EngineError& e) {
    g_err = e.what();
    return e.code;
  } catch (const PlanUnsupported& e) {
    g_err = e.what();
    return B200_ERR_UNSUPPORTED;
  } catch (const std::bad_alloc&) {
    g_err = "host out of memory";
    return B200_ERR_OOM;
  } catch (const std::exception& e) {
    g_err = e.what();
    return B200_ERR_INVALID;
  } catch (...) {
    g_err = "unknown error";
    return B200_ERR_INVALID;
  }
}

// guard() for an entry point that launches kernels for engine e: what this thread enqueued during the call, whether it
// succeeds or fails, goes to e's count (b200_engine_kernel_launches)
template <class F>
int guard(b200_engine* e, F&& f) {
  const uint64_t l0 = launches_on_thread();
  const int rc = guard(std::forward<F>(f));
  if (e) e->launches += launches_on_thread() - l0;
  return rc;
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
// ---- exchange window (fused shuffle): allocate, publish through CUDA IPC, map every peer's ---------------------------------
static void release_window(b200_engine* e) {
  for (size_t d = 0; d < e->win_peer.size(); d++)
    if (e->win_peer[d] && (int)d != e->rank) cudaIpcCloseMemHandle(e->win_peer[d]);
  e->win_peer.clear();
  if (e->win_local) cudaFree(e->win_local);
  e->win_local = nullptr;
  e->win_bytes = e->win_used = 0;
}

// all-gather of one fixed-size record per executor over the exchange communicator (setup path only)
static void comm_allgather(b200_engine* e, const void* mine, void* all, size_t rec) {
  NcclApi& N = NcclApi::get();
  const int W = e->world, me = e->rank;
  uint8_t* dev = nullptr;
  CUDA_CHECK(cudaMalloc((void**)&dev, rec * (size_t)W));
  try {
    CUDA_CHECK(cudaMemcpyAsync(dev + rec * (size_t)me, mine, rec, cudaMemcpyHostToDevice, e->stream));
    NCCL_CHECK(N.GroupStart());
    for (int d = 0; d < W; d++) {
      if (d == me) continue;
      NCCL_CHECK(N.Send(dev + rec * (size_t)me, rec, kNcclUint8, d, e->comm, e->stream));
      NCCL_CHECK(N.Recv(dev + rec * (size_t)d, rec, kNcclUint8, d, e->comm, e->stream));
    }
    NCCL_CHECK(N.GroupEnd());
    CUDA_CHECK(cudaMemcpyAsync(all, dev, rec * (size_t)W, cudaMemcpyDeviceToHost, e->stream));
    CUDA_CHECK(host_wait(e, e->stream));
  } catch (...) {
    cudaFree(dev);
    throw;
  }
  cudaFree(dev);
}

// Collective (called from b200_engine_comm_init on every executor).  Any executor that cannot provide or map a window
// makes all of them run without one: the fused shuffle needs every peer, the two-step exchange none.
static void setup_window(b200_engine* e) {
  const int W = e->world, me = e->rank;
  struct Rec {
    cudaIpcMemHandle_t h;
    uint64_t bytes, ok;
  };
  Rec mine;
  memset(&mine, 0, sizeof mine);
  const size_t want = (e->win_config_bytes + 4095) & ~(size_t)4095;
  uint8_t* ptr = nullptr;
  if (cudaMalloc((void**)&ptr, want) == cudaSuccess && cudaIpcGetMemHandle(&mine.h, ptr) == cudaSuccess) {
    mine.bytes = want;
    mine.ok = 1;
  } else {
    cudaGetLastError();
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
  }
  std::vector<Rec> all((size_t)W);
  comm_allgather(e, &mine, all.data(), sizeof(Rec));
  bool ok = true;
  for (auto& r : all) ok = ok && r.ok && r.bytes == want;
  std::vector<uint8_t*> peer((size_t)W, nullptr);
  if (ok) {
    for (int d = 0; d < W && ok; d++) {
      if (d == me) {
        peer[(size_t)d] = ptr;
        continue;
      }
      void* m = nullptr;
      if (cudaIpcOpenMemHandle(&m, all[(size_t)d].h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
        cudaGetLastError();
        ok = false;
      }
      peer[(size_t)d] = (uint8_t*)m;
    }
  }
  // second round: did everyone manage to map everyone?
  uint64_t flag = ok ? 1 : 0;
  std::vector<uint64_t> flags((size_t)W, 0);
  comm_allgather(e, &flag, flags.data(), sizeof flag);
  for (uint64_t f : flags) ok = ok && f;
  if (!ok) {
    for (int d = 0; d < W; d++)
      if (d != me && peer[(size_t)d]) cudaIpcCloseMemHandle(peer[(size_t)d]);
    if (ptr) cudaFree(ptr);
    return;
  }
  e->win_local = ptr;
  e->win_bytes = want;
  e->win_used = 0;
  e->win_peer = peer;
}


extern "C" {

const char* b200_version(void) { return "b200exec 0.1 sm_90a"; }
const char* b200_last_error(void) { return g_err.c_str(); }

// Ingest is a host<->GPU pipeline (pinned staging, a pool of narrowing threads, DMA): it only reaches the PCIe rate when
// the host side runs on the NUMA node the GPU hangs off -- across the socket interconnect the same copies run at about
// half speed.  The thread that creates the engine (and every thread it starts later, e.g. the ingest pool) is therefore
// bound to the CPUs of the GPU's node; pinned buffers it allocates afterwards are first-touched there.
// B200_NUMA_BIND=0 keeps the caller's affinity.
static void bind_to_gpu_numa_node(int device) {
  const char* env = getenv("B200_NUMA_BIND");
  if (env && env[0] == '0') return;
  char busid[64] = {0};
  if (cudaDeviceGetPCIBusId(busid, sizeof busid, device) != cudaSuccess) return;
  for (char* c = busid; *c; c++) *c = (char)tolower(*c);
  char path[256];
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", busid);
  int node = -1;
  if (FILE* f = fopen(path, "r")) {
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
  }
  if (node < 0) return;
  snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
  FILE* f = fopen(path, "r");
  if (!f) return;
  char list[4096] = {0};
  const size_t got = fread(list, 1, sizeof list - 1, f);
  fclose(f);
  if (!got) return;
  cpu_set_t want, cur, both;
  CPU_ZERO(&want);
  for (char* p = list; *p;) {
    char* end = nullptr;
    long a = strtol(p, &end, 10);
    if (end == p) break;
    long b = a;
    if (*end == '-') b = strtol(end + 1, &end, 10);
    for (long c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET((int)c, &want);
    p = (*end == ',') ? end + 1 : end;
    if (*end != ',' ) break;
  }
  if (sched_getaffinity(0, sizeof cur, &cur) != 0) return;
  CPU_AND(&both, &want, &cur);
  if (CPU_COUNT(&both) == 0) return;
  sched_setaffinity(0, sizeof both, &both);
}

int b200_engine_create(int device, uint64_t pool_bytes, int rank, int world, b200_engine** out) {
  return guard([&] {
    if (!out) throw EngineError(B200_ERR_INVALID, "null out pointer");
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev == 0)
      throw EngineError(B200_ERR_CUDA, std::string("no CUDA device available: the engine has no CPU path (") + cudaGetErrorString(ce) + ")");
    if (device < 0 || device >= ndev) throw EngineError(B200_ERR_INVALID, "bad device ordinal");
    CUDA_CHECK(cudaSetDevice(device));
    bind_to_gpu_numa_node(device);
    auto* e = new b200_engine();
    e->device = device;
    e->rank = rank;
    e->world = world;
    cudaDeviceProp prop;
    CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    e->sm_count = prop.multiProcessorCount;
    CUDA_CHECK(cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking));
    e->stream = e->own_stream;
    cudaMemPool_t pool;
    CUDA_CHECK(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t thr = pool_bytes ? pool_bytes : UINT64_MAX;
    CUDA_CHECK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    *out = e;
  });
}

void b200_engine_destroy(b200_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  e->tables.clear();
  e->shuffle.remove_all();
  cudaStreamSynchronize(e->stream);
  for (auto& sl : e->nslot) {
    if (sl.pinned) cudaFreeHost(sl.pinned);
    if (sl.dev) cudaFree(sl.dev);
    if (sl.done) cudaEventDestroy(sl.done);
  }
  release_window(e);
  e->regex.clear();
  if (e->comm && NcclApi::get().ok()) NcclApi::get().CommDestroy(e->comm);
  if (e->export_arena) cudaFreeHost(e->export_arena);
  // the calling thread's arena chunk is freed on the stream it was carved for: not after that stream is gone (at exit)
  if (arena_chunk() && arena_chunk()->stream == e->own_stream) arena_chunk().reset();
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  delete e;
}

int b200_engine_set_stream(b200_engine* e, void* cuda_stream) {
  return guard([&] {
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
    e->stream = cuda_stream ? (cudaStream_t)cuda_stream : e->own_stream;
  });
}
int b200_engine_synchronize(b200_engine* e) {
  return guard([&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
  });
}
uint64_t b200_engine_kernel_launches(b200_engine* e) { return e->launches; }
uint64_t b200_engine_counter(b200_engine* e, const char* name) {
  const std::string n = name ? name : "";
  if (n == "fused") return e->n_fused;
  if (n == "groupby_partition_first") return e->n_groupby_pf;
  if (n == "fused_static") return e->n_fused_static;
  if (n == "fused_exchanges") return e->fused_exchanges;
  if (n == "exchange_window_bytes") return e->win_bytes;
  if (n == "vm") return e->n_vm;
  if (n == "groupby") return e->n_groupby;
  if (n == "fastfilter") return e->n_fastfilter;
  if (n == "ingest_bytes_saved") return e->narrowed_bytes_saved;
  if (n == "nlj_pairs") return e->nlj_pairs;
  if (n == "window_sorts") return e->n_window_sorts;
  if (n == "host_syncs") return e->host_syncs;
  if (n == "regex_compiles") return e->regex.compiles;
  if (n == "string_arena_retries") return e->string_arena_retries;
  return 0;
}

int b200_engine_set_config(b200_engine* e, const char* key, const char* value) {
  return guard([&] {
    std::lock_guard<std::mutex> g(e->mu);
    e->config[key] = value;
    if (std::string(key) == "datafusion.execution.batch_size") e->batch_size = std::max<int64_t>(1, atoll(value));
    if (std::string(key) == "b200.ingest.chunk_rows") e->ingest_chunk_rows = std::max<int64_t>(1 << 16, atoll(value));
    if (std::string(key) == "b200.ingest.slots") e->ingest_slots = atoi(value);
    if (std::string(key) == "b200.exchange.window_bytes") e->win_config_bytes = (size_t)strtoull(value, nullptr, 10);  // read by b200_engine_comm_init
    if (std::string(key) == "b200.ingest.threads") e->pool.reset();  // re-created with the new size at the next ingest
    if (std::string(key) == "b200.agg.partition_first.bucket_slots") {
      const uint64_t v = strtoull(value, nullptr, 10);
      e->pf_bucket_slots = v ? std::max<uint64_t>(next_pow2(v), 64) : 0;
    }
    if (std::string(key) == "b200.agg.partition_first.min_rows") e->pf_min_rows = std::max<int64_t>(1, atoll(value));
    if (std::string(key) == "b200.agg.reset_hints") {
      e->agg_hint.clear();
      e->agg_groups.clear();
    }  // forget which aggregate strategy each plan shape needed
    if (std::string(key) == "b200.metrics.kernel_timing") e->kernel_timing = std::string(value) == "on" || std::string(value) == "1" || std::string(value) == "true";
  });
}

int b200_engine_register_batch(b200_engine* e, const char* table, int partition, struct ArrowArray* batch, struct ArrowSchema* schema) {
  return guard(e, [&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    DevBatchPtr b = import_batch(e, batch, schema);
    Exec x{e, nullptr, nullptr};
    build_column_images(x, *b);
    DevBatchPtr prev;
    {
      std::lock_guard<std::mutex> g(e->mu);
      auto& slot = e->tables[table][partition];
      prev = slot;
      if (!prev) slot = b;
    }
    if (prev) {  // append
      Schema s;
      for (auto& c : prev->cols) s.push_back(Field{c.name, c.type, true});
      DevBatchPtr cat = concat(x, {prev, b}, s);
      // registered tables keep the canonical Arrow layout (concat leaves strings as views) and their companion images
      for (auto& c : cat->cols) c = as_utf8(x, c);
      build_column_images(x, *cat);
      CUDA_CHECK(cudaStreamSynchronize(e->stream));
      std::lock_guard<std::mutex> g(e->mu);
      e->tables[table][partition] = cat;
    }
  });
}

int b200_engine_drop_table(b200_engine* e, const char* table) {
  return guard([&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    std::lock_guard<std::mutex> g(e->mu);
    e->tables.erase(table);
  });
}

int b200_engine_tpch_generate(b200_engine* e, const char* table, int64_t msf, int partition, int64_t row_begin, int64_t row_end, const char* columns_csv) {
  return guard(e, [&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    int t = table_id(table);
    if (t < 0) throw EngineError(B200_ERR_INVALID, std::string("unknown TPC-H table ") + table);
    std::vector<int> cols;
    if (columns_csv && *columns_csv) {
      std::string s(columns_csv);
      size_t p = 0;
      while (p <= s.size()) {
        size_t q = s.find(',', p);
        if (q == std::string::npos) q = s.size();
        std::string nm = s.substr(p, q - p);
        int found = -1;
        for (int c = 0; c < tpch::kNumCols[t]; c++)
          if (nm == tpch::kCols[t][c].name) found = c;
        if (found < 0) throw EngineError(B200_ERR_INVALID, "unknown column " + nm);
        cols.push_back(found);
        p = q + 1;
      }
    } else {
      for (int c = 0; c < tpch::kNumCols[t]; c++) cols.push_back(c);
    }
    const int64_t n = row_end - row_begin;
    if (n < 0) throw EngineError(B200_ERR_INVALID, "bad row range");
    cudaStream_t st = e->stream;
    auto b = std::make_shared<DevBatch>();
    b->n = n;
    for (int c : cols) {
      const tpch::ColDef& cd = tpch::kCols[t][c];
      DevColumn col;
      col.name = cd.name;
      col.n = n;
      col.nullable = false;
      switch (cd.kind) {
        case tpch::K_I64: col.type = DataType(TypeId::Int64); break;
        case tpch::K_I32: col.type = DataType(TypeId::Int32); break;
        case tpch::K_DEC: col.type = DataType::decimal(15, 2); break;
        case tpch::K_DATE: col.type = DataType(TypeId::Date32); break;
        default: col.type = DataType(TypeId::Utf8);
      }
      col.phys = phys_of(col.type);
      if (cd.kind == tpch::K_STR) {
        DevPtr lens = dev_alloc((size_t)(n + 1) * 4, st);
        DevPtr offs64 = dev_alloc((size_t)(n + 2) * 8, st);
        DevPtr scratch = dev_alloc((size_t)(n / 1024 + 4) * 8, st);
        launch_tpch_str_len(t, c, msf, row_begin, n, (uint32_t*)lens->ptr, st);
        launch_scan_u32_to_u64((const uint32_t*)lens->ptr, (uint64_t*)offs64->ptr, n, (uint64_t*)scratch->ptr, st);
        uint64_t total = Exec{e, nullptr, nullptr}.get<uint64_t>((const uint64_t*)offs64->ptr + n);
        if (total > 0x7FFFFFFFull) throw EngineError(B200_ERR_UNSUPPORTED, "generated string column exceeds 2 GiB; use more partitions");
        DevPtr offsets = dev_alloc((size_t)(n + 1) * 4 + 64, st);
        DevPtr chars = dev_alloc((size_t)total + 64, st);
        launch_tpch_str_fill(t, c, msf, row_begin, n, (const uint64_t*)offs64->ptr, (int32_t*)offsets->ptr, (uint8_t*)chars->ptr, st);
        col.data = (const uint8_t*)offsets->ptr;
        col.chars = (const uint8_t*)chars->ptr;
        col.chars_bytes = (int64_t)total;
        col.keep.push_back(offsets);
        col.keep.push_back(chars);
      } else {
        DevPtr d = dev_alloc((size_t)std::max<int64_t>(n, 1) * col.width() + 64, st);
        launch_tpch_fixed(t, c, cd.kind, msf, row_begin, n, d->ptr, st);
        col.data = (const uint8_t*)d->ptr;
        col.keep.push_back(d);
      }
      b->cols.push_back(col);
    }
    build_column_images(Exec{e, nullptr, nullptr}, *b);
    CUDA_CHECK(cudaStreamSynchronize(st));
    std::lock_guard<std::mutex> g(e->mu);
    e->tables[table][partition] = b;
  });
}

// Host-only view of what the device scan would be handed: schema, row counts and the page inventory of every column
// (JSON).  No CUDA call: used by the CPU tests to pin the Thrift footer / page-header reader against pyarrow's metadata.
int b200_parquet_describe(const char* path, char* out, uint64_t cap) {
  return guard([&] {
    if (!path || !out || cap < 2) throw EngineError(B200_ERR_INVALID, "bad argument");
    FILE* f = fopen(path, "rb");
    if (!f) throw EngineError(B200_ERR_NOT_FOUND, std::string("cannot open ") + path);
    fseek(f, 0, SEEK_END);
    const size_t fsize = (size_t)ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<uint8_t> buf(fsize);
    const size_t got = fread(buf.data(), 1, fsize, f);
    fclose(f);
    if (got != fsize) throw EngineError(B200_ERR_INVALID, "short read");
    pq::FileMeta fm;
    try {
      fm = pq::read_file_meta(buf.data(), fsize);
    } catch (const std::runtime_error& ex) {
      throw EngineError(B200_ERR_INVALID, ex.what());
    }
    std::string j = "{\"num_rows\":" + std::to_string(fm.num_rows) + ",\"row_groups\":" + std::to_string(fm.row_groups.size()) + ",\"columns\":[";
    for (size_t i = 1; i < fm.schema.size(); i++) {
      const pq::SchemaElement& se = fm.schema[i];
      int64_t data_pages = 0, dict_pages = 0, values = 0, dict_encoded = 0, codec = 0;  // codec: the last row group's
      std::set<int32_t> encodings;  // value encodings named by the column's data and dictionary page headers
      std::set<int32_t> codecs;     // compression codecs of all its chunks
      for (auto& rg : fm.row_groups) {
        if (i - 1 >= rg.columns.size()) continue;
        const pq::ColumnChunkMeta& cm = rg.columns[i - 1];
        codec = cm.codec;
        codecs.insert(cm.codec);
        int64_t start = cm.data_page_offset;
        if (cm.dictionary_page_offset > 0 && cm.dictionary_page_offset < start) start = cm.dictionary_page_offset;
        const uint8_t* hp = buf.data() + start;
        const uint8_t* hend = hp + cm.total_compressed;
        int64_t seen = 0;
        while (hp < hend && seen < cm.num_values) {
          pq::PageHeader h = pq::read_page_header(hp, hend);
          if (h.type == pq::P_DICTIONARY) {
            dict_pages++;
            encodings.insert(h.encoding);
          } else if (h.type == pq::P_DATA || h.type == pq::P_DATA_V2) {
            data_pages++;
            encodings.insert(h.encoding);
            seen += h.num_values;
            values += h.num_values;
            if (h.encoding == pq::E_PLAIN_DICTIONARY || h.encoding == pq::E_RLE_DICTIONARY) dict_encoded++;
          }
          hp += h.header_bytes + (size_t)h.compressed_size;
        }
      }
      if (i > 1) j += ",";
      j += "{\"name\":\"" + se.name + "\",\"physical\":" + std::to_string(se.type) + ",\"type_length\":" + std::to_string(se.type_length) + ",\"optional\":" +
           (se.repetition == 1 ? "true" : "false") + ",\"logical\":" + std::to_string(se.logical) + ",\"converted\":" + std::to_string(se.converted) +
           ",\"precision\":" + std::to_string(se.precision) + ",\"scale\":" + std::to_string(se.scale) + ",\"codec\":" + std::to_string(codec) +
           ",\"values\":" + std::to_string(values) + ",\"data_pages\":" + std::to_string(data_pages) + ",\"dict_pages\":" + std::to_string(dict_pages) +
           ",\"dict_encoded_pages\":" + std::to_string(dict_encoded) + ",\"encodings\":[";
      bool first = true;
      for (int32_t e : encodings) {
        j += (first ? "" : ",") + std::to_string(e);
        first = false;
      }
      j += "],\"codecs\":[";
      first = true;
      for (int32_t k : codecs) {
        j += (first ? "" : ",") + std::to_string(k);
        first = false;
      }
      j += "]}";
    }
    j += "]}";
    if (j.size() + 1 > cap) throw EngineError(B200_ERR_INVALID, "description buffer too small");
    memcpy(out, j.c_str(), j.size() + 1);
  });
}

int b200_engine_register_parquet(b200_engine* e, const char* table, int partition, const char* path, const char* columns_csv) {
  return guard(e, [&] {
    if (!e || !table || !path) throw EngineError(B200_ERR_INVALID, "null argument");
    CUDA_CHECK(cudaSetDevice(e->device));
    std::vector<std::string> cols;
    if (columns_csv && *columns_csv) {
      std::string sct(columns_csv);
      size_t p = 0;
      while (p <= sct.size()) {
        size_t q = sct.find(',', p);
        if (q == std::string::npos) q = sct.size();
        if (q > p) cols.push_back(sct.substr(p, q - p));
        p = q + 1;
      }
    }
    Exec x{e, nullptr, nullptr};
    DevBatchPtr b;
    try {
      b = scan_parquet(x, path, cols);
    } catch (...) {
      cudaStreamSynchronize(e->stream);
      Exec::abandon();
      throw;
    }
    std::lock_guard<std::mutex> g(e->mu);
    e->tables[table][partition] = b;
  });
}

int b200_engine_register_csv(b200_engine* e, const char* table, int partition, const char* scan_json) {
  return guard(e, [&] {
    if (!e || !table || !scan_json) throw EngineError(B200_ERR_INVALID, "null argument");
    const CsvScanSpec spec = parse_csv_scan(scan_json);
    CUDA_CHECK(cudaSetDevice(e->device));
    Exec x{e, nullptr, nullptr};
    DevBatchPtr b;
    try {
      b = scan_csv(x, spec);
    } catch (...) {
      cudaStreamSynchronize(e->stream);
      Exec::abandon();
      throw;
    }
    std::lock_guard<std::mutex> g(e->mu);
    e->tables[table][partition] = b;
  });
}

int64_t b200_tpch_table_rows(const char* table, int64_t msf) {
  const int t = table ? table_id(table) : -1;
  return t < 0 ? -1 : tpch::table_rows(t, msf);
}

int b200_engine_export_table(b200_engine* e, const char* table, int partition, struct ArrowArray* out, struct ArrowSchema* out_schema) {
  return guard(e, [&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    DevBatchPtr b;
    {
      std::lock_guard<std::mutex> g(e->mu);
      auto it = e->tables.find(table);
      if (it == e->tables.end() || !it->second.count(partition)) throw EngineError(B200_ERR_NOT_FOUND, "no such table partition");
      b = it->second[partition];
    }
    Exec x{e, nullptr, nullptr};
    export_batch(x, *b, 0, b->n, out, out_schema);
  });
}

int b200_stage_prepare(b200_engine* e, const char* job_id, int64_t stage_id, const char* plan_json, uint64_t plan_len, b200_stage** out) {
  ScopeTimer tm("stage_prepare");
  return guard([&] {
    if (!e || !plan_json || !out) throw EngineError(B200_ERR_INVALID, "null argument");
    const size_t len = plan_len ? (size_t)plan_len : strlen(plan_json);
    // strategy hints (which aggregate sink / table size worked) are remembered per plan SHAPE: the job id is taken out
    // of the hashed text so that the next job that runs the same stage plan starts from what the last one learnt
    std::string shape(plan_json, len);
    const std::string tag = "\"job_id\":\"";
    size_t at = shape.find(tag);
    if (at != std::string::npos) {
      size_t end = shape.find('"', at + tag.size());
      if (end != std::string::npos) shape.erase(at + tag.size(), end - at - tag.size());
    }
    // the same shape also shares the parsed plan: parsing and typing the JSON is most of the host time of preparing a
    // small stage, and a repeated query prepares the same few plans for every job.  Keyed by the stage id as well (the
    // writer stores under it).  Only when the caller names the job: otherwise the job id comes from the text itself.
    const std::string cache_key = std::to_string(stage_id) + ":" + shape;
    std::shared_ptr<const PlanNode> plan;
    if (job_id) {
      std::lock_guard<std::mutex> g(e->mu);
      auto it = e->plan_cache.find(cache_key);
      if (it != e->plan_cache.end()) plan = it->second;
    }
    if (!plan) {
      Json j = parse_json(plan_json, len);
      PlanPtr parsed = parse_plan(j);
      if (parsed->op != PlanNode::ShuffleWriter)
        throw EngineError(B200_ERR_INVALID, "Plan passed to new_query_stage_exec is not a ShuffleWriterExec");  // execution_engine.rs:164-167
      parsed->stage_id = stage_id;
      plan = std::shared_ptr<const PlanNode>(std::move(parsed));
      if (job_id) {
        static const size_t PLAN_CACHE_MAX = 256;  // distinct stage plans kept; a workload with more starts over
        std::lock_guard<std::mutex> g(e->mu);
        if (e->plan_cache.size() >= PLAN_CACHE_MAX) e->plan_cache.clear();
        e->plan_cache.emplace(cache_key, plan);
      }
    }
    auto* s = new b200_stage();
    s->eng = e;
    s->job_id = job_id ? job_id : plan->job_id;
    s->stage_id = stage_id;
    s->fingerprint = std::to_string(stage_id) + ":" + std::to_string(mix64(hash_bytes((const uint8_t*)shape.data(), (uint32_t)shape.size())));
    collect_nodes(*plan, s);
    s->plan = std::move(plan);
    *out = s;
  });
}

// The task's plan as the scheduler ships it (TaskDefinition.plan: protobuf datafusion.PhysicalPlanNode): decoded to the IR
// by csrc/common/plan_proto.hpp, then prepared like any other stage plan.  Pure host code, no CUDA call.
int b200_plan_proto_to_json(const void* plan_bytes, uint64_t n_bytes, const char* job_id, char** out_json) {
  return guard([&] {
    if (!plan_bytes || !out_json) throw EngineError(B200_ERR_INVALID, "null argument");
    std::string js;
    try {
      js = pbp::plan_proto_to_json(plan_bytes, (size_t)n_bytes, job_id ? std::string(job_id) : std::string());
    } catch (const pbp::Unsupported& u) {
      throw EngineError(B200_ERR_UNSUPPORTED, u.what());
    } catch (const std::runtime_error& r) {
      throw EngineError(B200_ERR_INVALID, r.what());
    }
    char* m = (char*)malloc(js.size() + 1);
    if (!m) throw EngineError(B200_ERR_OOM, "plan JSON");
    memcpy(m, js.c_str(), js.size() + 1);
    *out_json = m;
  });
}

void b200_string_free(char* s) { free(s); }

// EXPLAIN-style diagnostic: the typed plan the engine derived from a stage-plan IR text (column references resolved to
// indices, expression / aggregate result types, every node's output schema), as canonical JSON.  Host only.
int b200_plan_typed_json(const char* plan_json, uint64_t plan_len, char** out_json) {
  return guard([&] {
    if (!plan_json || !out_json) throw EngineError(B200_ERR_INVALID, "null argument");
    Json j = parse_json(plan_json, plan_len ? (size_t)plan_len : strlen(plan_json));
    PlanPtr plan = parse_plan(j);
    const std::string js = dump_plan(*plan);
    char* m = (char*)malloc(js.size() + 1);
    if (!m) throw EngineError(B200_ERR_OOM, "plan JSON");
    memcpy(m, js.c_str(), js.size() + 1);
    *out_json = m;
  });
}

int b200_stage_prepare_proto(b200_engine* e, const char* job_id, int64_t stage_id, const void* plan_bytes, uint64_t n_bytes, b200_stage** out) {
  char* js = nullptr;
  int rc = b200_plan_proto_to_json(plan_bytes, n_bytes, job_id, &js);
  if (rc != 0) return rc;
  rc = b200_stage_prepare(e, job_id, stage_id, js, 0, out);
  free(js);
  return rc;
}

// A whole task as the executor received it (TaskDefinition / MultiTaskDefinition bytes, ballista.proto:518-542): the session
// properties are applied like b200_engine_set_config (TaskDefinition.props -> SessionConfig, executor_server.rs), the embedded
// plan is prepared, and the task identities come back as JSON ({"job_id","stage_id","tasks":[{"task_id","partition_id",..}],..}):
// the caller then runs b200_stage_execute(stage, partition_id) per task.  e == NULL: decode only (*out_stage untouched).
int b200_stage_prepare_task(b200_engine* e, const void* task_bytes, uint64_t n_bytes, int multi, b200_stage** out_stage, char** out_task_json) {
  std::string job;
  int64_t stage_id = 0;
  pbp::Slice plan;
  int rc = guard([&] {
    if (!task_bytes || !out_task_json || (e && !out_stage)) throw EngineError(B200_ERR_INVALID, "null argument");
    pbp::TaskInfo t;
    try {
      t = pbp::decode_task_definition(task_bytes, (size_t)n_bytes, multi != 0);
    } catch (const std::runtime_error& r) {
      throw EngineError(B200_ERR_INVALID, r.what());
    }
    const std::string js = pbp::task_info_json(t);
    char* m = (char*)malloc(js.size() + 1);
    if (!m) throw EngineError(B200_ERR_OOM, "task JSON");
    memcpy(m, js.c_str(), js.size() + 1);
    *out_task_json = m;
    job = t.job_id;
    stage_id = (int64_t)t.stage_id;
    plan = t.plan;
    if (e)
      for (auto& kv : t.props) b200_engine_set_config(e, kv.first.c_str(), kv.second.c_str());
  });
  if (rc != 0 || !e) return rc;
  rc = b200_stage_prepare_proto(e, job.c_str(), stage_id, plan.p, plan.n, out_stage);
  if (rc != 0) {
    free(*out_task_json);
    *out_task_json = nullptr;
  }
  return rc;
}

// TaskStatus (ballista.proto:494-509) for a finished task; rules of executor/src/lib.rs:101-152 and core/src/error.rs:205-256.
int b200_task_status_encode(const char* job_id, const char* executor_id, const b200_task_result* r, const b200_shuffle_write_partition* parts, int n_parts,
                            const b200_operator_metrics* metrics, int n_metrics, char** out_bytes, uint64_t* out_len) {
  return guard([&] {
    if (!job_id || !r || !out_bytes || !out_len || (n_parts > 0 && !parts) || (n_metrics > 0 && !metrics)) throw EngineError(B200_ERR_INVALID, "null argument");
    pbp::Writer w;
    w.u64(1, r->task_id);
    w.str(2, job_id);
    w.u64(3, r->stage_id);
    w.u64(4, r->stage_attempt_num);
    w.u64(5, r->partition_id);
    w.u64(6, r->launch_time);
    w.u64(7, r->start_exec_time);
    w.u64(8, r->end_exec_time);
    if (r->status == B200_OK) {
      pbp::Writer ok;  // SuccessfulTask { executor_id = 1, partitions = 2 } (:453-458)
      ok.str(1, executor_id ? executor_id : "");
      for (int i = 0; i < n_parts; i++) {
        pbp::Writer p;  // ShuffleWritePartition { partition_id = 1, num_batches = 3, num_rows = 4, num_bytes = 5, optional file_id = 6, is_sort_shuffle = 7 } (:481-492)
        p.u64(1, parts[i].partition_id);
        p.u64(3, parts[i].num_batches);
        p.u64(4, parts[i].num_rows);
        p.u64(5, parts[i].num_bytes);
        if (parts[i].file_id >= 0) p.u64_always(6, (uint64_t)parts[i].file_id);
        p.boolean(7, parts[i].is_sort_shuffle != 0);
        ok.msg(2, p);
      }
      w.msg(11, ok);
    } else {
      pbp::Writer f;  // FailedTask { error = 1, retryable = 2, count_to_failures = 3, failed_reason 4..9 } (:437-451)
      const std::string msg = r->error_message ? r->error_message : "";
      if (r->status == B200_ERR_NOT_FOUND) {
        f.str(1, msg);
        pbp::Writer fe;  // FetchPartitionError { executor_id = 1, map_stage_id = 2, map_partition_id = 3 } (:463-467)
        fe.str(1, r->fetch_executor_id ? r->fetch_executor_id : "");
        fe.u64(2, r->fetch_map_stage_id);
        fe.u64(3, r->fetch_map_partition_id);
        f.msg(5, fe);
      } else if (r->status == B200_ERR_CANCELLED) {
        f.str(1, msg.empty() ? std::string("Task killed") : msg);
        f.msg(9, pbp::Writer());  // TaskKilled {}
      } else {
        f.str(1, "Task failed due to runtime execution error: " + msg);
        f.msg(4, pbp::Writer());  // ExecutionError {}
      }
      w.msg(10, f);
    }
    for (int i = 0; i < n_metrics; i++) {
      pbp::Writer set;  // OperatorMetricsSet { metrics = 1 } (:286-288); OperatorMetric oneof (:318-336)
      auto one = [&](uint32_t field, uint64_t v) {
        pbp::Writer m;
        m.u64_always(field, v);
        set.msg(1, m);
      };
      auto named = [&](const char* name, uint64_t v) {
        pbp::Writer nc;  // NamedCount { name = 1, value = 2 } (:291-294)
        nc.str(1, name);
        nc.u64(2, v);
        pbp::Writer m;
        m.msg(6, nc);
        set.msg(1, m);
      };
      one(1, metrics[i].output_rows);
      one(2, metrics[i].elapsed_compute_ns);
      one(12, metrics[i].bytes_written);
      named("input_rows", metrics[i].input_rows);
      named("bytes_read", metrics[i].bytes_read);
      named("kernel_launches", metrics[i].kernel_launches);
      w.msg(12, set);
    }
    char* m = (char*)malloc(w.out.size() + 1);
    if (!m) throw EngineError(B200_ERR_OOM, "task status");
    memcpy(m, w.out.data(), w.out.size());
    m[w.out.size()] = 0;
    *out_bytes = m;
    *out_len = w.out.size();
  });
}

int b200_stage_execute(b200_stage* s, int input_partition, const volatile int32_t* cancel_flag, b200_shuffle_write_partition* out, int cap, int* n_out) {
  ScopeTimer tm("stage_execute");
  return guard(s ? s->eng : nullptr, [&] {
    if (!s || !n_out) throw EngineError(B200_ERR_INVALID, "null argument");
    CUDA_CHECK(cudaSetDevice(s->eng->device));
    Exec x{s->eng, s, cancel_flag};
    Runner r{x, s->job_id};
    std::vector<b200_shuffle_write_partition> res;
    try {
      res = r.execute_stage(*s->plan, input_partition);
    } catch (...) {
      host_wait(s->eng, s->eng->stream);
      Exec::abandon();
      // a cancelled or failed task leaves nothing behind (Executor::cancel_task drops the future together with
      // its partial outputs, executor.rs:217-237): remove whatever this task already stored
      s->eng->shuffle.remove_task(s->job_id, s->stage_id, input_partition, s->eng->rank);
      throw;
    }
    if ((int)res.size() > cap) throw EngineError(B200_ERR_INVALID, "output array too small");
    for (size_t i = 0; i < res.size(); i++) out[i] = res[i];
    *n_out = (int)res.size();
  });
}

int b200_stage_execute_exchange(b200_stage* s, int input_partition, const volatile int32_t* cancel_flag, b200_shuffle_write_partition* out, int cap,
                                int* n_out, b200_exchange_stats* stats) {
  ScopeTimer tm("stage_execute_exchange");
  return guard(s ? s->eng : nullptr, [&] {
    if (!s || !n_out) throw EngineError(B200_ERR_INVALID, "null argument");
    b200_engine* e = s->eng;
    if (s->plan->op != PlanNode::ShuffleWriter || s->plan->n_out_partitions < 1)
      throw EngineError(B200_ERR_INVALID, "b200_stage_execute_exchange needs a hash-partitioning ShuffleWriterExec");
    CUDA_CHECK(cudaSetDevice(e->device));
    Exec x{e, s, cancel_flag};
    Runner r{x, s->job_id};
    Runner::FusedExchange fx;
    std::vector<b200_shuffle_write_partition> res;
    uint64_t sent = 0, recvd = 0;
    try {
      res = r.execute_stage(*s->plan, input_partition, &fx);
      if (fx.done) {
        sent = fx.sent;
        recvd = fx.recvd;
      } else if (e->world > 1) {
        // two-step path (strings in the payload, no window, or a window too small for this exchange)
        Exchange ex{x, e, s->job_id, s->stage_id, (int)s->plan->n_out_partitions, EXCH_HASH, 0, s->plan->schema, s->plan->schema.size()};
        ex.run(&sent, &recvd);
      }
    } catch (...) {
      host_wait(e, e->stream);
      Exec::abandon();
      throw;
    }
    e->exch_sent_bytes += sent;
    e->exch_recv_bytes += recvd;
    if (stats) {
      stats->sent_bytes = sent;
      stats->recv_bytes = recvd;
    }
    if ((int)res.size() > cap) throw EngineError(B200_ERR_INVALID, "output array too small");
    for (size_t i = 0; i < res.size(); i++) out[i] = res[i];
    *n_out = (int)res.size();
  });
}

int b200_stage_metrics(b200_stage* s, b200_operator_metrics* out, int cap, int* n_out) {
  return guard([&] {
    int n = (int)std::min<size_t>(s->metrics.size(), (size_t)cap);
    for (int i = 0; i < n; i++) {
      memset(&out[i], 0, sizeof out[i]);
      snprintf(out[i].name, sizeof out[i].name, "%s", s->metrics[(size_t)i].name.c_str());
      out[i].output_rows = s->metrics[(size_t)i].output_rows;
      out[i].input_rows = s->metrics[(size_t)i].input_rows;
      out[i].elapsed_compute_ns = s->metrics[(size_t)i].elapsed_ns;
      out[i].bytes_read = s->metrics[(size_t)i].bytes_read;
      out[i].bytes_written = s->metrics[(size_t)i].bytes_written;
      out[i].kernel_launches = s->metrics[(size_t)i].launches;
    }
    *n_out = n;
  });
}

void b200_stage_release(b200_stage* s) { delete s; }

int b200_partition_export(b200_engine* e, const char* job_id, int64_t stage_id, int out_partition, struct ArrowArray* out, struct ArrowSchema* out_schema) {
  ScopeTimer tm("partition_export");
  return guard(e, [&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    const std::vector<Piece> pieces = e->shuffle.pieces(ShuffleKey{job_id, stage_id, out_partition});
    if (pieces.empty()) throw EngineError(B200_ERR_NOT_FOUND, "no such shuffle partition");  // -> FetchFailed
    Exec x{e, nullptr, nullptr};
    if (pieces.size() == 1) {
      export_batch(x, *pieces[0].batch, pieces[0].r0, pieces[0].r1, out, out_schema);
      return;
    }
    Schema s;
    for (auto& c : pieces[0].batch->cols) s.push_back(Field{c.name, c.type, true});
    DevBatchPtr cat = concat_slices(x, pieces, s);
    export_batch(x, *cat, 0, cat->n, out, out_schema);
  });
}

int64_t b200_partition_rows(b200_engine* e, const char* job_id, int64_t stage_id, int out_partition) {
  return e->shuffle.rows(ShuffleKey{job_id, stage_id, out_partition});
}

int b200_remove_job_data(b200_engine* e, const char* job_id) {
  return guard([&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    std::lock_guard<std::mutex> g(e->mu);
    // partitions that arrived through the fused shuffle live in the exchange window: it is recycled as a whole once no
    // stored partition can refer to it any more (peers write into it only inside a collective this executor takes part in)
    if (e->shuffle.remove_job(job_id)) e->win_used = 0;
  });
}

int b200_remove_stage_data(b200_engine* e, const char* job_id, int64_t stage_id) {
  return guard([&] {
    CUDA_CHECK(cudaSetDevice(e->device));
    e->shuffle.remove_stage(job_id, stage_id);
  });
}

int b200_engine_kernel_stats(b200_engine* e, b200_kernel_stat* out, int cap, int* n_out, int reset) {
  return guard([&] {
    if (!e || !n_out) throw EngineError(B200_ERR_INVALID, "null argument");
    CUDA_CHECK(cudaSetDevice(e->device));
    CUDA_CHECK(cudaStreamSynchronize(e->stream));
    std::lock_guard<std::mutex> g(e->mu);
    for (auto& ks : e->ksamples) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, ks.e0, ks.e1) == cudaSuccess) {
        auto& st = e->kstats[ks.name];
        st.ms += ms;
        st.launches++;
        st.bytes += ks.bytes;
      }
      cudaEventDestroy(ks.e0);
      cudaEventDestroy(ks.e1);
    }
    e->ksamples.clear();
    int k = 0;
    for (auto& kv : e->kstats) {
      if (k >= cap) break;
      memset(&out[k], 0, sizeof out[k]);
      snprintf(out[k].name, sizeof out[k].name, "%s", kv.first.c_str());
      out[k].elapsed_ns = (uint64_t)(kv.second.ms * 1e6);
      out[k].launches = kv.second.launches;
      out[k].algorithmic_bytes = kv.second.bytes;
      k++;
    }
    *n_out = k;
    if (reset) e->kstats.clear();
  });
}


int b200_comm_unique_id(void* out, uint64_t cap) {
  return guard([&] {
    if (!out || cap < sizeof(ncclUniqueId)) throw EngineError(B200_ERR_INVALID, "b200_comm_unique_id needs a 128-byte buffer");
    NcclApi& N = NcclApi::get();
    if (!N.ok()) throw EngineError(B200_ERR_CUDA, "libnccl not available: " + N.error);
    ncclUniqueId id;
    NCCL_CHECK(N.GetUniqueId(&id));
    memcpy(out, &id, sizeof id);
  });
}

int b200_engine_comm_init(b200_engine* e, const void* nccl_id, uint64_t id_bytes) {
  return guard([&] {
    if (!e || !nccl_id || id_bytes < sizeof(ncclUniqueId)) throw EngineError(B200_ERR_INVALID, "b200_engine_comm_init: bad arguments");
    if (e->world <= 1) return;  // a single executor exchanges nothing
    NcclApi& N = NcclApi::get();
    if (!N.ok()) throw EngineError(B200_ERR_CUDA, "libnccl not available: " + N.error);
    CUDA_CHECK(cudaSetDevice(e->device));
    std::lock_guard<std::mutex> g(e->comm_mu);
    if (e->comm) {
      N.CommDestroy(e->comm);
      e->comm = nullptr;
    }
    ncclUniqueId id;
    memcpy(&id, nccl_id, sizeof id);
    NCCL_CHECK(N.CommInitRank(&e->comm, e->world, id, e->rank));
    release_window(e);
    if (e->win_config_bytes) setup_window(e);
  });
}

int b200_exchange_stage(b200_engine* e, const char* job_id, int64_t stage_id, int n_out_partitions, int mode, int root, const char* schema_json,
                        b200_exchange_stats* stats) {
  return guard(e, [&] {
    if (!e || !job_id || !schema_json) throw EngineError(B200_ERR_INVALID, "null argument");
    if (mode < 0 || mode > 2 || n_out_partitions < 0 || root < 0 || root >= std::max(e->world, 1)) throw EngineError(B200_ERR_INVALID, "b200_exchange_stage: bad mode / root");
    CUDA_CHECK(cudaSetDevice(e->device));
    Json j = parse_json(schema_json, strlen(schema_json));
    Exec x{e, nullptr, nullptr};
    Exchange ex{x, e, job_id, stage_id, n_out_partitions, mode, root, parse_schema(j), 0};
    ex.ncols = ex.schema.size();
    uint64_t sent = 0, recvd = 0;
    try {
      ex.run(&sent, &recvd);
    } catch (...) {
      host_wait(e, e->stream);
      Exec::abandon();
      throw;
    }
    e->exch_sent_bytes += sent;
    e->exch_recv_bytes += recvd;
    if (stats) {
      stats->sent_bytes = sent;
      stats->recv_bytes = recvd;
    }
  });
}

// ---- the reference's shuffle file format: Arrow IPC streams with LZ4_FRAME bodies (csrc/host/arrow_ipc.hpp) ----------------
static std::vector<HostCol> host_cols_from_arrow(ArrowArray* arr, ArrowSchema* sch, int64_t* n_rows) {
  std::vector<ImportedCol> ics = import_record_batch(arr, sch, n_rows);
  const int64_t n = *n_rows;
  std::vector<HostCol> out;
  for (auto& ic : ics) {
    HostCol h;
    h.name = ic.name;
    h.type = ic.type;
    h.nullable = ic.nullable;
    h.n = n;
    if (ic.large_offsets) throw EngineError(B200_ERR_UNSUPPORTED, "LargeUtf8 columns are not supported");
    auto bit = [](const uint8_t* bm, int64_t i) { return (bm[i >> 3] >> (i & 7)) & 1; };
    if (ic.null_count > 0 && ic.validity) {
      h.validity.assign((size_t)((n + 7) / 8), 0);
      for (int64_t i = 0; i < n; i++)
        if (bit(ic.validity, i + ic.offset)) h.validity[(size_t)(i >> 3)] |= (uint8_t)(1u << (i & 7));
        else h.null_count++;
      if (h.null_count == 0) h.validity.clear();
    }
    if (ic.type.id == TypeId::Null) {
      h.null_count = n;
    } else if (ic.type.id == TypeId::Bool) {
      h.data.assign((size_t)((n + 7) / 8), 0);
      for (int64_t i = 0; i < n; i++)
        if (bit(ic.data, i + ic.offset)) h.data[(size_t)(i >> 3)] |= (uint8_t)(1u << (i & 7));
    } else if (ic.type.id == TypeId::Utf8) {
      const int32_t* off = (const int32_t*)ic.data + ic.offset;
      h.data.resize((size_t)(n + 1) * 4);
      int32_t* po = (int32_t*)h.data.data();
      for (int64_t i = 0; i <= n; i++) po[i] = off[i] - off[0];
      if (n) h.extra.assign(ic.extra + off[0], ic.extra + off[n]);
    } else {
      const size_t w = (size_t)ic.type.width();
      h.data.assign(ic.data + (size_t)ic.offset * w, ic.data + (size_t)(ic.offset + n) * w);
    }
    out.push_back(std::move(h));
  }
  return out;
}

static std::vector<uint8_t> read_whole_file(const std::string& path, uint64_t offset, uint64_t length) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) throw EngineError(B200_ERR_NOT_FOUND, "cannot open " + path);  // -> FetchFailed
  fseek(f, 0, SEEK_END);
  const uint64_t fsize = (uint64_t)ftell(f);
  if (length == 0 && offset == 0) length = fsize;
  if (offset + length > fsize) {
    fclose(f);
    throw EngineError(B200_ERR_INVALID, "byte range outside " + path);
  }
  fseek(f, (long)offset, SEEK_SET);
  std::vector<uint8_t> buf((size_t)length);
  const size_t got = length ? fread(buf.data(), 1, (size_t)length, f) : 0;
  fclose(f);
  if (got != length) throw EngineError(B200_ERR_INVALID, "short read on " + path);
  return buf;
}

static void write_whole_file(const std::string& path, const std::vector<uint8_t>& bytes) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) throw EngineError(B200_ERR_INVALID, "cannot create " + path);
  const size_t put = bytes.empty() ? 0 : fwrite(bytes.data(), 1, bytes.size(), f);
  fclose(f);
  if (put != bytes.size()) throw EngineError(B200_ERR_INVALID, "short write on " + path);
}

static void make_dirs(const std::string& path) {
  std::string cur;
  for (size_t i = 0; i <= path.size(); i++) {
    if (i == path.size() || path[i] == '/') {
      if (!cur.empty() && cur != "/") mkdir(cur.c_str(), 0777);
    }
    if (i < path.size()) cur.push_back(path[i]);
  }
}

int b200_ipc_encode(struct ArrowArray* batch, struct ArrowSchema* schema, int compress, int64_t max_rows_per_message, uint8_t** out, uint64_t* out_len) {
  return guard([&] {
    if (!batch || !schema || !out || !out_len) throw EngineError(B200_ERR_INVALID, "null argument");
    int64_t n = 0;
    std::vector<HostCol> cols;
    try {
      cols = host_cols_from_arrow(batch, schema, &n);
    } catch (const std::runtime_error& ex) {
      throw EngineError(B200_ERR_INVALID, ex.what());
    }
    if (batch->release) batch->release(batch);
    if (schema->release) schema->release(schema);
    std::vector<uint8_t> bytes;
    ipc::write_stream(bytes, cols, n, compress != 0, max_rows_per_message);
    uint8_t* p = (uint8_t*)malloc(bytes.size() ? bytes.size() : 1);
    if (!p) throw EngineError(B200_ERR_OOM, "host out of memory");
    memcpy(p, bytes.data(), bytes.size());
    *out = p;
    *out_len = bytes.size();
  });
}

void b200_ipc_free(uint8_t* p) { free(p); }

int b200_ipc_decode(const uint8_t* buf, uint64_t len, struct ArrowArray* out, struct ArrowSchema* out_schema) {
  return guard([&] {
    if (!buf || !out || !out_schema) throw EngineError(B200_ERR_INVALID, "null argument");
    std::vector<HostCol> cols;
    int64_t n = 0;
    try {
      n = ipc::read_streams(buf, (size_t)len, cols);
    } catch (const std::runtime_error& ex) {
      throw EngineError(B200_ERR_INVALID, ex.what());
    }
    export_record_batch(std::move(cols), n, out, out_schema);
  });
}

// Every piece this executor's map tasks produced for (job, stage), as files in the reference's layout below work_dir
// (create_shuffle_path, execution_plans/mod.rs:66-99): what makes HBM-resident shuffle output survive the executor and
// readable by the reference's own readers (a CPU executor's ShuffleReaderExec, the Flight service).
int b200_shuffle_write_files(b200_engine* e, const char* job_id, int64_t stage_id, const char* work_dir, int n_out_partitions, int sort_layout,
                             uint64_t* files_written, uint64_t* bytes_written) {
  return guard(e, [&] {
    if (!e || !job_id || !work_dir) throw EngineError(B200_ERR_INVALID, "null argument");
    CUDA_CHECK(cudaSetDevice(e->device));
    Exec x{e, nullptr, nullptr};
    std::vector<StoredPiece> items = e->shuffle.of_rank(job_id, stage_id, e->rank);
    const std::string base = std::string(work_dir) + "/" + job_id + "/" + std::to_string(stage_id);
    uint64_t nfiles = 0, nbytes = 0;
    const int64_t bs = e->batch_size;
    if (!sort_layout) {
      for (auto& it : items) {
        std::vector<HostCol> cols = download_batch(x, *it.piece.batch, it.piece.r0, it.piece.r1);
        std::vector<uint8_t> bytes;
        ipc::write_stream(bytes, cols, it.piece.r1 - it.piece.r0, true, bs);
        const std::string dir = base + "/" + std::to_string(it.part);
        make_dirs(dir);
        const std::string path = dir + (it.piece.file_id >= 0 ? "/data-" + std::to_string(it.piece.file_id) + ".arrow" : "/data.arrow");
        write_whole_file(path, bytes);
        nfiles++;
        nbytes += bytes.size();
      }
    } else {
      // one consolidated file per map task: [schema-only stream][partition 0 streams][partition 1 streams]... + index
      std::map<int64_t, std::vector<StoredPiece*>> by_task;
      for (auto& it : items) by_task[it.piece.file_id].push_back(&it);
      for (auto& kv : by_task) {
        if (kv.first < 0) throw EngineError(B200_ERR_INVALID, "sort-shuffle layout needs a file id (un-partitioned stage output)");
        std::vector<uint8_t> bytes;
        std::vector<int64_t> offsets((size_t)n_out_partitions + 1, 0);
        bool header = false;
        std::vector<std::vector<HostCol>> parts((size_t)n_out_partitions);
        std::vector<int64_t> rows((size_t)n_out_partitions, 0);
        for (StoredPiece* it : kv.second) {
          if (it->part >= n_out_partitions) throw EngineError(B200_ERR_INVALID, "stored partition id beyond n_out_partitions");
          parts[(size_t)it->part] = download_batch(x, *it->piece.batch, it->piece.r0, it->piece.r1);
          rows[(size_t)it->part] = it->piece.r1 - it->piece.r0;
          if (!header) {
            ipc::write_schema(bytes, parts[(size_t)it->part]);
            ipc::write_eos(bytes);
            header = true;
          }
        }
        for (int p = 0; p < n_out_partitions; p++) {
          offsets[(size_t)p] = (int64_t)bytes.size();
          if (rows[(size_t)p] > 0) ipc::write_stream(bytes, parts[(size_t)p], rows[(size_t)p], true, bs);
        }
        offsets[(size_t)n_out_partitions] = (int64_t)bytes.size();
        const std::string dir = base + "/" + std::to_string(kv.first);
        make_dirs(dir);
        write_whole_file(dir + "/data.arrow", bytes);
        std::vector<uint8_t> idx((size_t)(n_out_partitions + 1) * 8);
        memcpy(idx.data(), offsets.data(), idx.size());
        write_whole_file(dir + "/data.arrow.index", idx);
        nfiles += 2;
        nbytes += bytes.size() + idx.size();
      }
    }
    if (files_written) *files_written = nfiles;
    if (bytes_written) *bytes_written = nbytes;
  });
}

// One reference-format shuffle file (or a byte range of it: a partition of a sort-shuffle data file) into the shuffle
// store as a piece of (job, stage, out_partition) -- the local-read path of ShuffleReaderExec (shuffle_reader.rs:698-771,
// sort_shuffle/reader.rs:51-84) with the decoded batches landing in HBM.  byte_length 0 with byte_offset 0 = whole file;
// use_index != 0: `path` is a sort-shuffle data file, the range of `out_partition` is taken from `path` + ".index".
int b200_shuffle_read_file(b200_engine* e, const char* job_id, int64_t stage_id, int out_partition, int64_t file_id, const char* path, uint64_t byte_offset,
                           uint64_t byte_length, int use_index) {
  return guard(e, [&] {
    if (!e || !job_id || !path) throw EngineError(B200_ERR_INVALID, "null argument");
    CUDA_CHECK(cudaSetDevice(e->device));
    std::vector<HostCol> cols;
    int64_t n = 0;
    try {
      if (use_index) {
        std::vector<uint8_t> idx = read_whole_file(std::string(path) + ".index", 0, 0);
        if (idx.size() % 8 || idx.size() < 16) throw EngineError(B200_ERR_INVALID, "invalid shuffle index file");
        const size_t entries = idx.size() / 8;
        if ((size_t)out_partition + 1 >= entries) throw EngineError(B200_ERR_NOT_FOUND, "partition not found in the shuffle index");
        int64_t o0, o1, first;
        memcpy(&first, idx.data(), 8);
        memcpy(&o0, idx.data() + 8 * (size_t)out_partition, 8);
        memcpy(&o1, idx.data() + 8 * (size_t)out_partition + 8, 8);
        if (o0 < 0 || o1 < o0 || first < 0) throw EngineError(B200_ERR_INVALID, "invalid partition byte range in the shuffle index");
        // the leading schema-only stream, then the partition's own streams
        if (first > 0) {
          std::vector<uint8_t> head = read_whole_file(path, 0, (uint64_t)first);
          ipc::read_streams(head.data(), head.size(), cols);
        }
        if (o1 > o0) {
          std::vector<uint8_t> body = read_whole_file(path, (uint64_t)o0, (uint64_t)(o1 - o0));
          n = ipc::read_streams(body.data(), body.size(), cols);
        }
      } else {
        std::vector<uint8_t> body = read_whole_file(path, byte_offset, byte_length);
        n = ipc::read_streams(body.data(), body.size(), cols);
      }
    } catch (const std::runtime_error& ex) {
      throw EngineError(B200_ERR_INVALID, ex.what());
    }
    // host columns -> Arrow C structs -> the ordinary ingest path
    ArrowArray arr;
    ArrowSchema sch;
    export_record_batch(std::move(cols), n, &arr, &sch);
    DevBatchPtr b = import_batch(e, &arr, &sch);
    std::vector<int64_t> sb;
    for (auto& c : b->cols)
      if (c.type.id == TypeId::Utf8) sb.push_back(c.chars_bytes);
    // src_rank -1: came from a file, not from one of the box's GPU executors
    e->shuffle.store(ShuffleKey{job_id, stage_id, out_partition}, Piece{file_id, b, 0, n, -1, sb}, true);
  });
}

void* b200_host_alloc_pinned(uint64_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, (size_t)bytes, cudaHostAllocDefault) != cudaSuccess) return nullptr;
  return p;
}
void b200_host_free_pinned(void* p) {
  if (p) cudaFreeHost(p);
}

}  // extern "C"
