// Host-callable launchers of every CUDA kernel in libb200exec (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "program.h"

namespace b200 {

// ---- launch accounting (kernels.cu) -------------------------------------------------------------
// Kernels the calling host thread has enqueued so far.  Per thread because several tasks, on one engine or several, run
// at once in one process: the launches of some piece of work are the difference of two readings around it.
uint64_t launches_on_thread();
// Adds n to the calling thread's count: launch_kernel below, and work enqueued by other libraries (an NCCL group).
void count_launches(uint64_t n = 1);
#ifdef __CUDACC__
// The one place the device module launches a kernel (every launcher calls it), so that every launch is counted.
template <class... P, class... A>
inline void launch_kernel(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const A&... args) {
  count_launches();
  kernel<<<grid, block, smem, st>>>(args...);
}
#endif

// ---- fused pipeline (pipeline.cu) ---------------------------------------------------------------
cudaError_t launch_pipeline(const Program& P, int reg_groups, int grid, int block, size_t smem, cudaStream_t st);
// fused scan->filter->project->aggregate kernel (fused.cuh); *is_static: 1 when an ahead-of-time shape ran
cudaError_t launch_fused_pipeline(const Program& P, const FusedSpec& F, FusedShape shape, int reg_groups, int grid, int block, size_t smem, cudaStream_t st,
                                  int* is_static);
bool fused_rows_ok(const Program& P, int grid, int block, int rows_per_thread);
bool pipeline_add_only(const Program& P, int grid, int block);

// ---- aggregate table (kernels.cu) ----------------------------------------------------------------
struct AccKinds {
  uint8_t kind[VM_MAX_ACC];
  int n;
};
void launch_agg_table_init(const AggTable& T, const AccKinds& kinds, cudaStream_t st);

enum AggOutKind : uint8_t {
  AO_KEY = 0,      // a: key index
  AO_ACC_I128,     // a: acc index, b: count-acc index (valid iff count > 0) or 255
  AO_ACC_I64,      // low 64 bits of an I128 accumulator (SUM(Int64) wraps) ; b as above
  AO_ACC_F64,      // f64 sum ; b as above
  AO_COUNT,        // a: acc index -> Int64/UInt64
  AO_MINMAX_F64,   // order-key -> double ; b count
  AO_AVG_DEC,      // a: sum acc, b: count acc, imm: 10^k multiplier exponent
  AO_AVG_F64,      // a: sum acc (f64), b: count acc
  AO_KEY_PACKED,   // a: key index holding a packed short string (OP_STR_PACK8); imm: bit position of the length; aux: 8 B/row chars
  AO_MINMAX_STR,   // a: MIN_STR / MAX_STR acc -> string view (points at the input's characters); b count
  AO_STAT          // VAR / STDDEV / COVAR / CORR result or partial state (Float64); imm: StatOut; st: the cells it reads
};
// what an AO_STAT column holds.  n = count, mean = sum / n, m2 / co = the pass-2 co-moments.  [EXT] NULL rules: sample
// variants n <= 1, population variants n = 0, CORR n < 2 or either m2 = 0; partial states are never NULL (an empty
// group's mean and moments are 0, as DataFusion's accumulators start)
// The regression aggregates (regr_*; [EXT], unpinned: DESIGN.md §6 (xvi)) with sxx, syy, sxy the co-moments: avgx / avgy /
// sxx / syy / sxy NULL when n = 0; slope = (sxy/n) / (sxx/n) and intercept = my - slope * mx NULL when n <= 1 or sxx = 0;
// r2 = (sxy/n)^2 / ((sxx/n)(syy/n)) NULL when n <= 1, sxx = 0 or syy = 0.
enum StatOut : uint8_t {
  SO_MEAN_X = 0, SO_MEAN_Y, SO_M2_X, SO_M2_Y, SO_CO,
  SO_VAR_SAMP, SO_VAR_POP, SO_STDDEV_SAMP, SO_STDDEV_POP, SO_COVAR_SAMP, SO_COVAR_POP, SO_CORR,
  SO_REGR_SLOPE, SO_REGR_INTERCEPT, SO_REGR_R2, SO_REGR_AVGX, SO_REGR_AVGY, SO_REGR_SXX, SO_REGR_SYY, SO_REGR_SXY
};
struct AggOut {
  void* data;
  uint8_t* valid;
  void* aux;
  uint8_t kind;
  uint8_t a, b;
  uint8_t phys;   // output encoding
  int32_t imm;
  // AO_STAT: count acc, sum-x acc, sum-y acc, xx / yy / xy co-moment columns; then (255: none) the RANGE_F64 accs of x, y
  // (raw rows) or of the states' means, and those of the states' m2_x, m2_y (Final): an argument is constant in the group
  // when its range is one value (and every state's m2 is 0), and then its m2 and co-moments are exactly 0 (DESIGN.md §4.1)
  uint8_t st[10];
  uint8_t prec;   // AO_AVG_DEC: result precision
  uint8_t _pad;
};
#ifdef __CUDACC__
// DecimalAverager::avg [EXT]: sum * 10^k / count, truncating toward zero, for the grouped and the window AVG.  Returns
// false (an overflow error) when sum * 10^k leaves the i128 range or the quotient has more than `prec` digits.
__device__ __forceinline__ bool avg_decimal(__int128 sum, unsigned long long count, int k, int prec, __int128* out) {
  __int128 mul = 1, lim = 1;
  for (int i = 0; i < k; i++) mul *= 10;
  for (int i = 0; i < prec; i++) lim *= 10;
  const __int128 max = (__int128)(~(unsigned __int128)0 >> 1), min = -max - 1;
  if (sum > max / mul || sum < min / mul) return false;
  *out = sum * mul / (__int128)count;
  return *out < lim && *out > -lim;
}
#endif
struct AggExtractArgs {
  AggOut out[VM_MAX_OUT];
  int n_out;
  int n_keys;
  unsigned long long* counter;   // device: rows emitted
  unsigned int* error;           // device: RunStatus.error
};
void launch_agg_extract(const AggTable& T, const AggExtractArgs& A, cudaStream_t st);

// ---- scans, histograms, scatter/gather ------------------------------------------------------------
// exclusive prefix sum of n uint32 -> uint64 (out[n] = total if out has n+1 slots)
void launch_scan_u32_to_u64(const uint32_t* in, uint64_t* out, int64_t n, uint64_t* scratch /* >= n/1024+2 */, cudaStream_t st);
void launch_histogram_u32(const uint32_t* ids, int64_t n, uint32_t n_bins, unsigned long long* counts, cudaStream_t st);
// dest[i] = cursor[ids[i]]++  (cursor pre-seeded with the exclusive scan of counts)
// stable placement of rows into hash partitions: dest[i] = rows of lower partitions + earlier rows of the same
// partition (input order kept inside a partition, like the reference's BatchPartitioner).  Scratch as for
// radix_sort_pairs_u64.
void launch_partition_dest_stable(const uint32_t* ids, int64_t n, uint32_t n_bins, uint32_t* dest, uint64_t* keys_a, uint32_t* vals_a, uint64_t* keys_b,
                                      uint32_t* vals_b, uint32_t* hist_scratch, uint64_t* scan_scratch, cudaStream_t st);
void launch_scatter_fixed(const void* in, void* out, const uint32_t* dest, int64_t n, int width, cudaStream_t st);
// out[i] = idx[i] >= 0 ? in[idx[i]] : 0 ; valid_out (optional) = idx>=0 && valid_in
void launch_gather_fixed(const void* in, const uint8_t* valid_in, void* out, uint8_t* valid_out, const int64_t* idx, int64_t n, int width, cudaStream_t st);
// the same for up to GATHER_MAX_COLS columns in one launch
static const int GATHER_MAX_COLS = 32;
struct GatherCol {
  const void* in;
  const uint8_t* valid_in;
  void* out;
  uint8_t* valid_out;
  int width;
  int _pad;
  // partition scatter only: when set, row `dst` of partition p is written to (byte address) part_base[p] + dst * width
  // instead of out + dst * width -- the bases may point into ANOTHER GPU's memory (fused shuffle: the scatter kernel
  // stores straight into the owning executor's window over NVLink)
  const unsigned long long* part_base;
};
struct GatherCols {
  GatherCol c[GATHER_MAX_COLS];
  int n;
};
void launch_gather_multi(const GatherCols& cols, const int64_t* idx, int64_t n, cudaStream_t st);
// ingest: int32 / int64 (width 4 / 8) -> sign-extended 16-byte Decimal128 values
void launch_widen_to_i128(const void* in, int width, void* out, int64_t n, cudaStream_t st);
// out[i] = in[i] - in[0] for i < n_plus_1; first_last[0..1] = in[0], in[n_plus_1 - 1] (device memory)
void launch_rebase_offsets(const int32_t* in, int64_t n_plus_1, int32_t* out, int32_t* first_last, cudaStream_t st);
void launch_iota_i64(int64_t* out, int64_t n, cudaStream_t st);

// ---- strings / validity ------------------------------------------------------------------------
void launch_utf8_to_views(const int32_t* offsets, const uint8_t* chars, unsigned long long* views, int64_t n, cudaStream_t st);
void launch_prepack3(const int32_t* offsets, const uint8_t* chars, int64_t n, uint32_t* out, unsigned int* too_long, cudaStream_t st);
void launch_dec128_image(const void* in, int64_t n, int32_t* out, unsigned int* too_wide, cudaStream_t st);
void launch_view_lengths(const unsigned long long* views, const uint8_t* valid, uint32_t* lens, int64_t n, cudaStream_t st);
void launch_views_to_utf8(const unsigned long long* views, const uint8_t* valid, const uint64_t* offs64, int32_t* offsets_out, uint8_t* chars_out, int64_t n, cudaStream_t st);
void launch_bitmap_to_bytes(const uint8_t* bitmap, int64_t bit_offset, uint8_t* bytes, int64_t n, cudaStream_t st);
void launch_bytes_to_bitmap(const uint8_t* bytes, uint8_t* bitmap, int64_t n, unsigned long long* null_count, cudaStream_t st);

// ---- hash join --------------------------------------------------------------------------------
struct KeyCol {
  const void* data;
  const uint8_t* valid;
  uint8_t phys;
  uint8_t width;
};
struct JoinKeys {
  KeyCol build[VM_MAX_KEYS];
  KeyCol probe[VM_MAX_KEYS];
  int n_keys;
  int null_equals_null;
};
// ---- one-pass stable radix partition + exchange / export packing (shuffle.cu) ---------------------
static const int PART_MAX_STR_COLS = 16;
static const uint32_t PART_MAX_FANOUT = 4096;   // per-warp counters of the scatter kernel must fit shared memory
struct PartStrCol {
  const void* data;       // views (16 B/row) or Arrow int32 offsets
  const uint8_t* valid;
  int is_view;
  int _pad;
};
struct PartStrCols {
  PartStrCol c[PART_MAX_STR_COLS];
  int n;
};
// Where a row's partition id comes from: a materialised uint32 column (computed by the child's pipeline kernel), or --
// when the shuffle keys are plain integer-like columns -- the key columns themselves: the partition kernels then apply the
// row hash of csrc/common/hash.hpp (first key sets, later keys combine, NULL skips) and `% P` on the fly, and the
// materialising pass disappears.
struct PidSrc {
  const uint32_t* pid;
  KeyCol keys[VM_MAX_KEYS];
  int n_keys;
  // 0: the shuffle's partition function, hash(keys) % P (what the reference computes).  != 0: the key hash is re-mixed with
  // this salt first -- used when rows are partitioned for a purpose of the engine's own (partition-first aggregation) whose
  // input may already be one shuffle partition: without the salt all of its keys agree on hash % P_shuffle and would pile
  // up in the few buckets b with b % P_shuffle == p
  int salt;
};
uint32_t partition_n_tiles(int64_t n);
// tile_hist: [P][n_tiles] u32 (may be nullptr when only totals are wanted); counts: [P] u64, pre-zeroed;
// str_bytes: [sc.n][P] u64, pre-zeroed; pid.pid == nullptr && pid.n_keys == 0 means "everything goes to partition 0"
cudaError_t launch_partition_hist(const PidSrc& pid, int64_t n, uint32_t P, uint32_t* tile_hist, unsigned long long* counts, const PartStrCols& sc,
                                  unsigned long long* str_bytes, cudaStream_t st);
// offsets: exclusive scan of tile_hist (partition-major); cols: every column to move (validity bytes as their own
// width-1 entries; only in/out/width are used); dest_out (optional): the destination row of every input row
cudaError_t launch_partition_scatter(const PidSrc& pid, int64_t n, uint32_t P, const uint64_t* offsets, const GatherCols& cols, uint32_t* dest_out,
                                     cudaStream_t st);
enum PackKind : int32_t { PK_COPY = 0, PK_STR_VIEWS = 1, PK_STR_UTF8 = 2, PK_BITMAP = 3, PK_UTF8_VIEWS = 4 };
struct PackJob {
  const void* src;        // bytes / views / int32 offsets (already positioned at the slice's first row)
  const uint8_t* valid;   // strings: validity bytes of the slice or nullptr
  const uint8_t* chars;   // PK_STR_UTF8: chars base the offsets are relative to
  void* dst;              // PK_COPY: destination; strings: int32 offsets out (rows + 1, starting at 0)
  void* dst2;             // strings: characters out
  uint64_t bytes;         // PK_COPY: bytes to copy; strings: capacity of the character area
  int64_t rows;           // strings, PK_BITMAP
  int32_t kind;
  int32_t _pad;
};
void launch_pack_jobs(const PackJob* jobs_dev, int n_jobs, cudaStream_t st);

// ---- FilterExec + column projection without the tile VM (filter.cu) ------------------------------------------
static const int FF_MAX_COLS = 16, FF_MAX_OPS = 48, FF_MAX_IMMS = 40, FF_MAX_OUT = 24;
enum FfOpKind : uint8_t { FF_CMP = 0, FF_AND = 1, FF_OR = 2, FF_NOT = 3, FF_FILTER_REG = 4 };
struct FfCol {
  const void* data;       // values / Arrow offsets / views
  const uint8_t* chars;   // PH_UTF8
  uint8_t phys, width;
  uint8_t _pad[6];
};
struct FfOp {
  uint8_t kind;           // FfOpKind
  uint8_t cmp;            // FF_CMP: 0 EQ 1 NE 2 LT 3 LE 4 GT 5 GE
  uint8_t vt;             // FF_CMP: 0 signed 64-bit, 1 signed 128-bit, 2 string (EQ / NE), 3 unsigned 64-bit
  uint8_t filter;         // 1: the result ANDs into the row's pass flag instead of landing in a register
  uint8_t dst;            // bool register (bit of the per-row register word)
  uint8_t a, b;           // FF_CMP: column or immediate index; logic: bool registers
  uint8_t a_imm, b_imm;   // FF_CMP: operand is an immediate
  uint8_t _pad[3];
};
struct FfImm {
  uint64_t lo, hi;        // integers: two's complement 128-bit; strings: device pointer, length
};
struct FastFilterSpec {
  FfCol cols[FF_MAX_COLS];
  FfOp ops[FF_MAX_OPS];
  FfImm imms[FF_MAX_IMMS];
  int n_cols, n_ops, n_out, _pad;
  uint8_t out_col[FF_MAX_OUT];
  void* out_data[FF_MAX_OUT];
  int64_t n_rows;
  unsigned long long* tile_state;   // one look-back word per 1024-row tile, zeroed
  RunStatus* status;
};
cudaError_t launch_fast_filter(const FastFilterSpec& S, int sm_count, cudaStream_t st);

// ---- high-cardinality group-by over plain columns (groupby.cu) ---------------------------------------
static const int GB_MAX_ACC = 8;
struct GroupBySpec {
  FusedCol cols[FUSED_MAX_COLS];   // data + width of every referenced column (no validity, 4 / 8 / 16 bytes wide)
  int n_cols;
  int n_filters;
  int f_col[FUSED_MAX_FILTERS], f_op[FUSED_MAX_FILTERS];   // op: 0 EQ 1 NE 2 LT 3 LE 4 GT 5 GE
  int64_t f_imm[FUSED_MAX_FILTERS];
  int n_keys;                       // 1 or 2 (two keys: both must lie in [0, 2^32), checked per row)
  int key_col[2];
  int n_prod;                       // decimal products: kind 0 a*(lit-b), 1 a*(lit+b), 2 a*b; a_src 1 = previous product
  int p_kind[2], p_a_src[2], p_a_col[2], p_b_col[2];
  int64_t p_lit[2];
  int n_acc;
  int a_src[GB_MAX_ACC], a_col[GB_MAX_ACC];   // src: 0 column, 1 / 2 product, 3 COUNT
  int64_t n_rows;
  AggTable table;
  RunStatus* status;
  // partition-first mode (pf_K > 0): the rows were radix-partitioned by hash(keys) % pf_K beforehand (shuffle.cu) and bucket
  // b aggregates into its own region [b * pf_slots, (b + 1) * pf_slots) of the table, small enough to stay in L2 while the
  // CTAs of that bucket run.  pf_row_start[b .. b+1] = the bucket's rows, pf_cta_start[b .. b+1] = the CTAs that process them
  // (launch_groupby_plan fills both from the partition counts on the device: no host round trip).
  int pf_K;
  unsigned long long pf_slots;                 // power of two
  const unsigned int* pf_cta_start;            // [pf_K + 1]
  const unsigned long long* pf_row_start;      // [pf_K + 1]
};
cudaError_t launch_groupby(const GroupBySpec& S, int sm_count, cudaStream_t st);
// counts[K] -> row_start[K + 1], cta_start[K + 1] (one CTA per GROUPBY_ROWS_PER_CTA rows of a bucket)
static const int GROUPBY_ROWS_PER_CTA = 1024;
cudaError_t launch_groupby_plan(const unsigned long long* counts, int K, unsigned long long* row_start, unsigned int* cta_start, cudaStream_t st);

// ---- single-pass join (join.cu) -----------------------------------------------------------------
struct JoinNode {   // one per build row
  uint64_t tag;     // exact mode: 64-bit image of the (single, integer-like) key; else the row hash
  int32_t next;     // previous head of the bucket, -1 = end of chain
  uint32_t _pad;
};
// exact == true: one integer-like key column, tag = key (build_hash / probe_hash unused)
void launch_join_build2(const JoinKeys& K, bool exact, const uint64_t* build_hash, int64_t n_build, int32_t* heads /* pre-set to -1 */, uint64_t n_buckets,
                        JoinNode* nodes, cudaStream_t st);
// mode bit 0: emit (build row, probe row) pairs -- *counter (pre-zeroed) ends up with the total number of pairs, of
// which the first `cap` were written; bit 1: probe_mark[j] = 1 for probe rows with a match; bit 2: build_mark[i] = 1
void launch_join_probe2(const JoinKeys& K, bool exact, int mode, const JoinNode* nodes, const int32_t* heads, uint64_t n_buckets, const uint64_t* probe_hash,
                        int64_t n_probe, unsigned long long* counter, uint64_t cap, int64_t* out_build_idx, int64_t* out_probe_idx, uint8_t* probe_mark,
                        uint8_t* build_mark, cudaStream_t st);
// compaction helpers: indices of rows whose flag byte == want
void launch_flag_to_u32(const uint8_t* flags, uint8_t want, uint32_t* out, int64_t n, cudaStream_t st);
void launch_select_indices(const uint32_t* flag01, const uint64_t* offs, int64_t* out_idx, int64_t n, cudaStream_t st);
void launch_mark_from_idx(const int64_t* idx, int64_t n, uint8_t* marks, cudaStream_t st);

// ---- nested-loop join (nlj.cu) ------------------------------------------------------------------
// The join filter as the kernels see it: a boolean program (AND / OR / NOT, Kleene logic) over at most NLJ_MAX_ATOMS
// atoms.  An atom is a Bool column of one side (evaluated beforehand by the VM) or a comparison f(build) op g(probe)
// of two columns, one per side.  Registers are bits of two words per pair: T (known true) and F (known false); NULL
// is neither.  Atom k lands in register k, step s of the program writes register NLJ_MAX_ATOMS + s.
static const int NLJ_MAX_ATOMS = 8;
static const int NLJ_MAX_STEPS = 24;
enum NljAtomKind : uint8_t { NLJ_BUILD_BOOL = 0, NLJ_PROBE_BOOL = 1, NLJ_CMP = 2 };
enum NljValueKind : uint8_t {
  NLJ_V_I64 = 0,   // integer-like columns (Int8..Int64, UInt8..UInt32, Date32, Timestamp, Bool), sign / zero extended
  NLJ_V_U64,       // UInt64, compared unsigned
  NLJ_V_F64,       // Float32 / Float64 in IEEE total order (-0.0 < +0.0, NaN above +inf)
  NLJ_V_I128,      // Decimal128 of one scale
  NLJ_V_STR        // 16-byte views: unsigned bytes, a proper prefix first
};
enum NljStepKind : uint8_t { NLJ_AND = 0, NLJ_OR = 1, NLJ_NOT = 2 };
struct NljAtom {
  KeyCol build, probe;  // NLJ_CMP: both operands; NLJ_BUILD_BOOL / NLJ_PROBE_BOOL: the Bool8 column in its side's slot
  uint8_t kind;         // NljAtomKind
  uint8_t cmp;          // NLJ_CMP: build op probe, 0 EQ 1 NE 2 LT 3 LE 4 GT 5 GE
  uint8_t vk;           // NLJ_CMP: NljValueKind
  uint8_t _pad[5];
};
struct NljStep {
  uint8_t kind, a, b, dst;
};
struct NljSpec {
  NljAtom atoms[NLJ_MAX_ATOMS];
  NljStep steps[NLJ_MAX_STEPS];
  int n_atoms, n_steps;
  int result;   // register holding the filter's value; -1: no filter, every pair matches
  int _pad;
};
// counts[j] = pairs of probe row j that pass; build_mark[i] / probe_mark[j] (optional) = 1 for rows with a pair
void launch_nlj_count(const NljSpec& S, int64_t n_build, int64_t n_probe, uint32_t* counts, uint8_t* build_mark, uint8_t* probe_mark, cudaStream_t st);
// the passing pairs in probe-row order, build-row order inside a probe row, at offsets = exclusive scan of counts
void launch_nlj_write(const NljSpec& S, int64_t n_build, int64_t n_probe, const uint32_t* counts, const uint64_t* offsets, int64_t* out_build_idx,
                      int64_t* out_probe_idx, cudaStream_t st);

// ---- sort -------------------------------------------------------------------------------------
struct SortWordArgs {
  const void* data;
  const uint8_t* valid;
  uint8_t phys;
  uint8_t asc;
  uint8_t nulls_first;
  int32_t word;   // which 64-bit word of the normalised key (strings / i128 have several); -1 = null rank word
};
void launch_sort_word(const SortWordArgs& A, const uint32_t* perm, uint64_t* out, int64_t n, cudaStream_t st);
// Small inputs (n <= SMALL_SORT_MAX_ROWS): stable sort permutation by direct comparison of up to SMALL_SORT_MAX_KEYS keys
// in ONE launch (rank = number of rows that order before), same ordering as the key-word radix sort: NULL placement
// per key, ascending/descending, IEEE total order for floats, bytewise strings with the shorter prefix first.
static const int SMALL_SORT_MAX_ROWS = 1024;
static const int SMALL_SORT_MAX_KEYS = 8;
struct SmallSortKeys {
  SortWordArgs k[SMALL_SORT_MAX_KEYS];  // `word` unused
  int n_keys;
};
void launch_small_sort(const SmallSortKeys& K, int64_t* perm_out, int64_t n, cudaStream_t st);
void launch_max_view_len(const unsigned long long* views, const uint8_t* valid, int64_t n, unsigned int* out_max, cudaStream_t st);
// stable LSD radix sort of (key, val) pairs on 64-bit keys; ping-pong buffers; returns via *result_in_a
void radix_sort_pairs_u64(uint64_t* keys_a, uint32_t* vals_a, uint64_t* keys_b, uint32_t* vals_b, int64_t n, uint32_t* hist_scratch,
                          uint64_t* scan_scratch, cudaStream_t st, bool* result_in_a);
void launch_iota_u32(uint32_t* out, int64_t n, cudaStream_t st);
void launch_u32_to_i64(const uint32_t* in, int64_t* out, int64_t n, cudaStream_t st);

// ---- Parquet page decode (parquet.cu) ----------------------------------------------------------------
enum PqOutKind : int32_t { PQ_OUT_I32 = 0, PQ_OUT_I64 = 1, PQ_OUT_F64 = 2, PQ_OUT_DEC128 = 3, PQ_OUT_STRVIEW = 4, PQ_OUT_BOOL8 = 5 };
// value encoding of a data page as the decode kernels see it (PQ_ENC_DBP and above: pq_delta_prepare + pq_values_delta)
enum PqEncoding : uint32_t {
  PQ_ENC_PLAIN = 0, PQ_ENC_DICT = 1, PQ_ENC_RLE_BOOL = 2,
  PQ_ENC_DBP = 3,   // DELTA_BINARY_PACKED (INT32 / INT64)
  PQ_ENC_DLBA = 4,  // DELTA_LENGTH_BYTE_ARRAY (BYTE_ARRAY)
  PQ_ENC_DBA = 5,   // DELTA_BYTE_ARRAY (BYTE_ARRAY, FIXED_LEN_BYTE_ARRAY)
  PQ_ENC_BSS = 6,   // BYTE_STREAM_SPLIT (INT32 / INT64 / DOUBLE / FIXED_LEN_BYTE_ARRAY)
};
struct PqPage {
  const uint8_t* data;      // page payload in HBM (after the Thrift page header)
  uint32_t n_values;        // values including NULLs (dictionary pages: entries)
  uint32_t def_off, def_len;  // definition-level section inside the payload; len 0 = required column / no levels
  uint32_t val_off, val_len;  // values section
  uint32_t encoding;        // PqEncoding
  uint32_t v1_levels;       // 1: data page V1 of a nullable column -- the payload starts with [u32 length][definition levels], values follow
                            //    (the length sits inside the possibly compressed payload, so it is read on the device); val_len = payload bytes
  int64_t row0;             // first row of the page inside the column (dictionary pages: first entry in the dictionary array)
  int64_t dict_base;        // data pages: first entry of their chunk's dictionary
};
struct PqColumn {
  int32_t phys;             // parquet physical type (pq::PhysType)
  int32_t type_length;      // FIXED_LEN_BYTE_ARRAY
  int32_t out_kind;         // PqOutKind
  int32_t _pad;
  void* dict;               // decoded dictionary entries (output type; byte arrays as 16-byte views)
};
struct PqDecompJob {
  const uint8_t* src;   // compressed (or stored) bytes in HBM
  uint8_t* dst;         // where the page payload is rebuilt
  uint32_t src_len, dst_len;
  uint32_t raw_copy;    // 1: plain copy (sections that are never compressed)
  uint32_t codec;       // the column chunk's parquet CompressionCodec: selects the kernel that runs the job
};
// One warp per job; a job that does not decode to exactly dst_len bytes sets a bit in *error: 1 Snappy, 2 GZIP, 4 LZ4_RAW.
void launch_pq_snappy(const PqDecompJob* jobs, int n_jobs, unsigned int* error, cudaStream_t st);
void launch_pq_inflate(const PqDecompJob* jobs, int n_jobs, unsigned int* error, cudaStream_t st);  // GZIP: gzip / zlib members
void launch_pq_lz4(const PqDecompJob* jobs, int n_jobs, unsigned int* error, cudaStream_t st);      // LZ4_RAW: one LZ4 block
void launch_pq_levels(const PqPage* pages, int n_pages, uint8_t* valid, uint32_t* nonnull, unsigned long long* total_nonnull, cudaStream_t st);
void launch_pq_page_scan(const uint32_t* nonnull, int n_pages, unsigned long long* dense_base, cudaStream_t st);
void launch_pq_dict(const PqColumn& C, const PqPage* dict_pages, int n_dicts, cudaStream_t st);
void launch_pq_values(const PqColumn& C, const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint32_t* nonnull, void* out, cudaStream_t st);
void launch_pq_expand(const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint8_t* valid, const void* dense, void* out, int width,
                      cudaStream_t st);
// Per-column state of the DELTA / BYTE_STREAM_SPLIT decoders.  pq_delta_prepare validates every such page (sets *error on
// malformed input), decodes DELTA_BYTE_ARRAY prefix / suffix lengths into pre / sfx (dense value index, like the values) and
// writes each page's reconstructed string bytes to page_bytes (0 for other pages) and their sum to *char_total; the
// exclusive scan of page_bytes (char_base) places each page's strings in `chars`.
struct PqDeltaAux {
  unsigned int* error;
  uint32_t* pre;                    // DELTA_BYTE_ARRAY columns: prefix length per value
  uint32_t* sfx;                    //                          suffix length per value
  uint32_t* page_bytes;             // DELTA_BYTE_ARRAY strings: bytes per page
  unsigned long long* char_total;
  const unsigned long long* char_base;
  uint8_t* chars;                   // reconstructed DELTA_BYTE_ARRAY strings (the views point here)
};
void launch_pq_delta_prepare(const PqColumn& C, const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint32_t* nonnull, const PqDeltaAux& A,
                             cudaStream_t st);
void launch_pq_values_delta(const PqColumn& C, const PqPage* pages, int n_pages, const unsigned long long* dense_base, const uint32_t* nonnull, void* out,
                            const PqDeltaAux& A, cudaStream_t st);

// ---- CSV / TPC-H .tbl scan (csv.cu) -------------------------------------------------------------------
static const int CSV_TILE = 1024;    // bytes per thread of the record-boundary passes
static const int CSV_BLOCK = 256;    // tiles per block
static const int CSV_STATES = 6;     // quote state machine: record start, field start, unquoted, quoted, quote seen, escape
struct CsvDialect {
  uint8_t delim, quote, escape, has_escape;
};
struct CsvTrans {   // what a run of bytes does to each entry state: exit state and record starts seen
  uint8_t exit[CSV_STATES];
  uint8_t _pad[2];
  uint32_t cnt[CSV_STATES];
};
int64_t csv_tile_count(int64_t bytes);
int64_t csv_block_count(int64_t bytes);
// passes 1 + 2: per-tile transitions (tiles: csv_tile_count), per-block entry state and first record (csv_block_count),
// *n_records, and *has_quote |= 1 when the span holds a quote or escape byte (both zeroed by the caller)
void launch_csv_records_count(const uint8_t* data, int64_t bytes, const CsvDialect& d, CsvTrans* tiles, CsvTrans* blocks, uint8_t* blk_state,
                              unsigned long long* blk_base, unsigned int* has_quote, unsigned long long* n_records, cudaStream_t st);
// pass 3: rec_start[r] = offset of record r's first byte (empty lines are no records)
void launch_csv_record_starts(const uint8_t* data, int64_t bytes, const CsvDialect& d, const CsvTrans* tiles, const uint8_t* blk_state,
                              const unsigned long long* blk_base, uint64_t* rec_start, cudaStream_t st);
// reasons in a CSV error word (bits 16-23; bits 0-15 detail, bits 24-63 the row)
enum CsvError : int {
  CSV_E_FIELDS = 1, CSV_E_NULL, CSV_E_INT, CSV_E_INT_RANGE, CSV_E_DEC, CSV_E_DEC_RANGE, CSV_E_DEC_SCALE, CSV_E_DEC_EXP, CSV_E_FLOAT, CSV_E_DATE,
  CSV_E_BOOL, CSV_E_UTF8
};
struct CsvFieldArgs {
  const uint8_t* data;
  int64_t bytes;
  const uint64_t* rec_start;
  int64_t n_records, skip;        // records of the span; skip = 1 drops the header record
  CsvDialect d;
  int n_fields;                   // schema columns
  const int32_t* slot_of_field;   // [n_fields] output slot of each schema column, -1 = not materialised
  unsigned long long* views;      // [slots][n_total] {pointer, length}
  int64_t n_total, row_base;      // rows of the scan; first row of this span
  uint8_t* side;                  // unquoting buffer, offsets as in data (nullptr when the span holds no quote byte)
  unsigned long long* err;        // field-count errors (CSV_E_FIELDS, detail = fields found)
};
void launch_csv_fields(const CsvFieldArgs& A, cudaStream_t st);
enum CsvFamily : int { CSV_FAM_INT = 0, CSV_FAM_DEC, CSV_FAM_F64, CSV_FAM_F32, CSV_FAM_DATE, CSV_FAM_BOOL, CSV_FAM_UTF8 };
struct CsvConvertArgs {
  const unsigned long long* views;  // [n] fields
  int64_t n;
  void* out;                        // values (CSV_FAM_UTF8: views)
  uint8_t* valid;
  unsigned long long* err;          // first failing row of the column
  unsigned long long* null_count;
  __int128 lo, hi;                  // CSV_FAM_INT: the type's range
  int width, is_signed, precision, scale, nullable;
};
void launch_csv_convert(const CsvConvertArgs& A, int family, cudaStream_t st);

// ---- newline-delimited JSON scan (json.cu) ------------------------------------------------------------
static const int JSON_TILE = 1024;   // bytes per thread of the record-boundary passes
static const int JSON_BLOCK = 256;   // tiles per block
int64_t json_tile_count(int64_t bytes);
int64_t json_block_count(int64_t bytes);
// passes 1 + 2: records (lines holding more than whitespace) per tile (tile_cnt: json_tile_count) and the first record of
// every block (blk_base: json_block_count), *n_records, and *has_backslash |= 1 when the span holds a '\' (both zeroed by
// the caller)
void launch_json_records_count(const uint8_t* data, int64_t bytes, uint32_t* tile_cnt, unsigned long long* blk_base, unsigned int* has_backslash,
                               unsigned long long* n_records, cudaStream_t st);
// pass 3: rec_start[r] = offset of record r's first byte
void launch_json_record_starts(const uint8_t* data, int64_t bytes, const uint32_t* tile_cnt, const unsigned long long* blk_base, uint64_t* rec_start,
                               cudaStream_t st);
// reasons in a JSON error word, after the converters' CSV_E_* (bits 16-23; bits 0-15 detail, bits 24-63 the row)
enum JsonError : int {
  JSON_E_NOT_OBJECT = 32,   // the line is not one object
  JSON_E_SYNTAX,            // a byte where the grammar allows none
  JSON_E_UNTERMINATED,      // the line ends inside the object
  JSON_E_TRAILING,          // bytes after the object
  JSON_E_CONTROL,           // raw byte below 0x20 in a string
  JSON_E_UTF8,              // invalid UTF-8 in a string
  JSON_E_ESCAPE,            // unknown escape or bad \uXXXX
  JSON_E_SURROGATE,         // lone surrogate
  JSON_E_NUMBER,            // not an RFC 8259 number
  JSON_E_LITERAL,           // not true / false / null
  JSON_E_DUPLICATE,         // a materialised key twice in one object (detail: the slot)
  JSON_E_DEPTH,             // a skipped value nested deeper than JSON_MAX_DEPTH
  JSON_E_KIND,              // a value of another JSON kind than the column reads (detail: the kind)
};
static const int JSON_MAX_DEPTH = 64;
// kinds of a JSON view (bits 32-39 of its length word; json_fields_kernel writes them, text_convert<FAM, true> checks them)
enum JsonKind : int { JK_NUMBER = 1, JK_STRING, JK_TRUE, JK_FALSE, JK_NULL, JK_NESTED };
// materialised names as the field pass looks them up: an open-addressing table of n_slots entries (power of two), each
// {FNV-1a hash, offset into names, length, output slot or -1}, staged in shared memory
struct JsonKey {
  uint32_t hash;
  uint16_t off, len;
  int32_t slot;
};
struct JsonFieldArgs {
  const uint8_t* data;
  int64_t bytes;
  const uint64_t* rec_start;
  int64_t n_records;
  const JsonKey* keys;            // [n_keys] (n_keys a power of two)
  int n_keys;
  const uint8_t* names;           // [names_bytes]
  int names_bytes;
  unsigned long long* views;      // [slots][n_total] {pointer, length | kind << 32}, zeroed by the caller (missing = NULL)
  int64_t n_total, row_base;      // rows of the scan; first row of this span
  uint8_t* side;                  // unescaping buffer, offsets as in data (nullptr when the span holds no '\')
  unsigned long long* err;        // structural errors (JSON_E_*)
};
void launch_json_fields(const JsonFieldArgs& A, cudaStream_t st);
// as launch_csv_convert, with JSON's NULL (null pointer) and kinds (text_convert.cuh)
void launch_json_convert(const CsvConvertArgs& A, int family, cudaStream_t st);
static inline __host__ __device__ uint32_t json_hash_step(uint32_t h, uint8_t b) { return (h ^ b) * 16777619u; }
static const uint32_t JSON_HASH_SEED = 2166136261u;  // FNV-1a

// ---- window functions (window.cu) ---------------------------------------------------------------
// Kernels work on sorted positions i; perm[i] is the input row there (nullptr: the input already is in sorted order).
static const int WIN_MAX_KEYS = 16;
struct WinKeys {
  KeyCol k[WIN_MAX_KEYS];  // partition keys, then order keys (strings as views)
  int n_part, n_order;
};
// part_flag / peer_flag[i] = 1 where sorted row i starts a partition / a peer group (a partition start is also a peer start)
void launch_window_flags(const WinKeys& K, const int64_t* perm, int64_t n, uint32_t* part_flag, uint32_t* peer_flag, cudaStream_t st);
struct WinBounds {
  uint32_t* pid;              // [n] partition of each sorted row
  uint32_t* gid;              // [n] peer group of each sorted row
  uint32_t* part_start;       // [partitions + 1] first sorted row of each partition, then n
  uint32_t* peer_start;       // [peer groups + 1] first sorted row of each peer group, then n
  uint32_t* part_first_peer;  // [partitions] peer group of each partition's first row
};
// part_ex / peer_ex: exclusive scans of the flags (launch_scan_u32_to_u64)
void launch_window_segments(const uint32_t* part_flag, const uint32_t* peer_flag, const uint64_t* part_ex, const uint64_t* peer_ex, int64_t n,
                            const WinBounds& B, cudaStream_t st);
// accumulator value types and their argument conversions
enum WinAcc : uint8_t { WACC_I64 = 0, WACC_F64 = 1, WACC_I128 = 2 };
enum WinConv : uint8_t {
  WCV_I64 = 0,     // integers, Date32, Bool: sign / zero extended (WACC_I64)
  WCV_U64_KEY,     // UInt64 with the sign bit flipped: signed order = unsigned order (MIN / MAX)
  WCV_F64,         // any number as double (float SUM / AVG, integer AVG)
  WCV_F64_KEY,     // Float32 / Float64 as an IEEE total-order key (MIN / MAX)
  WCV_I128,        // Decimal128
  WCV_VALID,       // COUNT(x): only the validity
  WCV_ONE          // COUNT(*): every row counts
};
struct WinLoad {
  const void* data;
  const uint8_t* valid;
  uint8_t phys, conv;
  void* out;           // [n] accumulator values in sorted order
  uint8_t* out_valid;  // [n]
};
void launch_window_load(const WinLoad& L, const int64_t* perm, int64_t n, cudaStream_t st);
enum WinOp : uint8_t { WOP_SUM = 0, WOP_MIN, WOP_MAX };
enum WinSeg : uint8_t { WSEG_PART = 0, WSEG_PEER, WSEG_BLOCK };
// segmented inclusive scan of (value, non-NULL count) over sorted rows; dir 1 runs from the last row to the first
struct WinScan {
  const void* vals;
  const uint8_t* valid;
  void* out_v;
  uint32_t* out_c;
  void* tiles;  // window_scan_tile_bytes(n)
  int64_t n, w;  // w: WSEG_BLOCK block length
  uint8_t acc, op, dir, seg;
};
int64_t window_scan_tile_bytes(int64_t n);
void launch_window_scan(const WinScan& S, const WinBounds& B, cudaStream_t st);
enum WinFnKind : uint8_t { WF_ROW_NUMBER = 0, WF_RANK, WF_DENSE_RANK, WF_PERCENT_RANK, WF_CUME_DIST, WF_NTILE, WF_OFFSET, WF_FIRST, WF_LAST, WF_NTH, WF_AGG };
enum WinBound : uint8_t { WB_UNBOUNDED_PRECEDING = 0, WB_PRECEDING, WB_CURRENT_ROW, WB_FOLLOWING, WB_UNBOUNDED_FOLLOWING };
enum WinUnits : uint8_t { WUNITS_ROWS = 0, WUNITS_RANGE };
// how WF_AGG reads a frame [fs, fe): the forward scan at fe - 1, the backward scan at fs, or both over blocks of w rows
enum WinRead : uint8_t { WRD_FWD = 0, WRD_BWD, WRD_BLOCKS };
enum WinFinish : uint8_t { WFIN_VALUE = 0, WFIN_COUNT, WFIN_AVG, WFIN_MINMAX_U64, WFIN_MINMAX_F64 };
struct WinEval {
  uint8_t fn, units, s_kind, e_kind;
  uint8_t acc, op, read, fin;
  uint8_t out_phys;
  uint8_t prec;         // WFIN_AVG over Decimal128: result precision
  int32_t imm;          // WFIN_AVG over Decimal128: result scale - input scale
  int64_t s_off, e_off;
  int64_t arg;          // WF_NTILE: n; WF_NTH: n; WF_OFFSET: signed distance (LEAD +k, LAG -k)
  int64_t w;
  const void* fwd_v;
  const uint32_t* fwd_c;
  const void* bwd_v;
  const uint32_t* bwd_c;
  void* out;            // result per input row
  uint8_t* out_valid;
  int64_t* idx_out;     // WF_OFFSET / WF_FIRST / WF_LAST / WF_NTH: input row to take per input row, -1 = none
  unsigned int* error;  // WFIN_AVG over Decimal128: overflow
};
void launch_window_eval(const WinEval& E, const WinBounds& B, const int64_t* perm, int64_t n, cudaStream_t st);
// LAG / LEAD default: rows with idx < 0 get the 16-byte literal image (its first `width` bytes) and valid = 1
void launch_window_fill(const int64_t* idx, int64_t n, void* out, uint8_t* valid, int width, const void* lit16, cudaStream_t st);

// ---- synthetic TPC-H input ----------------------------------------------------------------------
void launch_tpch_fixed(int table, int col, int kind, int64_t msf, int64_t row0, int64_t n, void* out, cudaStream_t st);
void launch_tpch_str_len(int table, int col, int64_t msf, int64_t row0, int64_t n, uint32_t* lens, cudaStream_t st);
void launch_tpch_str_fill(int table, int col, int64_t msf, int64_t row0, int64_t n, const uint64_t* offs64, int32_t* offsets, uint8_t* chars, cudaStream_t st);

}  // namespace b200
