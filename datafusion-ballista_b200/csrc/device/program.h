// Device "pipeline program": what the host lowers one operator pipeline
// (source -> [FilterExec | ProjectionExec]* -> sink) into, and what the fused pipeline kernel
// (pipeline.cu) interprets.  Plain-old-data only: the struct is passed to the kernel as a
// __grid_constant__ parameter and read through the constant cache (warp-uniform indices).
//
// Reference operators being fused here: FilterExec / ProjectionExec / AggregateExec partial+final
// (parameter surface: ballista/core/proto/datafusion.proto:1027-1034, :1211-1215, :1257-1271) and
// the PhysicalExpr tree (:851-901) which DataFusion evaluates column-at-a-time per 8192-row batch;
// here the same tree is evaluated tile-at-a-time with the tile resident in shared memory.
#pragma once
#include <stdint.h>

namespace b200 {

static const int VM_R = 2;            // rows per thread per tile (register-blocked)
static const int VM_MAX_COLS = 24;    // source columns of one pipeline
static const int VM_MAX_REGS = 40;    // VM value registers (shared-memory resident)
static const int VM_MAX_IMMS = 128;
static const int VM_MAX_INSTR = 224;
static const int VM_MAX_OUT = 32;     // materialize sink output columns
static const int VM_MAX_KEYS = 8;     // group-by / hash key columns
static const int VM_MAX_ACC = 16;     // physical accumulators of an aggregate sink
static const int VM_REG_ACC = 6;      // accumulators held in registers by the AGG_REG sink
static const int VM_REG_GROUPS = 4;   // groups held in registers by the AGG_REG sink
static const int VM_MAX_STAGES = 4;
static const int VM_MAX_MOM = 6;      // centred co-moments of one aggregate sink (VAR / STDDEV / COVAR / CORR)

// physical (in-HBM) column encodings
enum Phys : uint8_t {
  PH_I8 = 0, PH_I16, PH_I32, PH_I64, PH_U8, PH_U16, PH_U32, PH_U64, PH_F32, PH_F64,
  PH_DEC128,   // 16-byte little-endian two's complement (Arrow Decimal128)
  PH_BOOL8,    // one byte per value (device-internal; Arrow bitmaps are expanded at ingest)
  PH_UTF8,     // Arrow Utf8: int32 offsets (+ chars buffer)
  PH_STRVIEW   // device-internal string view {ptr, len}: 16 bytes
};

// value kinds inside the VM (== b200::PK)
enum VK : uint8_t { VK_BOOL = 0, VK_I64 = 1, VK_F64 = 2, VK_I128 = 3, VK_STR = 4 };

enum OperandKind : uint8_t { OPD_NONE = 0, OPD_COL = 1, OPD_REG = 2, OPD_IMM = 3 };

struct Operand {
  uint8_t kind;  // OperandKind
  uint8_t vk;    // VK of the value
  uint16_t idx;  // column / register / immediate index
};

enum VOp : uint8_t {
  OP_NOP = 0,
  OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_MOD, OP_NEG,             // t = VK_I64 | VK_F64 | VK_I128
  OP_CMP_EQ, OP_CMP_NE, OP_CMP_LT, OP_CMP_LE, OP_CMP_GT, OP_CMP_GE,  // t = operand VK
  OP_AND, OP_OR, OP_NOT, OP_IS_NULL, OP_IS_NOT_NULL,
  OP_CAST_I64_F64, OP_CAST_I64_I128,   // imm = scale exponent (value * 10^imm), aux: precision to check
  OP_CAST_I128_I128_UP,                // imm = exponent
  OP_CAST_I128_I128_DOWN,              // imm = exponent (round half away from zero)
  OP_CAST_I128_F64,                    // imm = scale
  OP_CAST_F64_I64, OP_CAST_I128_I64,   // imm = scale (truncate)
  OP_CAST_F64_I128,                    // imm = scale
  OP_WRAP_I64,                         // aux = Phys of the logical integer width (wrapping arithmetic)
  OP_NARROW_I64,                       // aux = Phys; out of range -> NULL (safe cast)
  OP_CHECK_PRECISION,                  // aux = precision; out of range -> NULL
  OP_SELECT,                           // dst = a(bool) ? b : dst      (CASE lowering)
  OP_MOV,                              // dst = a
  OP_LIKE,                             // a: STR, imm: immediate index of pattern; aux: 1 = negated
  OP_DATE_PART,                        // a: I64 days -> I64 field; aux = DatePart
  OP_SUBSTR,                           // a: STR, b: I64 start, imm: immediate idx of len or -1
  OP_HASH,                             // dst(I64) = hash(a)                 (first key column)
  OP_HASH_COMBINE,                     // dst(I64) = a valid ? combine(hash(a), dst) : dst
  OP_FILTER,                           // active &= a.value & a.valid
  OP_MOD_U64,                          // dst = (uint64)a % imm64 (partition id); imm = immediate idx
  OP_DEC_MUL_LIT_MINUS,                // fused: dst = a * (imm - b)   [I128 x (I64-range)] checked
  OP_DEC_MUL_LIT_PLUS,                 // fused: dst = a * (imm + b)
  OP_MADD_I64,                         // dst = a + b * imm64 (imm = immediate index); wrapping
  OP_STR_PACK8,                        // dst(I64) = len<<imm | bytes of a string of <= aux bytes (imm = 56/aux = 7 or imm = 24/aux = 3); longer -> pack_overflow
  // CASE (lower.hpp compile_case): m = a (a bool register) or, without a, the rows active now; with b, m &= b (TRUE rows;
  // aux = 1: m &= ~b); dst (a never-NULL bool register), if given, = m; with a, the rows active from here on = m
  OP_ACTIVE,
  // scalar functions (cold: scalar_num_op / scalar_nullif_op / scalar_str_op in pipeline.cu); every op from OP_ABS on is one
  OP_ABS,                              // t = VK_I64 | VK_F64 | VK_I128; aux = Phys of a signed integer (its minimum raises overflow)
  OP_ROUND,                            // t = VK_F64; imm = immediate idx of the factor f; aux = PH_F32 for f32 arithmetic
  OP_FLOOR, OP_CEIL,                   // t = VK_F64
  OP_NULLIF,                           // t = operand VK; dst = a, NULL where a = b (floats: bitwise, i.e. total order)
  OP_CHAR_LENGTH, OP_OCTET_LENGTH,     // a: STR -> I64
  OP_STARTS_WITH, OP_ENDS_WITH,        // a, b: STR -> BOOL
  OP_TRIM,                             // a: STR -> STR view; aux = TrimSide; imm = immediate idx of the set (" " by default)
  // bitwise operators (scalar_bit_op): t = VK_I64, a and b of one integer type; aux = Phys of that type (shift counts are
  // taken modulo its bit width; >> is arithmetic for signed types, logical for unsigned ones)
  OP_BIT_AND, OP_BIT_OR, OP_BIT_XOR, OP_SHL, OP_SHR,
  // regular expressions (scalar_regex_op): ILIKE, ~ / ~* / !~ / !~* and regexp_like.  a: STR -> BOOL; aux: 1 = negated;
  // imm: immediate with the DFA's device pointer in lo and its shape (csrc/common/regex_dfa.hpp dfa_shape_pack) in hi
  OP_REGEX,
  // string builders (scalar_build_op): each writes its result's bytes into the launch's character arena (Program::arena)
  // and yields an ordinary {ptr, len} view.  Semantics: DESIGN.md §6 (xi).
  OP_CONCAT,    // imm: first immediate of the argument operands (below); aux: BUILD_* flags; a: separator (BUILD_WS)
  OP_REPEAT,    // a: STR, b: I64 count
  OP_REVERSE,   // a: STR -> its code points in reverse order
  OP_TO_STR     // CAST(a AS Utf8); aux = ToStrKind; imm = scale (TS_DEC128)
};
enum BuildFlags : uint8_t {
  BUILD_NULLS = 1,  // `||`: NULL if any argument is NULL (else NULL arguments are skipped: concat, concat_ws)
  BUILD_WS = 2      // concat_ws: operand a is the separator, written between the present arguments; NULL iff it is
};
enum ToStrKind : uint8_t { TS_INT = 0, TS_UINT64, TS_DEC128, TS_DATE32, TS_BOOL };
// OP_CONCAT's arguments travel in consecutive immediates, eight per immediate: 16 bits each (kind << 12 | idx, all
// VK_STR), four in lo and four in hi; the first immediate's _pad holds their count

enum DatePart : uint8_t { DP_YEAR = 0, DP_QUARTER, DP_MONTH, DP_WEEK, DP_DAY, DP_DOY, DP_DOW };
enum TrimSide : uint8_t { TRIM_BOTH = 0, TRIM_LEADING, TRIM_TRAILING };

enum InstrFlags : uint8_t {
  IF_NULLCHK = 1,   // some operand may be NULL: compute validity
  IF_CHECKED = 2,   // overflow / divide-by-zero raise an execution error
  IF_FILTER = 4     // comparison fused with FilterExec: active &= result (no destination register)
};

struct VInstr {
  uint8_t op;
  uint8_t t;
  uint8_t flags;
  uint8_t aux;
  Operand dst, a, b;
  int32_t imm;
};

struct ColDesc {
  const void* data;        // values / offsets / views
  const uint8_t* valid;    // byte per row or nullptr
  const uint8_t* chars;    // PH_UTF8: character bytes
  const void* img32;       // 4-byte image per row (DevColumn::img32): PH_UTF8 len<<24|bytes, PH_DEC128 int32 value; else nullptr
  uint32_t smem_off;       // offset of this column's tile inside a stage buffer
  uint32_t valid_smem_off; // offset of the validity tile (if valid != nullptr)
  uint8_t phys;
  uint8_t width;           // bytes per row in `data`
  uint8_t in_tile;         // staged through shared memory by the tile loader
  uint8_t _pad;
};

struct RegDesc {
  uint32_t smem_off;   // value storage: width * TILE bytes, [r][thread] interleaved
  uint32_t valid_off;  // u32 mask per thread (bit r), or 0xFFFFFFFF if never NULL
  uint8_t vk;
  uint8_t _pad[3];
};

struct ImmDesc {
  uint64_t lo, hi;  // I64/F64 bits in lo; I128 lo/hi; STR: ptr in lo, len in hi
  uint32_t is_null;
  uint32_t _pad;
};

// ---- sinks ---------------------------------------------------------------------------------------
enum SinkKind : uint8_t { SINK_MATERIALIZE = 0, SINK_AGG_REG = 1, SINK_AGG_GLOBAL = 2 };

struct OutCol {
  Operand src;
  void* data;          // output values
  uint8_t* valid;      // output validity bytes or nullptr
  uint8_t phys;        // output encoding (PH_STRVIEW for strings)
  uint8_t _pad[7];
};

// Accumulators.  A cell is 16 bytes (lo, hi):
//  SUM_I128 / MIN_I128 / MAX_I128: 128-bit two's complement; COUNT / COUNT_STAR: count in lo;
//  SUM_F64: the double's bits in lo; MIN_F64 / MAX_F64: the total-order key of the double in lo;
//  MIN_STR / MAX_STR: the string view {ptr, len} of the best value so far (unsigned bytewise order, a proper prefix
//  first), len = ACC_STR_NONE while no value has been seen -- the identity of both (an empty string is a value).
//  The characters stay where the rows had them; the host copies the extracted results into buffers of their own.
//  String MIN / MAX and the zero-extended UInt64 MIN / MAX are the register sink's "side" accumulators (pipeline.cu).
enum AccKind : uint8_t { ACC_SUM_I128 = 0, ACC_SUM_F64, ACC_COUNT, ACC_MIN_I128, ACC_MAX_I128, ACC_MIN_F64, ACC_MAX_F64, ACC_COUNT_STAR,
                         ACC_MIN_STR, ACC_MAX_STR };
static const unsigned long long ACC_STR_NONE = ~0ull;

struct AccDesc {
  Operand src;      // value operand (ignored for ACC_COUNT_STAR)
  uint8_t kind;     // AccKind
  uint8_t nullable; // operand may be NULL
  uint8_t zext;     // MIN_I128 / MAX_I128 over UInt64: the operand's 64 bits are zero-extended, not sign-extended
  uint8_t _pad;
};

// Global aggregate hash table (SoA), shared by both aggregate sinks and by the extraction kernel.
// Centred co-moment of the statistical aggregates, filled by the second launch of an aggregate program ("pass 2"):
//   table column `col`     += w * (x - mx) * (y - my) + b   over the rows where x, y (and w, b when present) are not NULL,
//   table column `col` + 1 += w * (x - mx),  `col` + 2 += w * (y - my)
// (the corrected two-pass algorithm: the extraction subtracts col+1 * col+2 / n, which removes the error of a rounded
// centre to first order -- a plain f64 mean of values near 1e12 is off by far more than their spread allows),
// where the centres mx = acc[sx] / acc[cnt] and my = acc[sy] / acc[cnt] are the group's cells of the first launch (pass 1:
// a COUNT or an integer SUM of weights, and f64 SUMs of w * x and w * y).  Raw rows: w = 1 (OPD_NONE), no b.  Merging
// partial states (Chan et al.): w = the state's count, x / y its means, b its m2 or co-moment.  x and y are f64 operands.
struct MomDesc {
  Operand x, y, w, b;   // w, b: OPD_NONE when absent
  uint8_t cnt, sx, sy;  // pass-1 accumulator columns of the centres
  uint8_t col;          // first of the three table accumulator columns of the co-moment
  uint8_t _pad[4];
};

struct AggTable {
  unsigned long long* hash;   // [cap] 0 = empty
  unsigned int* state;        // [cap] 0 empty, 1 claimed, 2 keys published
  unsigned int* lock;         // [cap] merge lock
  unsigned long long* keys;   // [n_keys][cap][2]  (16 B per key: I64/F64 in word 0, I128 lo/hi, STR ptr/len)
  unsigned char* key_valid;   // [n_keys][cap]
  unsigned long long* acc;    // [n_acc][cap][2]
  unsigned long long* seen;   // [n_acc][cap]  number of non-NULL contributions
  unsigned long long cap;     // power of two
  unsigned int* n_groups;     // occupied slots
};

struct RunStatus {
  unsigned int error;       // 0 ok; 1 arithmetic overflow; 2 divide by zero; 3 other
  unsigned int overflow;    // aggregate table / register-group overflow: retry with a bigger sink
  unsigned long long out_rows;   // materialize sink: rows written
  unsigned long long in_active;  // rows that passed all filters
  unsigned int pack_overflow;    // OP_STR_PACK8 met a string longer than 7 bytes: re-lower without packing
  unsigned int _pad;             // (keeps the struct 8-byte aligned; the group-by kernel reports "outside my pattern" through pack_overflow too)
  unsigned long long arena_need; // string builders: bytes reserved in the character arena, counted past its capacity
};

struct Program {
  // source
  int32_t n_cols;
  int32_t n_regs;
  int32_t n_imms;
  int32_t n_instr;
  uint32_t stage_bytes;   // shared memory per stage buffer
  uint32_t regs_bytes;    // shared memory for VM registers
  uint32_t n_stages;
  uint32_t use_tma;       // all staged columns are 16-byte aligned: cp.async.bulk path
  ColDesc cols[VM_MAX_COLS];
  RegDesc regs[VM_MAX_REGS];
  ImmDesc imms[VM_MAX_IMMS];
  VInstr code[VM_MAX_INSTR];
  // sink
  uint8_t sink;
  uint8_t n_out;
  uint8_t n_keys;
  uint8_t n_acc;
  uint32_t _pad0;
  OutCol out[VM_MAX_OUT];       // SINK_MATERIALIZE
  Operand keys[VM_MAX_KEYS];    // aggregate sinks: group keys
  Operand key_hash;             // aggregate sinks: I64 register holding the row hash (OPD_NONE if no keys)
  uint8_t keys_all_i64;         // every key is an integer-like 64-bit value (ints, dates, bools, packed strings)
  uint8_t has_side_acc;         // some accumulator is a string MIN / MAX or a UInt64 MIN / MAX (zext)
  uint8_t _pad1[2];
  AccDesc acc[VM_MAX_ACC];
  AggTable table;
  unsigned long long* acc_hi;   // register sink: high 64-bit words [cta][thread][group][acc], pre-zeroed
  RunStatus* status;
  unsigned long long* tile_state;  // materialize sink: one look-back word per tile, zeroed before the launch
  int64_t n_rows;
  unsigned long long* acc_side; // register sink with has_side_acc: the side accumulators' 64-bit values, laid out as acc_hi
  // statistical aggregates: the co-moments (all the fields above describe pass 1 and stay as they are for pass 2)
  uint8_t n_mom;
  uint8_t mom_pass;             // 1: this launch is pass 2 and folds rows into the co-moments only
  uint8_t _pad2[6];
  MomDesc mom[VM_MAX_MOM];
  // grouping sets (global sink only): every live row is upserted once per set s, with the keys whose bit is set in
  // set_mask[s] replaced by NULL and set_id[s] as one more VK_I64 key (index n_keys).  key_hashes[k] is the I64
  // register holding the hash of key k (0 for NULL); the table hash of a set combines those of its present keys.
  uint8_t n_sets;               // 0: a plain aggregate
  uint8_t _pad3[7];
  uint8_t set_mask[32];
  uint64_t set_id[32];
  Operand key_hashes[VM_MAX_KEYS];
  // string builders (OP_CONCAT and up): the launch's character arena; a reservation beyond arena_cap writes nothing
  uint8_t* arena;
  unsigned long long arena_cap;
};

// ---- fused fast path (scan -> filter -> decimal products -> <=4-group SUM/COUNT aggregate) -----------
// A pattern-matched specialisation of the lowered program for the TPC-H q1/q6 shape (SURVEY.md 7.1
// step 3): FilterExec + ProjectionExec + AggregateExec(Partial) run in one kernel whose every value
// lives in registers.  Each WARP owns a private ring of TMA-filled stage buffers (no CTA barrier on
// the data path).  The kernel is compiled once per "shape" (widths, compare ops, product kinds,
// accumulator sources -- see FusedShape) for the shapes listed in pipeline.cu, plus one variant that
// reads the same description from constant memory at run time for everything else.
static const int FUSED_MAX_FILTERS = 6;
static const int FUSED_MAX_COLS = 12;
static const int FUSED_MAX_STAGES = 8;
static const int FUSED_MAX_WARPS = 16;
struct FusedCol {
  const void* data;     // column values (Utf8: the int32 offsets)
  uint32_t width;       // bytes per row
  uint32_t off;         // offset inside a warp's stage buffer (16-byte aligned)
  uint32_t tile_bytes;  // bytes one warp tile copies (Utf8: one extra offset, padded to 16)
  uint32_t utf8;
};
struct FusedFilter {
  uint32_t off;   // tile column offset inside the stage buffer
  uint8_t w;      // element width 4 / 8 / 16 (low word)
  uint8_t op;     // VOp compare
  uint8_t _pad[2];
  int64_t imm;
};
struct FusedProd {
  uint32_t a_off, b_off;
  uint8_t a_src;   // 0: tile column, 1: previous product
  uint8_t a_w, b_w;
  uint8_t kind;    // 0: a*(lit-b)  1: a*(lit+b)  2: a*b
  uint64_t lit_lo, lit_hi;
};
struct FusedKey {
  uint32_t off;
  uint8_t kind;    // 0: integer column, 1: short Utf8 packed as len<<shift | bytes
  uint8_t w;       // integer column: element width; packed: 4 = 32-bit image (shift 24, <= 3 bytes), 8 = 64-bit image
  uint8_t max_len, shift;
  const uint8_t* chars;
  const int32_t* offsets;  // packed keys: the column's Arrow offsets in global memory
  int64_t bias;    // added to integer keys (non-negative 32-bit image)
};
struct FusedAcc {
  uint32_t off;
  uint8_t src;     // 0: tile column, 1: product 0, 2: product 1, 3: constant one (COUNT)
  uint8_t w;
  uint8_t _pad[2];
};
struct FusedSpec {
  int32_t n_filters, n_prod, n_keys, n_acc;
  int32_t combine;  // 1: key image = k0 + k1 * 2^32
  int32_t n_cols;
  int32_t rows_per_thread;  // R: a warp tile is 32 * R rows
  int32_t n_stages;         // per-warp ring depth
  uint32_t stage_bytes;     // one warp stage
  uint32_t tile_tx;         // bytes one tile's bulk copies deliver (fixed-width columns)
  uint32_t tile_tx_utf8;    // ... plus the Utf8 offset slices, which belong to the warp's NEXT tile
  uint32_t use_tma;
  uint32_t acc_off;         // grouped shapes: byte offset of the [group][acc][thread] int64 partials
  FusedCol cols[FUSED_MAX_COLS];
  FusedFilter f[FUSED_MAX_FILTERS];
  FusedProd p[2];
  FusedKey k[2];
  FusedAcc a[VM_REG_ACC];
};

// Compile-time image of everything in a FusedSpec that changes the generated code (not offsets,
// pointers or literals).  (0, 0) means "not static: read the spec at run time".
struct FusedShape {
  uint64_t a, b;
};
#if defined(__CUDACC__)
#define B200_CX __host__ __device__
#else
#define B200_CX
#endif
B200_CX constexpr uint64_t fused_wcode(uint32_t w) { return w == 16 ? 2u : (w == 8 ? 1u : 0u); }
B200_CX constexpr uint32_t fused_wbytes(uint64_t c) { return c == 2 ? 16u : (c == 1 ? 8u : 4u); }
// layout of FusedShape::a : [0..2] n_filters | 6 x {w:2, op:3} from bit 3 | [33..34] n_keys | 2 x {kind:1, w:2} from
// bit 35 | [41] combine | [42..43] n_prod | 2 x {kind:2, a_src:1, a_w:2, b_w:2} from bit 44 | [63] static marker
// layout of FusedShape::b : [0..2] n_acc | 6 x {src:2, w:2} from bit 3
struct FusedShapeDesc {
  int nf;
  uint8_t fw[FUSED_MAX_FILTERS], fop[FUSED_MAX_FILTERS];  // fop: 0 EQ 1 NE 2 LT 3 LE 4 GT 5 GE
  int nk;
  uint8_t kkind[2], kw[2];
  int combine;
  int np;
  uint8_t pkind[2], pasrc[2], paw[2], pbw[2];
  int na;
  uint8_t asrc[VM_REG_ACC], aw[VM_REG_ACC];
};
B200_CX constexpr FusedShape fused_shape_encode(const FusedShapeDesc& d) {
  uint64_t a = (uint64_t)d.nf | (1ull << 63), b = (uint64_t)d.na;
  for (int i = 0; i < d.nf; i++) a |= (fused_wcode(d.fw[i]) | ((uint64_t)d.fop[i] << 2)) << (3 + 5 * i);
  a |= (uint64_t)d.nk << 33;
  for (int k = 0; k < d.nk; k++) a |= ((uint64_t)d.kkind[k] | (fused_wcode(d.kw[k]) << 1)) << (35 + 3 * k);
  a |= (uint64_t)(d.combine ? 1 : 0) << 41;
  a |= (uint64_t)d.np << 42;
  for (int j = 0; j < d.np; j++)
    a |= ((uint64_t)d.pkind[j] | ((uint64_t)d.pasrc[j] << 2) | ((d.pasrc[j] ? 0ull : fused_wcode(d.paw[j])) << 3) | (fused_wcode(d.pbw[j]) << 5)) << (44 + 7 * j);
  for (int i = 0; i < d.na; i++) b |= ((uint64_t)d.asrc[i] | ((d.asrc[i] == 0 ? fused_wcode(d.aw[i]) : 0ull) << 2)) << (3 + 4 * i);
  return FusedShape{a, b};
}

}  // namespace b200
