// Fused scan -> FilterExec -> ProjectionExec (decimal products) -> AggregateExec(Partial) kernel.
//
// Included by pipeline.cu (shares its __constant__ program, PTX wrappers and the group-table code).
// Reference operators replaced: the per-partition pipeline DataFusion builds for TPC-H q1/q6 inside
// ShuffleWriterExec's input (ballista/core/src/execution_plans/shuffle_writer.rs:150-260 drives it;
// the operators themselves are [EXT] datafusion FilterExec/ProjectionExec/AggregateExec).
//
// Design
//   * one CTA per SM, 16 warps; every WARP owns a private ring of S stage buffers in shared memory
//     and streams its own tiles (32*R rows) with 1-D TMA bulk copies signalled on per-warp
//     mbarriers.  There is no CTA-wide barrier on the data path: a warp only ever waits for its
//     own bytes.
//   * all arithmetic is in registers; aggregate partials are exact int64 per (group, accumulator)
//     per thread (|addend| < 2^40 checked per row, rare large addends go straight to the global
//     table), reduced over the CTA and merged into the global table once at the end.
//   * the code is compiled per FusedShape (program.h): widths, compare operators, product kinds and
//     accumulator sources are template constants for the listed shapes; shape (0,0) reads them from
//     constant memory so that any matching program still runs.
#pragma once

namespace b200 {

template <uint64_t SA, uint64_t SB>
struct FusedX {
  static constexpr bool ST = (SA >> 63) != 0;
  static __device__ __forceinline__ int nf() { return ST ? (int)(SA & 7) : c_fused.n_filters; }
  static __device__ __forceinline__ uint32_t fw(int i) { return ST ? fused_wbytes((SA >> (3 + 5 * i)) & 3) : (uint32_t)c_fused.f[i].w; }
  static __device__ __forceinline__ int fop(int i) { return ST ? (int)((SA >> (5 + 5 * i)) & 7) : (int)c_fused.f[i].op - (int)OP_CMP_EQ; }
  static __device__ __forceinline__ int nk() { return ST ? (int)((SA >> 33) & 3) : c_fused.n_keys; }
  static __device__ __forceinline__ int kkind(int k) { return ST ? (int)((SA >> (35 + 3 * k)) & 1) : (int)c_fused.k[k].kind; }
  static __device__ __forceinline__ uint32_t kw(int k) { return ST ? fused_wbytes((SA >> (36 + 3 * k)) & 3) : (uint32_t)c_fused.k[k].w; }
  static __device__ __forceinline__ bool combine() { return ST ? ((SA >> 41) & 1) != 0 : c_fused.combine != 0; }
  static __device__ __forceinline__ int np() { return ST ? (int)((SA >> 42) & 3) : c_fused.n_prod; }
  static __device__ __forceinline__ int pkind(int j) { return ST ? (int)((SA >> (44 + 7 * j)) & 3) : (int)c_fused.p[j].kind; }
  static __device__ __forceinline__ int pasrc(int j) { return ST ? (int)((SA >> (46 + 7 * j)) & 1) : (int)c_fused.p[j].a_src; }
  static __device__ __forceinline__ uint32_t paw(int j) { return ST ? fused_wbytes((SA >> (47 + 7 * j)) & 3) : (uint32_t)c_fused.p[j].a_w; }
  static __device__ __forceinline__ uint32_t pbw(int j) { return ST ? fused_wbytes((SA >> (49 + 7 * j)) & 3) : (uint32_t)c_fused.p[j].b_w; }
  static __device__ __forceinline__ int na() { return ST ? (int)(SB & 7) : c_fused.n_acc; }
  static __device__ __forceinline__ int asrc(int i) { return ST ? (int)((SB >> (3 + 4 * i)) & 3) : (int)c_fused.a[i].src; }
  static __device__ __forceinline__ uint32_t aw(int i) { return ST ? fused_wbytes((SB >> (5 + 4 * i)) & 3) : (uint32_t)c_fused.a[i].w; }
};

// One batch of bulk copies: the fixed-width columns of tile `row0` and -- software pipelining of the
// string keys -- the Utf8 offset slices of the warp's NEXT tile `row0n` (< 0: none).  Lane c issues
// column c (the whole warp takes part so that the address arithmetic is not a single-lane detour).
struct FusedLaneCol {  // lane c's column, read from constant memory once per kernel
  const uint8_t* data;
  uint32_t width, off, bytes, utf8;
};
__device__ __forceinline__ FusedLaneCol fused_lane_col(int lane) {
  const FusedSpec& F = c_fused;
  FusedLaneCol lc;
  const bool on = lane < F.n_cols;
  const FusedCol& fc = F.cols[on ? lane : 0];
  lc.data = (const uint8_t*)fc.data;
  lc.width = fc.width;
  lc.off = fc.off;
  lc.bytes = on ? fc.tile_bytes : 0u;
  lc.utf8 = fc.utf8;
  return lc;
}
__device__ __forceinline__ void fused_issue(uint8_t* stage, uint64_t* bar, int64_t row0, int64_t row0n, int lane, const FusedLaneCol& lc) {
  const FusedSpec& F = c_fused;
  if (lane == 0) mbar_expect_tx(bar, F.tile_tx + (row0n >= 0 ? F.tile_tx_utf8 : 0u));
  __syncwarp();
  const int64_t r0 = lc.utf8 ? row0n : row0;
  if (lc.bytes && r0 >= 0) bulk_g2s(stage + lc.off, lc.data + r0 * lc.width, lc.bytes, bar);
}

// ragged last tile / unaligned slices: the warp loads the fixed-width columns of its tile itself,
// zero fill past the end (string offsets are then read from global memory by fused_key_loads)
__device__ __noinline__ void fused_load_coop(uint8_t* stage, int64_t row0, int rows, int tile_rows, int lane) {
  const FusedSpec& F = c_fused;
  const int n = F.n_cols;
  for (int c = 0; c < n; c++) {
    const FusedCol& fc = F.cols[c];
    if (fc.utf8) continue;
    uint8_t* dst = stage + fc.off;
    const uint8_t* src = (const uint8_t*)fc.data + row0 * fc.width;
    const uint32_t nb = (uint32_t)rows * fc.width, tb = (uint32_t)tile_rows * fc.width;
    if ((fc.width & 3) == 0 && (((uintptr_t)src) & 3) == 0) {
      const uint32_t* s4 = (const uint32_t*)src;
      uint32_t* d4 = (uint32_t*)dst;
      for (uint32_t k = lane; k < tb / 4; k += 32) d4[k] = (k * 4 < nb) ? s4[k] : 0u;
    } else {
      for (uint32_t k = lane; k < tb; k += 32) dst[k] = (k < nb) ? src[k] : 0;
    }
  }
}

__device__ __forceinline__ bool fused_cmp(int fop, int64_t v, int64_t imm) {
  switch (fop) {
    case 0: return v == imm;
    case 1: return v != imm;
    case 2: return v < imm;
    case 3: return v <= imm;
    case 4: return v > imm;
    default: return v >= imm;
  }
}

// |v| < 2^40 test: returns bits that are non-zero iff (lo, hi) is NOT a small value.  A thread adds
// at most 2^22 small addends into an int64 partial (fused_rows_ok), so the partials are exact.
__device__ __forceinline__ uint64_t fused_range_bits(uint64_t lo, uint64_t hi) {
  const uint64_t s = (uint64_t)((int64_t)hi >> 63);
  return (hi ^ s) | ((lo ^ s) >> 40);
}

// ------------------------------------------------------------------------------------------------
// One row, every exceptional case, out of line and shape-agnostic (reads the spec at run time):
// operands wider than 64 bits, literal +- operand overflow, keys longer than the packed image,
// a group this thread has not cached yet, addends >= 2^40.  Returns 1 when the row takes part in
// the aggregate; then *gid_out is its group and out_add[] its int64 addends (0 for addends that
// were merged straight into the global table).
// ------------------------------------------------------------------------------------------------
__device__ __noinline__ uint32_t fused_row_slow(const uint8_t* stage, int e, int64_t row0, int G, RegGroupTable* gt, uint64_t* out_add, uint32_t* gid_out) {
  const FusedSpec& F = c_fused;
  for (int i = 0; i < F.n_filters; i++) {
    const int64_t v = ld_w(stage + F.f[i].off, F.f[i].w, e);
    if (!fused_cmp((int)F.f[i].op - (int)OP_CMP_EQ, v, F.f[i].imm)) return 0;
  }
  i128 prod[2] = {0, 0};
  for (int j = 0; j < F.n_prod; j++) {
    const FusedProd& q = F.p[j];
    i128 a = (j == 1 && q.a_src) ? prod[0] : ld_w128(stage + q.a_off, q.a_w, e);
    i128 b = ld_w128(stage + q.b_off, q.b_w, e);
    const i128 lit = make_i128(q.lit_lo, q.lit_hi);
    bool ovf = false;
    if (q.kind == 0) ovf = sub_i128_checked(lit, b, &b);
    else if (q.kind == 1) ovf = add_i128_checked(lit, b, &b);
    i128 out = 0;
    ovf |= mul_i128_slow(a, b, &out);
    if (ovf) raise(1);
    prod[j] = out;
  }
  uint32_t g = 0;
  if (G > 1) {
    unsigned long long kv[2] = {0, 0};
    for (int k = 0; k < F.n_keys; k++) {
      const FusedKey& fk = F.k[k];
      if (fk.kind == 1) {
        const int32_t* off = fk.offsets + row0;  // the stage holds the NEXT tile's offsets
        const int32_t o0 = off[e];
        uint32_t len = (uint32_t)(off[e + 1] - o0);
        if (len > fk.max_len) {
          atomicExch(&PROG.status->pack_overflow, 1u);  // the host re-runs with a wider key image
          len = 0;
        }
        unsigned long long v = 0;
        for (uint32_t c = 0; c < len; c++) v |= (unsigned long long)fk.chars[o0 + c] << (8 * c);
        kv[k] = len ? (v | ((unsigned long long)len << fk.shift)) : 0ull;
      } else {
        kv[k] = (unsigned long long)ld_w(stage + fk.off, fk.w, e);
      }
    }
    const unsigned long long ck = F.combine ? ((kv[0] + (unsigned long long)F.k[0].bias) + (kv[1] + (unsigned long long)F.k[1].bias) * 4294967296ull) : kv[0];
    const int gg = fused_resolve_slow(gt, G, F.n_keys, ck, kv[0], kv[1]);
    if (gg < 0) {
      atomicExch(&PROG.status->overflow, 1u);
      return 0;
    }
    g = (uint32_t)gg;
  }
  *gid_out = g;
  for (int a = 0; a < F.n_acc; a++) {
    const FusedAcc& fa = F.a[a];
    i128 v = fa.src == 3 ? (i128)1 : fa.src == 1 ? prod[0] : fa.src == 2 ? prod[1] : ld_w128(stage + fa.off, fa.w, e);
    if (fused_range_bits(lo64(v), hi64(v))) {
      reg_merge_big(gt, G, (int)g, a, v);
      v = 0;
    }
    out_add[a] = lo64(v);
  }
  return 1;
}

// 64x64 -> 128 signed product without branches (operands already known to fit 64 bits)
__device__ __forceinline__ void fused_mul64(uint64_t a, uint64_t b, uint64_t& lo, uint64_t& hi) {
  lo = a * b;
  hi = __umul64hi(a, b) - (((int64_t)a < 0) ? b : 0ull) - (((int64_t)b < 0) ? a : 0ull);
}
__device__ __forceinline__ uint32_t fused_wide(uint64_t lo, uint64_t hi) {  // non-zero iff (lo, hi) does not fit int64
  const uint64_t d = hi ^ (uint64_t)((int64_t)lo >> 63);
  return (uint32_t)d | (uint32_t)(d >> 32);
}

// ---- string keys, software-pipelined one tile ahead -------------------------------------------------
// fused_key_loads (start of the iteration that processes the PREVIOUS tile): offsets of the rows,
// then the dependent chars loads (aligned words; allocations carry slack).  fused_key_finish (end of
// that iteration, a whole tile's arithmetic later): the packed images.  Two widths: kw == 4:
// len<<24 | <=3 bytes (32-bit arithmetic, funnel shift), kw == 8: len<<shift | <=7 bytes.
template <int R, class X>
__device__ __forceinline__ void fused_key_loads(const uint8_t* stage /* null: offsets from global */, int64_t row0, int lim, int lane, uint32_t (&klen)[2][R],
                                                uint32_t (&ksh)[2][R], uint64_t (&kw0)[2][R], uint64_t (&kw1)[2][R], uint32_t& kslow) {
  const FusedSpec& F = c_fused;
  kslow = 0;
#pragma unroll
  for (int k = 0; k < 2; k++) {
#pragma unroll
    for (int r = 0; r < R; r++) {
      klen[k][r] = 0;
      ksh[k][r] = 0;
      kw0[k][r] = kw1[k][r] = 0;
    }
    if (k >= X::nk() || X::kkind(k) != 1) continue;
    const FusedKey& fk = F.k[k];
    const int32_t* off = stage ? (const int32_t*)(stage + fk.off) : fk.offsets + row0;
    const uint8_t* chars = fk.chars;
    const uint32_t max_len = fk.max_len;
    const bool short4 = X::kw(k) == 4;
#pragma unroll
    for (int r = 0; r < R; r++) {
      const int e = lane + 32 * r;
      const int32_t o0 = off[min(e, lim)];
      const uint32_t len = (uint32_t)(off[min(e + 1, lim)] - o0);
      kslow |= (len > max_len ? 1u : 0u) << r;
      const uint8_t* p = chars + o0;
      klen[k][r] = len;
      if (short4) {
        const uint32_t* base = (const uint32_t*)((uintptr_t)p & ~(uintptr_t)3);
        ksh[k][r] = (uint32_t)((uintptr_t)p & 3) * 8;
        kw0[k][r] = base[0];
        kw1[k][r] = base[1];
      } else {
        const uint64_t* base = (const uint64_t*)((uintptr_t)p & ~(uintptr_t)7);
        ksh[k][r] = (uint32_t)((uintptr_t)p & 7) * 8;
        kw0[k][r] = base[0];
        kw1[k][r] = base[1];
      }
    }
  }
}
template <int R, class X>
__device__ __forceinline__ void fused_key_finish(const uint32_t (&klen)[2][R], const uint32_t (&ksh)[2][R], const uint64_t (&kw0)[2][R], const uint64_t (&kw1)[2][R],
                                                 uint64_t (&kv)[2][R]) {
  const FusedSpec& F = c_fused;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const bool packed = k < X::nk() && X::kkind(k) == 1;
    const bool short4 = packed && X::kw(k) == 4;
    const int shift = F.k[k].shift;
#pragma unroll
    for (int r = 0; r < R; r++) {
      uint64_t v = 0;
      if (short4) {
        const uint32_t len = klen[k][r];
        const uint32_t x = __funnelshift_r((uint32_t)kw0[k][r], (uint32_t)kw1[k][r], ksh[k][r]);
        v = (uint64_t)((x & ((1u << ((len * 8) & 31)) - 1u)) | (len << 24));
      } else if (packed) {
        const uint32_t len = klen[k][r], sh = ksh[k][r];
        uint64_t w = kw0[k][r] >> sh;
        if (sh) w |= kw1[k][r] << ((64 - sh) & 63);
        w &= (1ull << ((len * 8) & 63)) - 1;
        v = len ? (w | ((uint64_t)len << shift)) : 0ull;
      }
      kv[k][r] = v;
    }
  }
}

// add the tile's addends to the per-thread partials
template <int G, int R, class X>
__device__ __forceinline__ void fused_accumulate(const uint32_t active, const uint32_t (&gid)[R], const uint64_t (&add)[VM_REG_ACC][R], RegAggState<G>& S, uint64_t* accs,
                                                 const int B) {
  if (G == 1) {
    // scalar aggregate: the partials live in registers
#pragma unroll
    for (int r = 0; r < R; r++) {
      const uint64_t m = ((active >> r) & 1) ? ~0ull : 0ull;
#pragma unroll
      for (int a = 0; a < VM_REG_ACC; a++)
        if (a < X::na()) S.lo[0][a] += add[a][r] & m;
    }
  } else {
    // grouped aggregate: per-thread partials in shared memory, [group][acc][thread] (conflict-free),
    // indexed by the row's group -- no G-fold work and no accumulator registers
#pragma unroll
    for (int r = 0; r < R; r++) {
      if ((active >> r) & 1) {
        uint64_t* pa = accs + (size_t)gid[r] * (VM_REG_ACC * B);
#pragma unroll
        for (int a = 0; a < VM_REG_ACC; a++)
          if (a < X::na()) pa[a * B] += add[a][r];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Speculative narrow path.  Money columns are Decimal128 in Arrow but their values almost always fit
// 31 bits; then a*(lit-b) is one 32x32->64 multiply instead of checked 128-bit arithmetic.  The
// function computes the whole tile in 32/64-bit arithmetic WITHOUT side effects and reports whether
// every active row of this thread stayed inside the assumptions (operands in [0, 2^31), literal
// differences non-negative, products and addends < 2^40, key cached, key short enough).  If any lane
// of the warp says no, the warp redoes the tile with fused_rows (general, exact for everything).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t fused_ld_narrow(const uint8_t* base, uint32_t w, int e, uint32_t& bad) {
  if (w == 16) {
    const uint4 v = ((const uint4*)base)[e];
    bad |= v.y | v.z | v.w | (v.x & 0x80000000u);
    return v.x;
  }
  if (w == 8) {
    const uint2 v = ((const uint2*)base)[e];
    bad |= v.y | (v.x & 0x80000000u);
    return v.x;
  }
  const uint32_t v = ((const uint32_t*)base)[e];
  bad |= v & 0x80000000u;
  return v;
}

template <int G, int R, class X>
__device__ __forceinline__ bool fused_try_narrow(const uint8_t* __restrict__ stage, const int lane, uint32_t& active_io, uint32_t (&gid)[R],
                                                 uint64_t (&add)[VM_REG_ACC][R], const unsigned long long (&dir)[G], const uint32_t dir_n,
                                                 const uint64_t (&kvs)[2][R], const uint32_t kslow) {
  const FusedSpec& F = c_fused;
  uint32_t active = active_io;
  uint32_t bad[R];
#pragma unroll
  for (int r = 0; r < R; r++) bad[r] = (kslow >> r) & 1;
  // ---- group resolution against the register-cached directory
#pragma unroll
  for (int r = 0; r < R; r++) gid[r] = 0;
  if (G > 1) {
    unsigned long long kv0[R], kv1[R];
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const bool intkey = k < X::nk() && X::kkind(k) == 0;
      const uint8_t* p = stage + F.k[k].off;
      const uint32_t w = X::kw(k);
#pragma unroll
      for (int r = 0; r < R; r++) {
        const unsigned long long v = intkey ? (unsigned long long)ld_w(p, w, lane + 32 * r) : kvs[k][r];
        if (k == 0) kv0[r] = v;
        else kv1[r] = v;
      }
    }
    const unsigned long long bias0 = (unsigned long long)F.k[0].bias, bias1 = (unsigned long long)F.k[1].bias;
    const bool combine = X::combine();
#pragma unroll
    for (int r = 0; r < R; r++) {
      const unsigned long long ck = combine ? ((kv0[r] + bias0) + (kv1[r] + bias1) * 4294967296ull) : kv0[r];
      uint32_t g = 0, hit = 0;
#pragma unroll
      for (int q = 0; q < G; q++) {
        const bool m = q < (int)dir_n && dir[q] == ck;
        g = m ? (uint32_t)q : g;
        hit |= m ? 1u : 0u;
      }
      gid[r] = g;
      bad[r] |= hit ^ 1u;
    }
  }
  // ---- filters
#pragma unroll
  for (int i = 0; i < FUSED_MAX_FILTERS; i++) {
    if (i >= X::nf()) break;
    const uint8_t* p = stage + F.f[i].off;
    const uint32_t w = X::fw(i);
    const int fop = X::fop(i);
    const int64_t imm = F.f[i].imm;
    uint32_t pass = 0;
#pragma unroll
    for (int r = 0; r < R; r++) pass |= (fused_cmp(fop, ld_w(p, w, lane + 32 * r), imm) ? 1u : 0u) << r;
    active &= pass;
  }
  // ---- products in 32x32->64 / 64x32->96 bit arithmetic
  uint64_t prod0[R], prod1[R];
#pragma unroll
  for (int r = 0; r < R; r++) prod0[r] = prod1[r] = 0;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    if (j >= X::np()) break;
    const FusedProd& q = F.p[j];
    const uint8_t* pa = stage + q.a_off;
    const uint8_t* pb = stage + q.b_off;
    const uint32_t aw = X::paw(j), bw = X::pbw(j);
    const int kind = X::pkind(j);
    const bool a_prev = j == 1 && X::pasrc(j) != 0;
    const uint32_t lit = (uint32_t)q.lit_lo;
    const uint32_t lit_bad = (kind != 2 && (q.lit_hi != 0 || q.lit_lo >= 0x80000000ull)) ? 1u : 0u;
#pragma unroll
    for (int r = 0; r < R; r++) {
      const int e = lane + 32 * r;
      const uint32_t b = fused_ld_narrow(pb, bw, e, bad[r]);
      const uint32_t m = kind == 0 ? lit - b : kind == 1 ? lit + b : b;
      if (kind == 0) bad[r] |= m & 0x80000000u;
      bad[r] |= lit_bad;
      uint64_t pr;
      if (a_prev) {
        // prod0 < 2^40 on rows that are still good: 64 x 32 -> bits 0..95, must stay below 2^40
        const uint64_t lo = (uint64_t)(uint32_t)prod0[r] * m;
        const uint64_t hi = (uint64_t)(uint32_t)(prod0[r] >> 32) * m + (lo >> 32);
        bad[r] |= (uint32_t)(hi >> 8) | (uint32_t)(hi >> 32);
        pr = (hi << 32) | (uint32_t)lo;
      } else {
        const uint32_t a = fused_ld_narrow(pa, aw, e, bad[r]);
        pr = (uint64_t)a * m;
        bad[r] |= (uint32_t)(pr >> 40);
      }
      if (j == 0) prod0[r] = pr;
      else prod1[r] = pr;
    }
  }
  // ---- addends
#pragma unroll
  for (int a = 0; a < VM_REG_ACC; a++) {
#pragma unroll
    for (int r = 0; r < R; r++) add[a][r] = 0;
    if (a >= X::na()) continue;
    const int src = X::asrc(a);
#pragma unroll
    for (int r = 0; r < R; r++) {
      if (src == 3) add[a][r] = 1;
      else if (src == 1) add[a][r] = prod0[r];
      else if (src == 2) add[a][r] = prod1[r];
      else add[a][r] = (uint64_t)fused_ld_narrow(stage + F.a[a].off, X::aw(a), lane + 32 * r, bad[r]);
    }
  }
  uint32_t any_bad = 0;
#pragma unroll
  for (int r = 0; r < R; r++) any_bad |= ((active >> r) & 1) ? bad[r] : 0u;
  active_io = active;
  return any_bad == 0;
}

// Hot path: straight-line code for the tile's R rows per thread.  Anything unusual about a row only
// sets its bit in `slow`; those rows are redone by fused_row_slow afterwards.  kvs/kslow: the packed
// string-key images of this tile, prepared during the previous iteration.
template <int G, int R, class X>
__device__ __forceinline__ uint32_t fused_rows(const uint8_t* __restrict__ stage, const int64_t row0, const int lane, uint32_t active, RegAggState<G>& S,
                                               uint64_t* accs, const int B, RegGroupTable* gt, unsigned long long (&dir)[G], uint32_t& dir_n,
                                               const uint64_t (&kvs)[2][R], const uint32_t kslow) {
  const FusedSpec& F = c_fused;
  uint32_t slow = kslow;
  // ---- filters
#pragma unroll
  for (int i = 0; i < FUSED_MAX_FILTERS; i++) {
    if (i >= X::nf()) break;
    const uint8_t* p = stage + F.f[i].off;
    const uint32_t w = X::fw(i);
    const int fop = X::fop(i);
    const int64_t imm = F.f[i].imm;
    uint32_t pass = 0;
#pragma unroll
    for (int r = 0; r < R; r++) pass |= (fused_cmp(fop, ld_w(p, w, lane + 32 * r), imm) ? 1u : 0u) << r;
    active &= pass;
  }
  // ---- products: operands that fit 64 bits multiply inline; wider ones mark the row slow
  uint64_t p0lo[R], p0hi[R], p1lo[R], p1hi[R];
#pragma unroll
  for (int r = 0; r < R; r++) p0lo[r] = p0hi[r] = p1lo[r] = p1hi[r] = 0;
  if (X::np() >= 1) {
    const FusedProd& q = F.p[0];
    const uint8_t* pa = stage + q.a_off;
    const uint8_t* pb = stage + q.b_off;
    const uint32_t aw = X::paw(0), bw = X::pbw(0);
    const int kind = X::pkind(0);
    const uint64_t llo = q.lit_lo, lhi = q.lit_hi;
#pragma unroll
    for (int r = 0; r < R; r++) {
      uint64_t alo, ahi, blo, bhi;
      ld_raw128(pa, aw, lane + 32 * r, alo, ahi);
      ld_raw128(pb, bw, lane + 32 * r, blo, bhi);
      uint32_t odd = 0;
      if (kind != 2) odd = addsub128(kind == 0, llo, lhi, blo, bhi);
      if (aw == 16) odd |= fused_wide(alo, ahi);
      if (bw == 16 || kind != 2) odd |= fused_wide(blo, bhi);
      slow |= (odd ? 1u : 0u) << r;
      fused_mul64(alo, blo, p0lo[r], p0hi[r]);
    }
  }
  if (X::np() >= 2) {
    const FusedProd& q = F.p[1];
    const uint8_t* pa = stage + q.a_off;
    const uint8_t* pb = stage + q.b_off;
    const uint32_t aw = X::paw(1), bw = X::pbw(1);
    const int kind = X::pkind(1), a_src = X::pasrc(1);
    const uint64_t llo = q.lit_lo, lhi = q.lit_hi;
#pragma unroll
    for (int r = 0; r < R; r++) {
      uint64_t alo = p0lo[r], ahi = p0hi[r], blo, bhi;
      if (!a_src) ld_raw128(pa, aw, lane + 32 * r, alo, ahi);
      ld_raw128(pb, bw, lane + 32 * r, blo, bhi);
      uint32_t odd = 0;
      if (kind != 2) odd = addsub128(kind == 0, llo, lhi, blo, bhi);
      if (a_src || aw == 16) odd |= fused_wide(alo, ahi);
      if (bw == 16 || kind != 2) odd |= fused_wide(blo, bhi);
      slow |= (odd ? 1u : 0u) << r;
      fused_mul64(alo, blo, p1lo[r], p1hi[r]);
    }
  }
  // ---- group resolution against the register-cached directory
  uint32_t gid[R];
#pragma unroll
  for (int r = 0; r < R; r++) gid[r] = 0;
  if (G > 1) {
    unsigned long long kv0[R], kv1[R];
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const bool intkey = k < X::nk() && X::kkind(k) == 0;
      const uint8_t* p = stage + F.k[k].off;
      const uint32_t w = X::kw(k);
#pragma unroll
      for (int r = 0; r < R; r++) {
        const unsigned long long v = intkey ? (unsigned long long)ld_w(p, w, lane + 32 * r) : kvs[k][r];
        if (k == 0) kv0[r] = v;
        else kv1[r] = v;
      }
    }
    const unsigned long long bias0 = (unsigned long long)F.k[0].bias, bias1 = (unsigned long long)F.k[1].bias;
    const bool combine = X::combine();
#pragma unroll
    for (int r = 0; r < R; r++) {
      const unsigned long long ck = combine ? ((kv0[r] + bias0) + (kv1[r] + bias1) * 4294967296ull) : kv0[r];
      uint32_t g = 0, hit = 0;
#pragma unroll
      for (int q = 0; q < G; q++) {
        const bool m = q < (int)dir_n && dir[q] == ck;
        g = m ? (uint32_t)q : g;
        hit |= m ? 1u : 0u;
      }
      gid[r] = g;
      slow |= (hit ^ 1u) << r;
    }
  }
  // ---- addends (exact int64 partials); anything >= 2^40 in magnitude marks the row slow
  uint64_t add[VM_REG_ACC][R];
#pragma unroll
  for (int a = 0; a < VM_REG_ACC; a++) {
#pragma unroll
    for (int r = 0; r < R; r++) add[a][r] = 0;
    if (a >= X::na()) continue;
    const int src = X::asrc(a);
    if (src == 3) {  // COUNT
#pragma unroll
      for (int r = 0; r < R; r++) add[a][r] = 1;
      continue;
    }
    uint64_t vhi[R];
    const uint32_t w = (src == 0) ? X::aw(a) : 16u;
    if (src == 1) {
#pragma unroll
      for (int r = 0; r < R; r++) {
        add[a][r] = p0lo[r];
        vhi[r] = p0hi[r];
      }
    } else if (src == 2) {
#pragma unroll
      for (int r = 0; r < R; r++) {
        add[a][r] = p1lo[r];
        vhi[r] = p1hi[r];
      }
    } else {
      const uint8_t* p = stage + F.a[a].off;
#pragma unroll
      for (int r = 0; r < R; r++) ld_raw128(p, w, lane + 32 * r, add[a][r], vhi[r]);
    }
    if (w != 4) {
#pragma unroll
      for (int r = 0; r < R; r++) slow |= (fused_range_bits(add[a][r], vhi[r]) ? 1u : 0u) << r;
    }
  }
  // ---- the unusual rows (none in steady state), one at a time
  slow &= active;
  if (slow) {
#pragma unroll
    for (int r = 0; r < R; r++) {
      if ((slow >> r) & 1) {
        uint64_t out[VM_REG_ACC];
        uint32_t g = 0;
        const uint32_t on = fused_row_slow(stage, lane + 32 * r, row0, G, gt, out, &g);
        if (!on) active &= ~(1u << r);
        gid[r] = g;
#pragma unroll
        for (int a = 0; a < VM_REG_ACC; a++) add[a][r] = out[a];
      }
    }
    if (G > 1) {  // pick up the groups published so far
      uint32_t pub = 0;
#pragma unroll
      for (int q = 0; q < G; q++) {
        const bool ok = (q == (int)pub) && (*(volatile unsigned int*)&gt->state[q] == 2u);
        if (ok) {
          dir[q] = *(volatile unsigned long long*)&gt->hash[q];
          pub++;
        }
      }
      dir_n = pub;
    }
  }
  fused_accumulate<G, R, X>(active, gid, add, S, accs, B);
  return active;
}

// The general path as a real call for grouped shapes, so that its register appetite (checked 128-bit
// arithmetic for R rows) does not dictate the allocation of the speculative path around it.  The
// caller's register-resident directory travels by value.
template <int G, int R>
struct FusedGeneralIO {
  uint32_t active, dir_n, kslow, _pad;
  unsigned long long dir[G];
  uint64_t kvs[2][R];
};
template <int G, int R, class X>
__device__ __noinline__ FusedGeneralIO<G, R> fused_rows_call(const uint8_t* stage, const int64_t row0, const int lane, uint64_t* accs, const int B, RegGroupTable* gt,
                                                              FusedGeneralIO<G, R> io) {
  RegAggState<G> unused;  // grouped partials live in shared memory
  io.active = fused_rows<G, R, X>(stage, row0, lane, io.active, unused, accs, B, gt, io.dir, io.dir_n, io.kvs, io.kslow);
  return io;
}

template <int G, int R, int BT, uint64_t SA, uint64_t SB>
__global__ void __launch_bounds__(BT, 1) fused_kernel() {
  typedef FusedX<SA, SB> X;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bars[FUSED_MAX_WARPS * FUSED_MAX_STAGES];
  __shared__ uint32_t stage_tile[FUSED_MAX_WARPS * FUSED_MAX_STAGES];  // tile held by each (warp, stage)
  __shared__ uint32_t stage_next[FUSED_MAX_WARPS * FUSED_MAX_STAGES];  // ... and the warp's following tile
  __shared__ unsigned int next_claim;                                   // CTA-wide tile dispenser
  __shared__ RegGroupTable gtable;
  const FusedSpec& F = c_fused;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, B = blockDim.x;
  constexpr int TR = 32 * R;
  const int64_t n_rows = PROG.n_rows;
  const uint32_t n_tiles = (uint32_t)((n_rows + TR - 1) / TR);      // host guarantees < 2^31
  const uint32_t n_full = F.use_tma ? (uint32_t)(n_rows / TR) : 0u;  // tiles below n_full arrive by TMA
  const int S = F.n_stages;
  const uint32_t stage_bytes = F.stage_bytes;
  uint8_t* ring = smem + (size_t)warp * S * stage_bytes;
  uint64_t* bar = bars + warp * FUSED_MAX_STAGES;
  uint32_t* my_tile = stage_tile + warp * FUSED_MAX_STAGES;
  if (lane == 0) {
    for (int s = 0; s < S; s++) mbar_init(&bar[s], 1);
    mbar_fence_init();
  }
  if (tid == 0) next_claim = 0;
  if (tid < VM_REG_GROUPS) {
    gtable.state[tid] = 0;
    gtable.hash[tid] = 0;
    if (tid == 0) gtable.n_groups = 0;
  }
  __syncthreads();

  RegAggState<G> S_reg;
#pragma unroll
  for (int g = 0; g < G; g++) {
#pragma unroll
    for (int a = 0; a < VM_REG_ACC; a++) S_reg.lo[g][a] = 0;
  }
  // grouped shapes keep the per-thread partials in shared memory behind the rings
  uint64_t* accs = (uint64_t*)(smem + F.acc_off) + tid;
  if (G > 1) {
    for (int i = 0; i < G * VM_REG_ACC; i++) accs[i * B] = 0;
  }
  unsigned long long dir[G];
  uint32_t dir_n = 0;
#pragma unroll
  for (int q = 0; q < G; q++) dir[q] = 0xFFFFFFFFFFFFFFFFull;
  uint32_t live_rows = 0;

  // Warp tiles are claimed dynamically from a CTA-wide counter (warps of one CTA do not run at the
  // same speed; a static deal leaves the fast ones idle at the end): the c-th claim of CTA b is
  // tile c * gridDim.x + b, so the grid sweeps the table front to back.  Every batch also carries
  // the string offsets of the warp's following tile, so claims run one tile ahead of the issues.
  uint32_t* my_next = stage_next + warp * FUSED_MAX_STAGES;
  auto claim = [&]() -> uint32_t {
    unsigned int c = 0;
    if (lane == 0) c = atomicAdd(&next_claim, 1u);
    c = __shfl_sync(0xFFFFFFFFu, c, 0);
    const unsigned long long t64 = (unsigned long long)c * gridDim.x + blockIdx.x;
    return t64 < n_tiles ? (uint32_t)t64 : 0xFFFFFFFFu;
  };
  const FusedLaneCol lane_col = fused_lane_col(lane);
  uint32_t ahead = claim();
  const uint32_t first = ahead;
  auto issue_into = [&](int st) {
    const uint32_t cur = ahead;
    if (cur != 0xFFFFFFFFu) ahead = claim();
    if (lane == 0) {
      my_tile[st] = cur;
      my_next[st] = ahead;
    }
    if (cur < n_full) fused_issue(ring + (size_t)st * stage_bytes, &bar[st], (int64_t)cur * TR, ahead < n_full ? (int64_t)ahead * TR : -1, lane, lane_col);
  };
  for (int k = 0; k < S - 1; k++) issue_into(k);
  // string keys of the first tile: straight from global memory (the only exposed latency)
  uint64_t kv_cur[2][R];
  uint32_t kslow_cur = 0;
  {
    uint32_t klen[2][R], ksh[2][R];
    uint64_t kw0[2][R], kw1[2][R];
    const int64_t r0 = first != 0xFFFFFFFFu ? (int64_t)first * TR : 0;
    const int lim = first != 0xFFFFFFFFu ? (int)((n_rows - r0) < TR ? (n_rows - r0) : TR) : 0;
    if (G > 1) fused_key_loads<R, X>(nullptr, r0, lim, lane, klen, ksh, kw0, kw1, kslow_cur);
    fused_key_finish<R, X>(klen, ksh, kw0, kw1, kv_cur);
  }
  uint32_t phase_bits = 0;
  int s = 0;
  uint32_t it = 0;
  for (;; s = (s + 1 == S) ? 0 : s + 1, it++) {
    uint8_t* stage = ring + (size_t)s * stage_bytes;
    // every lane is done with the buffer consumed in the previous iteration: refill it
    __syncwarp();
    issue_into((s == 0) ? S - 1 : s - 1);
    __syncwarp();
    const uint32_t t = my_tile[s], tn = my_next[s];
    if (t == 0xFFFFFFFFu) break;  // claims are monotonic: nothing of this warp is in flight any more
    // the sink-overflow flag (another CTA met a 5th group, ...) is polled every 8th tile; all lanes
    // read the same word, the value is consumed at the end of the tile
    unsigned int stop = 0;
    const bool poll = (it & 7u) == 7u;
    if (poll) stop = *(volatile unsigned int*)&PROG.status->overflow;
    const int64_t row0 = (int64_t)t * TR;
    const int rows = (int)((n_rows - row0) < TR ? (n_rows - row0) : TR);
    if (t < n_full) {
      mbar_wait(&bar[s], (phase_bits >> s) & 1);
      phase_bits ^= 1u << s;
    } else {
      fused_load_coop(stage, row0, rows, TR, lane);
      __syncwarp();
    }
    // string keys of the NEXT tile: issue the loads now, finish them after this tile's arithmetic
    uint32_t klen[2][R], ksh[2][R];
    uint64_t kw0[2][R], kw1[2][R];
    uint32_t kslow_next = 0;
    if (G > 1) {
      const bool in_stage = t < n_full && tn < n_full;  // the batch carried the next tile's offsets
      const int64_t rn = tn != 0xFFFFFFFFu ? (int64_t)tn * TR : 0;
      const int limn = tn != 0xFFFFFFFFu ? (int)((n_rows - rn) < TR ? (n_rows - rn) : TR) : 0;
      fused_key_loads<R, X>(in_stage ? stage : nullptr, rn, limn, lane, klen, ksh, kw0, kw1, kslow_next);
    }
    uint32_t active = 0;
#pragma unroll
    for (int r = 0; r < R; r++)
      if (lane + 32 * r < rows) active |= 1u << r;
    {
      uint32_t gid[R];
      uint64_t add[VM_REG_ACC][R];
      uint32_t act = active;
      const bool ok = fused_try_narrow<G, R, X>(stage, lane, act, gid, add, dir, dir_n, kv_cur, kslow_cur);
      if (__all_sync(0xFFFFFFFFu, ok)) {
        active = act;
        fused_accumulate<G, R, X>(active, gid, add, S_reg, accs, B);
      } else if (G == 1) {
        active = fused_rows<G, R, X>(stage, row0, lane, active, S_reg, accs, B, &gtable, dir, dir_n, kv_cur, kslow_cur);
      } else {
        FusedGeneralIO<G, R> io;
        io.active = active;
        io.dir_n = dir_n;
        io.kslow = kslow_cur;
#pragma unroll
        for (int q = 0; q < G; q++) io.dir[q] = dir[q];
#pragma unroll
        for (int k = 0; k < 2; k++) {
#pragma unroll
          for (int r = 0; r < R; r++) io.kvs[k][r] = kv_cur[k][r];
        }
        io = fused_rows_call<G, R, X>(stage, row0, lane, accs, B, &gtable, io);
        active = io.active;
        dir_n = io.dir_n;
#pragma unroll
        for (int q = 0; q < G; q++) dir[q] = io.dir[q];
      }
    }
    live_rows += __popc(active);
    if (G > 1) {
      fused_key_finish<R, X>(klen, ksh, kw0, kw1, kv_cur);
      kslow_cur = kslow_next;
    }
    if (poll && stop) {
      __syncwarp();
      int sj = s;
      for (int j = 1; j < S; j++) {  // drain bulk copies still in flight before the CTA may exit
        sj = (sj + 1 == S) ? 0 : sj + 1;
        if (my_tile[sj] < n_full) mbar_wait(&bar[sj], (phase_bits >> sj) & 1);
      }
      break;
    }
  }
  live_rows = __reduce_add_sync(0xFFFFFFFFu, live_rows);
  if (lane == 0 && live_rows) atomicAdd(&PROG.status->in_active, (unsigned long long)live_rows);
  if (G > 1) {
#pragma unroll
    for (int g = 0; g < G; g++) {
#pragma unroll
      for (int a = 0; a < VM_REG_ACC; a++) S_reg.lo[g][a] = accs[(g * VM_REG_ACC + a) * B];
    }
  }
  __syncthreads();
  // scalar aggregates emit their single group even when no CTA saw a row: CTA 0 always flushes
  const bool has_rows = blockIdx.x < n_tiles;
  if (has_rows || (G == 1 && blockIdx.x == 0)) reg_agg_flush<G, true>(S_reg, nullptr, &gtable, (Acc128*)smem, tid, B);
}

template <int G, int R, int BT, uint64_t SA, uint64_t SB>
static cudaError_t launch_fused_one(int grid, int block, size_t smem, cudaStream_t st) {
  if (block > BT) return cudaErrorInvalidValue;
  cudaError_t e = cudaFuncSetAttribute(fused_kernel<G, R, BT, SA, SB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  launch_kernel(fused_kernel<G, R, BT, SA, SB>, grid, block, smem, st);
  return cudaGetLastError();
}

// ---- shapes compiled ahead of time -----------------------------------------------------------------
// TPC-H q1 (benchmarks/queries/q1.sql): 1 date filter, 2 packed single-character keys,
// disc_price = price*(1-disc), charge = disc_price*(1+tax); count + 4 decimal sums + sum(disc)
constexpr FusedShapeDesc kShapeQ1 = {1, {4}, {3 /*LE*/}, 2, {1, 1}, {4, 4}, 1, 2, {0, 1}, {0, 1}, {16, 0}, {16, 16}, 6,
                                     {3, 0, 0, 1, 2, 0}, {0, 16, 16, 0, 0, 16}};
// TPC-H q6 (benchmarks/queries/q6.sql): date range, discount BETWEEN, quantity <; count + sum(price*disc)
constexpr FusedShapeDesc kShapeQ6 = {5, {4, 4, 16, 16, 16}, {5 /*GE*/, 2 /*LT*/, 5, 3 /*LE*/, 2}, 0, {0, 0}, {0, 0}, 0, 1, {2, 0}, {0, 0}, {16, 0}, {16, 0}, 2,
                                     {3, 1}, {0, 0}};
// the same query when the two key columns carry pre-packed 4-byte images (registered tables, engine.cpp build_column_images):
// the keys are plain 32-bit integer tile columns, no offsets / character gathers
constexpr FusedShapeDesc kShapeQ1P = {1, {4}, {3 /*LE*/}, 2, {0, 0}, {4, 4}, 1, 2, {0, 1}, {0, 1}, {16, 0}, {16, 16}, 6,
                                      {3, 0, 0, 1, 2, 0}, {0, 16, 16, 0, 0, 16}};
// q1 and q6 when the decimal columns carry their int32 images as well (registered tables whose values fit 32 bits, as
// every TPC-H value does): 28 and 16 bytes per row instead of 76 and 52
constexpr FusedShapeDesc kShapeQ1N = {1, {4}, {3 /*LE*/}, 2, {0, 0}, {4, 4}, 1, 2, {0, 1}, {0, 1}, {4, 0}, {4, 4}, 6,
                                      {3, 0, 0, 1, 2, 0}, {0, 4, 4, 0, 0, 4}};
constexpr FusedShapeDesc kShapeQ6N = {5, {4, 4, 4, 4, 4}, {5 /*GE*/, 2 /*LT*/, 5, 3 /*LE*/, 2}, 0, {0, 0}, {0, 0}, 0, 1, {2, 0}, {0, 0}, {4, 0}, {4, 0}, 2,
                                      {3, 1}, {0, 0}};
constexpr FusedShape kQ1P = fused_shape_encode(kShapeQ1P);
constexpr FusedShape kQ1 = fused_shape_encode(kShapeQ1);
constexpr FusedShape kQ6 = fused_shape_encode(kShapeQ6);
constexpr FusedShape kQ1N = fused_shape_encode(kShapeQ1N);
constexpr FusedShape kQ6N = fused_shape_encode(kShapeQ6N);

// (rows per thread, launch bound) variants compiled for each shape
template <int G, uint64_t SA, uint64_t SB>
static cudaError_t launch_fused_variant(int R, int grid, int block, size_t smem, cudaStream_t st) {
  if (R == 2) {
    if (block <= 256) return launch_fused_one<G, 2, 256, SA, SB>(grid, block, smem, st);
    if (block <= 384) return launch_fused_one<G, 2, 384, SA, SB>(grid, block, smem, st);
    if (block <= 416) return launch_fused_one<G, 2, 416, SA, SB>(grid, block, smem, st);
    return launch_fused_one<G, 2, 512, SA, SB>(grid, block, smem, st);
  }
  if (R == 4) {
    if (block <= 256) return launch_fused_one<G, 4, 256, SA, SB>(grid, block, smem, st);
    return launch_fused_one<G, 4, 384, SA, SB>(grid, block, smem, st);
  }
  return cudaErrorInvalidValue;
}

// *is_static tells whether an ahead-of-time shape ran (else the run-time-described variant)
static cudaError_t launch_fused(const FusedSpec& F, FusedShape shape, int reg_groups, int grid, int block, size_t smem, cudaStream_t st, int* is_static) {
  const int R = F.rows_per_thread;
  *is_static = 1;
  if (reg_groups > 1 && shape.a == kQ1.a && shape.b == kQ1.b) return launch_fused_variant<VM_REG_GROUPS, kQ1.a, kQ1.b>(R, grid, block, smem, st);
  if (reg_groups > 1 && shape.a == kQ1P.a && shape.b == kQ1P.b) return launch_fused_variant<VM_REG_GROUPS, kQ1P.a, kQ1P.b>(R, grid, block, smem, st);
  if (reg_groups <= 1 && shape.a == kQ6.a && shape.b == kQ6.b) return launch_fused_variant<1, kQ6.a, kQ6.b>(R, grid, block, smem, st);
  if (reg_groups > 1 && shape.a == kQ1N.a && shape.b == kQ1N.b) return launch_fused_variant<VM_REG_GROUPS, kQ1N.a, kQ1N.b>(R, grid, block, smem, st);
  if (reg_groups <= 1 && shape.a == kQ6N.a && shape.b == kQ6N.b) return launch_fused_variant<1, kQ6N.a, kQ6N.b>(R, grid, block, smem, st);
  *is_static = 0;
  if (reg_groups > 1) return launch_fused_variant<VM_REG_GROUPS, 0, 0>(R, grid, block, smem, st);
  return launch_fused_variant<1, 0, 0>(R, grid, block, smem, st);
}

}  // namespace b200
