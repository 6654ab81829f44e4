// Lowering of FilterExec / ProjectionExec chains and PhysicalExpr trees to the device pipeline
// program (csrc/device/program.h).  The expression semantics implemented here are the ones the
// CPU oracle restates from DataFusion/arrow-rs (see oracle/oracle.cpp and DESIGN.md "Semantics"):
// decimal result types and rescaling, checked decimal arithmetic, wrapping integer arithmetic,
// Kleene AND/OR, safe casts, CASE / IN / LIKE.
#pragma once
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>

#include "device_mem.hpp"

namespace b200 {

struct ColRef {
  Operand op;
  DataType type;
  bool nullable = false;
  std::string name;
  std::vector<DevPtr> keep;  // allocations a string value may point into
  uint64_t str_bound = ~0ull;  // strings: bound on the bytes of all its rows in one launch (~0: unknown)
};

inline Operand mk_operand(uint8_t kind, uint8_t vk, int idx) {
  Operand o;
  o.kind = kind;
  o.vk = vk;
  o.idx = (uint16_t)idx;
  return o;
}

// Device copies of the regex DFAs compiled at typing (Expr::regex), one per pattern and flags (Expr::regex_key), kept for
// the engine's lifetime: a warm stage builds and uploads nothing.  `compiles` counts the uploads (b200_engine_counter
// "regex_compiles").  An upload waits for its copy before the pointer is published: a copy from pageable memory may still
// be in flight when cudaMemcpy returns, and another task's stream may use the table next.
struct RegexCache {
  std::mutex mu;
  std::map<std::string, void*> dev;
  std::atomic<uint64_t> compiles{0};
  const void* get(const std::string& key, const rx::Dfa& d, cudaStream_t st) {
    std::lock_guard<std::mutex> g(mu);
    auto it = dev.find(key);
    if (it != dev.end()) return it->second;
    void* p = nullptr;
    CUDA_CHECK(cudaMalloc(&p, d.blob.size()));
    cudaError_t ce = cudaMemcpyAsync(p, d.blob.data(), d.blob.size(), cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) {
      cudaFree(p);
      CUDA_CHECK(ce);
    }
    dev[key] = p;
    compiles++;
    return p;
  }
  void clear() {
    std::lock_guard<std::mutex> g(mu);
    for (auto& kv : dev) cudaFree(kv.second);
    dev.clear();
  }
};

class PipelineBuilder {
 public:
  Program prog;
  std::vector<ColRef> cols;  // current (virtual) schema
  std::vector<DevPtr> keep;  // literal pools etc.
  int block = 512;
  // string builders (OP_CONCAT and up): how many the program holds and the sum of their outputs' bounds (~0: some
  // output has none); arena_floor: the need a previous launch of this program reported (launch_program sizes the arena)
  int arena_ops = 0;
  uint64_t arena_bound = 0;
  uint64_t arena_floor = 0;

  PipelineBuilder(const DevBatch& src, cudaStream_t st, RegexCache* regex) : src_(src), st_(st), regex_(regex) {
    memset(&prog, 0, sizeof prog);
    src_map_.assign(src.cols.size(), -1);
    for (size_t i = 0; i < src.cols.size(); i++) {
      ColRef c;
      c.op = mk_operand(OPD_NONE, vk_of(src.cols[i].type), (int)i);  // resolved lazily by use_source()
      c.type = src.cols[i].type;
      c.nullable = src.cols[i].valid != nullptr;
      c.name = src.cols[i].name;
      c.keep = src.cols[i].keep;
      if (src.cols[i].phys == PH_UTF8 && src.cols[i].chars_bytes >= 0) c.str_bound = (uint64_t)src.cols[i].chars_bytes;
      lazy_src_.push_back((int)i);
      cols.push_back(c);
    }
    prog.n_rows = src.n;
  }

  // ---- schema-level steps --------------------------------------------------------------------
  void apply_filter(const Expr& pred) {
    // FilterExec keeps a row iff the predicate is TRUE; an AND chain therefore decomposes exactly
    // into successive filters, and a comparison conjunct is fused with the filter itself
    if (pred.kind == Expr::Bin && pred.op == BinOp::And) {
      apply_filter(*pred.args[0]);
      apply_filter(*pred.args[1]);
      return;
    }
    if (pred.kind == Expr::Bin && is_compare(pred.op)) {
      ColRef a = compile(*pred.args[0]);
      pin(a);
      ColRef b = compile(*pred.args[1]);
      unpin(a);
      ColRef r = compare(pred.op, a, b);
      prog.code[prog.n_instr - 1].flags |= IF_FILTER;
      release(a);
      release(b);
      release(r);
      return;
    }
    ColRef p = compile(pred);
    VInstr ins = blank(OP_FILTER, VK_BOOL);
    ins.a = resolve(p);
    emit(ins);
    release(p);
  }
  void apply_select(const std::vector<int>& projection) {
    std::vector<ColRef> nc;
    for (int i : projection) nc.push_back(cols.at((size_t)i));
    for (size_t i = 0; i < cols.size(); i++) {
      bool kept = false;
      for (int j : projection) kept |= (size_t)j == i;
      if (!kept) release(cols[i]);
    }
    cols.swap(nc);
  }
  void apply_projection(const std::vector<NamedExpr>& exprs) {
    std::vector<ColRef> nc;
    for (auto& ne : exprs) {
      ColRef c = compile(*ne.expr);
      pin(c);
      c.name = ne.name;
      nc.push_back(c);
    }
    cols.swap(nc);
  }

  // ---- expression compiler -------------------------------------------------------------------
  ColRef compile(const Expr& e) {
    switch (e.kind) {
      case Expr::Col: {
        ColRef c = cols.at((size_t)e.col);
        return c;
      }
      case Expr::Lit: return literal(e.type, e.lit);
      case Expr::Bin:
        if (e.op == BinOp::StringConcat) return compile_concat(e, 0, BUILD_NULLS);
        return is_regex(e.op) ? compile_regex(e) : compile_bin(e);
      case Expr::Not: {
        ColRef a = compile(*e.args[0]);
        ColRef r = new_reg(DataType(TypeId::Bool), a.nullable);
        VInstr ins = blank(OP_NOT, VK_BOOL);
        ins.a = resolve(a);
        ins.dst = r.op;
        if (a.nullable) ins.flags |= IF_NULLCHK;
        emit(ins);
        release(a);
        return r;
      }
      case Expr::Neg: {
        ColRef a = compile(*e.args[0]);
        ColRef r = new_reg(e.type, a.nullable);
        VInstr ins = blank(OP_NEG, vk_of(e.type));
        ins.a = resolve(a);
        ins.dst = r.op;
        if (a.nullable) ins.flags |= IF_NULLCHK;
        emit(ins);
        release(a);
        if (e.type.pk() == PK::I64) return wrap_int(r, e.type);
        return r;
      }
      case Expr::IsNull:
      case Expr::IsNotNull: {
        ColRef a = compile(*e.args[0]);
        ColRef r = new_reg(DataType(TypeId::Bool), false);
        VInstr ins = blank(e.kind == Expr::IsNull ? OP_IS_NULL : OP_IS_NOT_NULL, VK_BOOL);
        ins.a = resolve(a);
        ins.dst = r.op;
        emit(ins);
        release(a);
        return r;
      }
      case Expr::Cast: {
        ColRef a = compile(*e.args[0]);
        return cast_to(a, e.type);
      }
      case Expr::Case: return compile_case(e);
      case Expr::InList: {
        ColRef x = compile(*e.args[0]);
        pin(x);
        ColRef acc;
        bool have = false;
        for (size_t i = 1; i < e.args.size(); i++) {
          ColRef it = compile(*e.args[i]);
          ColRef eq = compare(BinOp::Eq, x, it);
          release(it);
          if (!have) {
            acc = eq;
            have = true;
          } else {
            ColRef o = logic(OP_OR, acc, eq);
            release(acc);
            release(eq);
            acc = o;
          }
        }
        unpin(x);
        release(x);
        if (!have) return literal_bool(false);
        if (e.negated) {
          ColRef r = new_reg(DataType(TypeId::Bool), acc.nullable);
          VInstr ins = blank(OP_NOT, VK_BOOL);
          ins.a = resolve(acc);
          ins.dst = r.op;
          if (acc.nullable) ins.flags |= IF_NULLCHK;
          emit(ins);
          release(acc);
          return r;
        }
        return acc;
      }
      case Expr::Like: {
        if (e.case_insensitive) return compile_regex(e);
        ColRef a = compile(*e.args[0]);
        ColRef r = new_reg(DataType(TypeId::Bool), a.nullable);
        VInstr ins = blank(OP_LIKE, VK_STR);
        ins.a = resolve(a);
        ins.dst = r.op;
        ins.imm = string_imm(e.pattern);
        ins.aux = e.negated ? 1 : 0;
        if (a.nullable) ins.flags |= IF_NULLCHK;
        emit(ins);
        release(a);
        return r;
      }
      case Expr::Fn: {
        if (e.fn == "regexp_like") return compile_regex(e);
        if (is_string_builder(e.fn)) return compile_build_fn(e);
        const int part = date_part_index(e.fn);
        if (part >= 0) return unary_fn(e, OP_DATE_PART, VK_I64, (uint8_t)part, 0);
        if (e.fn == "substr") {
          ColRef a = compile(*e.args[0]);
          ColRef s = compile(*e.args[1]);
          ColRef r = new_reg(e.type, a.nullable || s.nullable);
          r.keep = a.keep;
          r.str_bound = a.str_bound;
          VInstr ins = blank(OP_SUBSTR, VK_STR);
          ins.a = resolve(a);
          ins.b = resolve(s);
          ins.dst = r.op;
          ins.imm = -1;
          if (e.args.size() > 2) {
            if (e.args[2]->kind != Expr::Lit) throw EngineError(B200_ERR_UNSUPPORTED, "substr: length must be a literal");
            ins.imm = int_imm(e.args[2]->lit.i);
          }
          if (a.nullable || s.nullable) ins.flags |= IF_NULLCHK;
          emit(ins);
          release(a);
          release(s);
          return r;
        }
        return compile_scalar_fn(e);
      }
    }
    throw EngineError(B200_ERR_UNSUPPORTED, "expression kind");
  }

  // ILIKE, ~ / ~* / !~ / !~* and regexp_like: one OP_REGEX over the DFA typing compiled (NULL when the pattern is NULL)
  ColRef compile_regex(const Expr& e) {
    if (!e.regex || e.args[0]->type.id == TypeId::Null) return null_of(DataType(TypeId::Bool));
    if (!regex_) throw EngineError(B200_ERR_UNSUPPORTED, "regular expressions are not evaluated in this pipeline");
    ColRef a = compile(*e.args[0]);
    ColRef r = new_reg(DataType(TypeId::Bool), a.nullable);
    VInstr ins = blank(OP_REGEX, VK_STR);
    ins.a = resolve(a);
    ins.dst = r.op;
    ImmDesc d;
    memset(&d, 0, sizeof d);
    d.lo = (uint64_t)regex_->get(e.regex_key, *e.regex, st_);
    d.hi = e.regex->shape();
    ins.imm = add_imm(d);
    ins.aux = e.negated ? 1 : 0;
    if (a.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    release(a);
    return r;
  }

  // ---- string builders: results written into the launch's character arena (DESIGN.md §4.1) ------------------------
  static uint64_t sat_add(uint64_t a, uint64_t b) { return a > ~0ull - b ? ~0ull : a + b; }
  static uint64_t sat_mul(uint64_t a, uint64_t b) { return b && a > ~0ull / b ? ~0ull : a * b; }
  // a builder's result register; `bound`: at most that many bytes over the launch's rows (~0: unknown)
  ColRef built_reg(bool nullable, uint64_t bound) {
    ColRef r = new_reg(DataType(TypeId::Utf8), nullable);
    r.str_bound = bound;
    arena_ops++;
    arena_bound = sat_add(arena_bound, bound);
    return r;
  }
  // the arena a launch starts with: the sum of the builders' bounds when every one has a bound, else a guess the retry
  // corrects (launch_program); never below what an earlier launch of this program needed
  uint64_t arena_capacity() const {
    const uint64_t first = arena_sound() ? arena_bound : std::min(sat_mul(rows(), 32 * (uint64_t)arena_ops), arena_first_cap());
    return std::max<uint64_t>(std::max(first, arena_floor), 256);
  }
  // the first arena holds the builders' bound only up to max(64 bytes per row, 64 MiB): a bound over all input rows can be
  // far above the need (a long literal behind a selective filter, repeat(s, 1000)); above it the launch starts from that
  // size and learns the need (launch_program waits for it)
  uint64_t arena_first_cap() const { return std::max<uint64_t>(sat_mul(rows(), 64), 64ull << 20); }
  bool arena_sound() const { return arena_bound != ~0ull && arena_bound <= arena_first_cap(); }
  uint64_t rows() const { return (uint64_t)std::max<int64_t>(prog.n_rows, 0); }
  // concat(args[from..]) (NULL arguments skipped), concat_ws(args[0], args[1..]) (BUILD_WS) or a || b (BUILD_NULLS)
  ColRef compile_concat(const Expr& e, size_t from, uint8_t flags) {
    const bool ws = flags & BUILD_WS;
    ColRef sep;
    if (ws) {
      sep = compile(*e.args[0]);
      pin(sep);
    }
    std::vector<ColRef> parts;
    auto drop_parts = [&]() {
      for (auto& c : parts) {
        unpin(c);
        release(c);
      }
    };
    uint64_t bound = 0;
    bool nullable = false;
    for (size_t i = from; i < e.args.size(); i++) {
      ColRef a = compile(*e.args[i]);
      if (a.type.id == TypeId::Null) {
        if (!(flags & BUILD_NULLS)) continue;  // concat / concat_ws skip it
        drop_parts();
        return null_of(e.type);
      }
      pin(a);
      parts.push_back(a);
      bound = sat_add(bound, a.str_bound);
      nullable = nullable || a.nullable;
    }
    if (ws) bound = sat_add(bound, sat_mul(sep.str_bound, parts.size() > 1 ? parts.size() - 1 : 0));
    ColRef r = emit_concat(parts, ws ? &sep : nullptr, flags, bound, (flags & BUILD_NULLS) ? nullable : (ws && sep.nullable));
    drop_parts();
    if (ws) {
      unpin(sep);
      release(sep);
    }
    return r;
  }
  ColRef emit_concat(const std::vector<ColRef>& parts, const ColRef* sep, uint8_t flags, uint64_t bound, bool nullable) {
    // the arguments in consecutive immediates, eight per immediate (program.h); the first holds their count
    std::vector<ImmDesc> ds(std::max<size_t>((parts.size() + 7) / 8, 1));
    memset(ds.data(), 0, ds.size() * sizeof(ImmDesc));
    for (size_t i = 0; i < parts.size(); i++) {
      const Operand o = resolve(parts[i]);
      const uint64_t w = ((uint64_t)o.kind << 12) | o.idx;
      ImmDesc& d = ds[i / 8];
      ((i & 7) < 4 ? d.lo : d.hi) |= w << (16 * (i & 3));
    }
    ds[0]._pad = (uint32_t)parts.size();
    if (prog.n_imms + (int)ds.size() > VM_MAX_IMMS) throw EngineError(B200_ERR_UNSUPPORTED, "too many literals in one pipeline");
    const int imm = prog.n_imms;
    for (auto& d : ds) prog.imms[prog.n_imms++] = d;
    ColRef r = built_reg(nullable, bound);
    VInstr ins = blank(OP_CONCAT, VK_STR);
    ins.imm = imm;
    ins.aux = flags;
    if (sep) ins.a = resolve(*sep);
    ins.dst = r.op;
    ins.flags = IF_NULLCHK;
    emit(ins);
    return r;
  }
  ColRef compile_build_fn(const Expr& e) {
    const std::string& f = e.fn;
    if (f == "concat") return compile_concat(e, 0, 0);
    if (f == "concat_ws") {
      if (e.args[0]->type.id == TypeId::Null) return null_of(e.type);
      return compile_concat(e, 1, BUILD_WS);
    }
    for (auto& a : e.args)
      if (a->type.id == TypeId::Null) return null_of(e.type);
    ColRef a = compile(*e.args[0]);
    pin(a);
    ColRef b;
    uint64_t bound = a.str_bound;
    if (f == "repeat") {
      b = compile(*e.args[1]);
      if (b.op.kind != OPD_IMM) bound = ~0ull;  // a column count: no bound, the launch's need decides
      else bound = sat_mul(bound, (uint64_t)std::max<int64_t>((int64_t)prog.imms[b.op.idx].lo, 0));
    }
    unpin(a);
    ColRef r = built_reg(a.nullable || b.nullable, bound);
    VInstr ins = blank(f == "repeat" ? OP_REPEAT : OP_REVERSE, VK_STR);
    ins.a = resolve(a);
    if (f == "repeat") ins.b = resolve(b);
    ins.dst = r.op;
    ins.flags = IF_NULLCHK;
    emit(ins);
    release(a);
    release(b);
    return r;
  }
  // CAST(a AS Utf8) of the source types DESIGN.md §6 (xi) lists; each has a longest text, which bounds the arena
  ColRef cast_to_utf8(const ColRef& a) {
    const DataType& t = a.type;
    uint8_t kind;
    uint64_t widest;
    if (t.is_signed_int() || t.is_unsigned_int()) {
      kind = t.id == TypeId::UInt64 ? TS_UINT64 : TS_INT;
      widest = 20;
    } else if (t.is_decimal() && t.scale >= 0) {
      kind = TS_DEC128;
      widest = 41;
    } else if (t.id == TypeId::Date32) {
      kind = TS_DATE32;
      widest = 13;
    } else if (t.id == TypeId::Bool) {
      kind = TS_BOOL;
      widest = 5;
    } else {
      throw EngineError(B200_ERR_UNSUPPORTED, "cast " + t.str() + " -> Utf8");
    }
    ColRef r = built_reg(a.nullable, sat_mul(widest, (uint64_t)std::max<int64_t>(prog.n_rows, 0)));
    VInstr ins = blank(OP_TO_STR, vk_of(t));
    ins.a = resolve(a);
    ins.dst = r.op;
    ins.aux = kind;
    ins.imm = kind == TS_DEC128 ? t.scale : 0;
    ins.flags = IF_NULLCHK;
    emit(ins);
    release(a);
    return r;
  }

  // one-operand function: dst = op(a); string results are views into a's bytes
  ColRef unary_fn(const Expr& e, uint8_t op, uint8_t t, uint8_t aux, int32_t imm) {
    ColRef a = compile(*e.args[0]);
    ColRef r = new_reg(e.type, a.nullable);
    r.keep = a.keep;
    r.str_bound = a.str_bound;
    VInstr ins = blank(op, t);
    ins.a = resolve(a);
    ins.dst = r.op;
    ins.aux = aux;
    ins.imm = imm;
    if (a.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    release(a);
    return r;
  }
  ColRef null_of(const DataType& t) {
    LitValue l;
    l.is_null = true;
    return literal(t, l);
  }
  // a literal operand of a function, which travels as an immediate; NULL gives a NULL result
  const Expr& literal_arg(const Expr& e, size_t i, const char* what) {
    if (e.args[i]->kind != Expr::Lit) throw EngineError(B200_ERR_UNSUPPORTED, e.fn + ": " + what + " must be a literal");
    return *e.args[i];
  }

  // the scalar functions of DESIGN.md §3 besides date_part and substr; typing (plan.hpp) has checked the argument types
  ColRef compile_scalar_fn(const Expr& e) {
    const std::string& f = e.fn;
    if (f == "abs") {
      const DataType& t = e.args[0]->type;
      if (t.is_unsigned_int()) return compile(*e.args[0]);
      return unary_fn(e, OP_ABS, vk_of(t), t.is_signed_int() ? phys_of(t) : 0, 0);
    }
    if (f == "floor" || f == "ceil") return unary_fn(e, f == "floor" ? OP_FLOOR : OP_CEIL, VK_F64, 0, 0);
    if (f == "round") {
      int64_t n = 0;
      if (e.args.size() > 1) {
        const Expr& d = literal_arg(e, 1, "the digit count");
        if (d.lit.is_null) return null_of(e.type);
        n = d.lit.i;
      }
      if (n > 22 || n < -22) throw EngineError(B200_ERR_UNSUPPORTED, "round to " + std::to_string(n) + " digits is not supported (|digits| <= 22)");
      double p = 1;
      for (int64_t i = 0; i < (n < 0 ? -n : n); i++) p *= 10;  // exact: 10^22 is the largest power of ten binary64 holds
      const bool f32 = e.type.id == TypeId::Float32;
      LitValue fl;
      fl.f = f32 ? (n >= 0 ? (double)(float)p : (double)(1.0f / (float)p)) : (n >= 0 ? p : 1.0 / p);
      const int fi = literal(DataType(TypeId::Float64), fl).op.idx;
      return unary_fn(e, OP_ROUND, VK_F64, f32 ? PH_F32 : 0, fi);
    }
    if (f == "character_length" || f == "octet_length") return unary_fn(e, f == "octet_length" ? OP_OCTET_LENGTH : OP_CHAR_LENGTH, VK_STR, 0, 0);
    if (f == "btrim" || f == "ltrim" || f == "rtrim") {
      int set = -1;
      if (e.args.size() > 1) {
        const Expr& s = literal_arg(e, 1, "the character set");
        if (s.lit.is_null) return null_of(e.type);
        set = string_imm(s.lit.s);
      } else {
        set = string_imm(" ");  // DataFusion's default removes spaces only, not all whitespace [EXT]
      }
      return unary_fn(e, OP_TRIM, VK_STR, f == "btrim" ? TRIM_BOTH : f == "ltrim" ? TRIM_LEADING : TRIM_TRAILING, set);
    }
    if (f == "coalesce") {
      // the CASE lowering's shape, CASE WHEN a0 IS NOT NULL THEN a0 ... ELSE a_last END, with every argument compiled
      // once: dst = a_last, then from the back dst = a_i where a_i is not NULL (OP_SELECT)
      if (e.args.size() == 1) return cast_to(compile(*e.args[0]), e.type);
      ColRef dst = new_reg(e.type, true);
      pin(dst);
      {
        ColRef v = cast_to(compile(*e.args.back()), e.type);
        VInstr ins = blank(OP_MOV, vk_of(e.type));
        ins.a = resolve(v);
        ins.dst = dst.op;
        ins.flags = IF_NULLCHK;
        emit(ins);
        dst.keep.insert(dst.keep.end(), v.keep.begin(), v.keep.end());
        release(v);
      }
      for (size_t i = e.args.size() - 1; i-- > 0;) {
        ColRef v = cast_to(compile(*e.args[i]), e.type);
        pin(v);
        ColRef c = new_reg(DataType(TypeId::Bool), false);
        VInstr t = blank(OP_IS_NOT_NULL, VK_BOOL);
        t.a = resolve(v);
        t.dst = c.op;
        emit(t);
        unpin(v);
        VInstr ins = blank(OP_SELECT, vk_of(e.type));
        ins.a = c.op;
        ins.b = resolve(v);
        ins.dst = dst.op;
        ins.flags = IF_NULLCHK;
        emit(ins);
        dst.keep.insert(dst.keep.end(), v.keep.begin(), v.keep.end());
        release(c);
        release(v);
      }
      unpin(dst);
      return dst;
    }
    if (f == "nullif" || f == "starts_with" || f == "ends_with") {
      ColRef a = compile(*e.args[0]);
      pin(a);
      ColRef b = compile(*e.args[1]);
      unpin(a);
      const bool nullif = f == "nullif";
      if (nullif && (a.type.id == TypeId::Null || b.type.id == TypeId::Null)) {
        release(b);
        if (a.type.id == TypeId::Null) return null_of(e.type);
        return a;  // nullif(a, NULL) = a
      }
      ColRef r = new_reg(e.type, nullif || a.nullable || b.nullable);
      if (nullif) r.keep = a.keep;
      VInstr ins = blank(nullif ? OP_NULLIF : f == "starts_with" ? OP_STARTS_WITH : OP_ENDS_WITH, nullif ? vk_of(a.type) : VK_STR);
      ins.a = resolve(a);
      ins.b = resolve(b);
      ins.dst = r.op;
      ins.flags = IF_NULLCHK;
      emit(ins);
      release(a);
      release(b);
      return r;
    }
    throw EngineError(B200_ERR_UNSUPPORTED, "scalar function " + f);
  }

  // hash of key columns in the structure of create_hashes (see csrc/common/hash.hpp)
  ColRef hash_of(const std::vector<ColRef>& keys) {
    ColRef h = new_reg(DataType(TypeId::Int64), false);
    pin(h);
    for (size_t k = 0; k < keys.size(); k++) {
      VInstr ins = blank(k == 0 ? OP_HASH : OP_HASH_COMBINE, vk_of(keys[k].type));
      ins.a = resolve(keys[k]);
      ins.dst = h.op;
      emit(ins);
    }
    if (keys.empty()) {
      VInstr ins = blank(OP_MOV, VK_I64);
      ins.a = mk_operand(OPD_IMM, VK_I64, int_imm(0));
      ins.dst = h.op;
      emit(ins);
    }
    return h;
  }
  // OP_STR_PACK8: optimistic packing of a short string into an Int64 (len << shift | bytes)
  ColRef str_pack(const ColRef& s, int max_len, int shift) {
    ColRef r = new_reg(DataType(TypeId::Int64), s.nullable);
    VInstr ins = blank(OP_STR_PACK8, VK_STR);
    ins.a = resolve(s);
    ins.dst = r.op;
    ins.aux = (uint8_t)max_len;
    ins.imm = shift;
    if (s.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    return r;
  }
  ColRef add_literal_i64(const ColRef& a, int64_t v) {
    ColRef r = new_reg(DataType(TypeId::Int64), a.nullable);
    VInstr ins = blank(OP_ADD, VK_I64);
    ins.a = resolve(a);
    ins.b = mk_operand(OPD_IMM, VK_I64, int_imm(v));
    ins.dst = r.op;
    if (a.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    return r;
  }
  // lo + hi * 2^32 for two values known to lie in [0, 2^32)
  ColRef combine32(const ColRef& lo, const ColRef& hi) {
    ColRef t = new_reg(DataType(TypeId::Int64), false);
    VInstr m = blank(OP_MADD_I64, VK_I64);
    m.a = resolve(lo);
    m.b = resolve(hi);
    m.dst = t.op;
    m.imm = int_imm(4294967296ll);
    emit(m);
    return t;
  }
  ColRef mod_u64(const ColRef& h, uint64_t m) {
    ColRef r = new_reg(DataType(TypeId::UInt32), false);
    VInstr ins = blank(OP_MOD_U64, VK_I64);
    ins.a = resolve(h);
    ins.dst = r.op;
    ins.imm = int_imm((int64_t)m);
    emit(ins);
    return r;
  }

  Operand resolve(const ColRef& c) {
    if (c.op.kind != OPD_NONE) return c.op;
    return use_source(c.op.idx);
  }
  // index of the source-batch column this reference forwards untouched, or -1 for a computed value
  int source_index(const ColRef& c) const {
    if (c.op.kind == OPD_NONE) return (int)c.op.idx;
    if (c.op.kind == OPD_COL)
      for (size_t i = 0; i < src_map_.size(); i++)
        if (src_map_[i] == (int)c.op.idx) return (int)i;
    return -1;
  }
  void pin(const ColRef& c) {
    if (c.op.kind == OPD_REG) pins_[c.op.idx]++;
  }
  void unpin(const ColRef& c) {
    if (c.op.kind == OPD_REG && pins_[c.op.idx] > 0) pins_[c.op.idx]--;
  }
  void release(const ColRef& c) {
    if (c.op.kind != OPD_REG) return;
    if (pins_[c.op.idx] > 0) return;
    if (reg_free_[c.op.idx]) return;
    reg_free_[c.op.idx] = true;
  }

  // ---- layout --------------------------------------------------------------------------------
  // Must be called after all instructions are emitted and the sink is described.
  void finalize_layout(size_t min_total) {
    static const bool no_tma = getenv("B200_NO_TMA") != nullptr;
    for (int attempt = 0; attempt < 3; attempt++) {
      const int tile = block * VM_R;
      uint32_t off = 0;
      bool aligned = true;
      for (int i = 0; i < prog.n_cols; i++) {
        ColDesc& cd = prog.cols[i];
        cd.smem_off = off;
        off += (uint32_t)tile * cd.width + (cd.phys == PH_UTF8 ? 16u : 0u);
        off = (off + 127u) & ~127u;
        if (((uintptr_t)cd.data & 15) != 0) aligned = false;
        if (cd.valid) {
          cd.valid_smem_off = off;
          off += (uint32_t)tile;
          off = (off + 127u) & ~127u;
          if (((uintptr_t)cd.valid & 15) != 0) aligned = false;
        }
      }
      prog.stage_bytes = off;
      uint32_t roff = 0;
      for (int i = 0; i < prog.n_regs; i++) {
        RegDesc& rd = prog.regs[i];
        uint32_t unit = rd.vk == VK_BOOL ? 4u : (rd.vk == VK_I128 || rd.vk == VK_STR ? 16u * VM_R : 8u * VM_R);
        rd.smem_off = roff;
        roff += unit * (uint32_t)block;
        if (reg_nullable_[i]) {
          rd.valid_off = roff;
          roff += 4u * (uint32_t)block;
        } else {
          rd.valid_off = 0xFFFFFFFFu;
        }
        roff = (roff + 15u) & ~15u;
      }
      prog.regs_bytes = (roff + 127u) & ~127u;
      const uint32_t budget = 208 * 1024;  // dynamic part; ~16 KB of static shared memory (decoded micro-ops) come on top
      int S = prog.stage_bytes ? (int)((budget - prog.regs_bytes) / prog.stage_bytes) : VM_MAX_STAGES;
      if (prog.regs_bytes >= budget) S = 0;
      if (S > VM_MAX_STAGES) S = VM_MAX_STAGES;
      prog.use_tma = (aligned && !no_tma) ? 1 : 0;
      if (S >= 2) {
        prog.n_stages = (uint32_t)S;
        // the register-sink flush stages its reduction in the (idle) tile buffers
        const size_t total = (size_t)S * prog.stage_bytes + prog.regs_bytes;
        if (total < min_total) prog.regs_bytes += (uint32_t)((min_total - total + 127) & ~(size_t)127);
        return;
      }
      if (block > 128) {
        block /= 2;
        continue;
      }
      throw EngineError(B200_ERR_UNSUPPORTED, "pipeline too wide for shared memory (" + std::to_string(prog.stage_bytes) + " B/stage)");
    }
  }
  size_t smem_bytes() const { return (size_t)prog.n_stages * prog.stage_bytes + prog.regs_bytes; }

  int int_imm(int64_t v) {
    ImmDesc d;
    memset(&d, 0, sizeof d);
    d.lo = (uint64_t)v;
    d.hi = v < 0 ? ~0ull : 0ull;
    return add_imm(d);
  }

 private:
  const DevBatch& src_;
  cudaStream_t st_;
  RegexCache* regex_;
  std::vector<int> src_map_;
  std::vector<int> lazy_src_;
  std::map<int, int> pins_;
  std::map<int, bool> reg_free_;
  std::map<int, bool> reg_nullable_;
  std::map<std::string, int> string_imms_;

  VInstr blank(uint8_t op, uint8_t t) {
    VInstr i;
    memset(&i, 0, sizeof i);
    i.op = op;
    i.t = t;
    return i;
  }
  void emit(const VInstr& i) {
    if (prog.n_instr >= VM_MAX_INSTR) throw EngineError(B200_ERR_UNSUPPORTED, "expression program too long");
    prog.code[prog.n_instr++] = i;
  }
  int add_imm(const ImmDesc& d) {
    for (int i = 0; i < prog.n_imms; i++)
      if (!memcmp(&prog.imms[i], &d, sizeof d)) return i;
    if (prog.n_imms >= VM_MAX_IMMS) throw EngineError(B200_ERR_UNSUPPORTED, "too many literals in one pipeline");
    prog.imms[prog.n_imms] = d;
    return prog.n_imms++;
  }
  int string_imm(const std::string& s) {
    auto it = string_imms_.find(s);  // the same literal appears many times in IN lists / OR-ed conjunctions (q19)
    if (it != string_imms_.end()) return it->second;
    DevPtr p = dev_alloc(s.size() + 16, st_);
    if (!s.empty()) CUDA_CHECK(cudaMemcpyAsync(p->ptr, s.data(), s.size(), cudaMemcpyHostToDevice, st_));
    keep.push_back(p);
    ImmDesc d;
    memset(&d, 0, sizeof d);
    d.lo = (uint64_t)p->ptr;
    d.hi = s.size();
    const int idx = add_imm(d);
    string_imms_[s] = idx;
    return idx;
  }
  Operand use_source(int src_idx) {
    if (src_map_[(size_t)src_idx] < 0) {
      if (prog.n_cols >= VM_MAX_COLS) throw EngineError(B200_ERR_UNSUPPORTED, "pipeline reads too many columns");
      const DevColumn& sc = src_.cols[(size_t)src_idx];
      ColDesc& cd = prog.cols[prog.n_cols];
      memset(&cd, 0, sizeof cd);
      cd.data = sc.data;
      cd.valid = sc.valid;
      cd.chars = sc.chars;
      cd.img32 = sc.img32;
      cd.phys = sc.phys;
      cd.width = (uint8_t)sc.width();
      cd.in_tile = 1;
      src_map_[(size_t)src_idx] = prog.n_cols++;
    }
    return mk_operand(OPD_COL, vk_of(src_.cols[(size_t)src_idx].type), src_map_[(size_t)src_idx]);
  }

 public:
  ColRef new_reg(const DataType& t, bool nullable) {
    const uint8_t vk = vk_of(t);
    auto unit = [](uint8_t k) { return k == VK_BOOL ? 0 : (k == VK_I128 || k == VK_STR ? 2 : 1); };
    int idx = -1;
    for (int i = 0; i < prog.n_regs; i++)
      if (reg_free_[i] && unit(prog.regs[i].vk) == unit(vk) && reg_nullable_[i] == nullable) {
        idx = i;
        break;
      }
    if (idx < 0) {
      if (prog.n_regs >= VM_MAX_REGS) throw EngineError(B200_ERR_UNSUPPORTED, "expression needs too many VM registers");
      idx = prog.n_regs++;
    }
    memset(&prog.regs[idx], 0, sizeof(RegDesc));
    prog.regs[idx].vk = vk;
    reg_free_[idx] = false;
    reg_nullable_[idx] = nullable;
    pins_[idx] = 0;
    ColRef c;
    c.op = mk_operand(OPD_REG, vk, idx);
    c.type = t;
    c.nullable = nullable;
    return c;
  }

 private:
  ColRef literal(const DataType& t, const LitValue& l) {
    ImmDesc d;
    memset(&d, 0, sizeof d);
    d.is_null = l.is_null ? 1 : 0;
    ColRef c;
    c.type = t;
    c.nullable = l.is_null;
    int idx;
    switch (t.pk()) {
      case PK::F64: memcpy(&d.lo, &l.f, 8); idx = add_imm(d); break;
      case PK::I128:
        d.lo = (uint64_t)l.d;
        d.hi = (uint64_t)((u128)l.d >> 64);
        idx = add_imm(d);
        break;
      case PK::Str:
        if (l.is_null) idx = add_imm(d);
        else idx = string_imm(l.s);
        prog.imms[idx].is_null = d.is_null;
        break;
      default:
        d.lo = (uint64_t)l.i;
        d.hi = l.i < 0 ? ~0ull : 0ull;
        idx = add_imm(d);
    }
    c.op = mk_operand(OPD_IMM, vk_of(t), idx);
    if (t.pk() == PK::Str) c.str_bound = l.is_null ? 0 : sat_mul(l.s.size(), (uint64_t)std::max<int64_t>(prog.n_rows, 0));
    return c;
  }
  ColRef literal_bool(bool v) {
    LitValue l;
    l.i = v;
    return literal(DataType(TypeId::Bool), l);
  }
  bool is_literal(const ColRef& c) const { return c.op.kind == OPD_IMM; }
  i128 imm_i128(const ColRef& c) const {
    const ImmDesc& d = prog.imms[c.op.idx];
    if (c.op.vk == VK_I128) return (i128)(((u128)d.hi << 64) | d.lo);
    return (i128)(int64_t)d.lo;
  }
  ColRef dec_literal(i128 v, const DataType& t) {
    LitValue l;
    l.d = v;
    return literal(t, l);
  }

  ColRef wrap_int(const ColRef& r, const DataType& t) {
    if (t.width() >= 8 || t.pk() != PK::I64 || t.id == TypeId::Bool) return r;
    VInstr ins = blank(OP_WRAP_I64, VK_I64);
    ins.a = resolve(r);
    ins.dst = r.op.kind == OPD_REG ? r.op : new_reg(t, r.nullable).op;
    ins.aux = phys_of(t);
    if (r.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    ColRef o = r;
    o.op = ins.dst;
    o.type = t;
    return o;
  }

  // decimal operand rescaled up by 10^by (compile-time for literals)
  ColRef rescale_up(const ColRef& a, int by, const DataType& out_t) {
    if (by <= 0) {
      ColRef o = a;
      o.type = out_t;
      return o;
    }
    if (is_literal(a) && !prog.imms[a.op.idx].is_null) {
      i128 v = imm_i128(a);
      i128 lim = ((i128)1 << 126) / pow10_i128(by);
      if (v < lim && v > -lim) return dec_literal(v * pow10_i128(by), out_t);
    }
    ColRef r = new_reg(out_t, a.nullable);
    VInstr ins = blank(OP_CAST_I128_I128_UP, VK_I128);
    ins.a = resolve(a);
    ins.dst = r.op;
    ins.imm = by;
    ins.flags = IF_CHECKED | (a.nullable ? IF_NULLCHK : 0);
    emit(ins);
    return r;
  }
  static int scale_of(const DataType& t) { return t.is_decimal() ? t.scale : 0; }
  static int precision_of(const DataType& t) { return t.is_decimal() ? t.precision : int_as_decimal(t).precision; }

  // a UInt64 operand meeting a decimal: its value as Decimal128(20, 0), zero-extended (a 64-bit operand of a 128-bit
  // instruction is sign-extended); any other operand as it is
  ColRef widen_u64(const ColRef& a) {
    if (a.type.id != TypeId::UInt64) return a;
    const DataType t = DataType::decimal(20, 0);
    if (is_literal(a)) {
      if (prog.imms[a.op.idx].is_null) return null_of(t);
      return dec_literal((i128)prog.imms[a.op.idx].lo, t);
    }
    ColRef r = new_reg(t, a.nullable);
    VInstr ins = blank(OP_CAST_I64_I128, VK_I128);
    ins.a = resolve(a);
    ins.dst = r.op;
    ins.aux = PH_U64;
    if (a.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    return r;
  }

  ColRef to_f64(const ColRef& a) {
    if (a.type.pk() == PK::F64) return a;
    if (is_literal(a) && !prog.imms[a.op.idx].is_null) {
      LitValue l;
      if (a.type.is_decimal()) l.f = (double)imm_i128(a) / pow10_f64(a.type.scale);
      else if (a.type.id == TypeId::UInt64) l.f = (double)prog.imms[a.op.idx].lo;
      else l.f = (double)(int64_t)prog.imms[a.op.idx].lo;
      return literal(DataType(TypeId::Float64), l);
    }
    ColRef r = new_reg(DataType(TypeId::Float64), a.nullable);
    VInstr ins = blank(a.type.is_decimal() ? OP_CAST_I128_F64 : OP_CAST_I64_F64, VK_F64);
    ins.a = resolve(a);
    ins.dst = r.op;
    ins.imm = a.type.is_decimal() ? a.type.scale : 0;
    ins.aux = a.type.id == TypeId::UInt64 ? PH_U64 : 0;
    if (a.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    return r;
  }

  ColRef logic(uint8_t op, const ColRef& a, const ColRef& b) {
    ColRef r = new_reg(DataType(TypeId::Bool), a.nullable || b.nullable);
    VInstr ins = blank(op, VK_BOOL);
    ins.a = resolve(a);
    ins.b = resolve(b);
    ins.dst = r.op;
    if (a.nullable || b.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    return r;
  }

  ColRef compare(BinOp op, const ColRef& a0, const ColRef& b0) {
    ColRef a = a0, b = b0;
    uint8_t t;
    uint8_t aux = 0;
    std::vector<ColRef> temps;
    if (a.type.pk() == PK::Str || b.type.pk() == PK::Str) {
      if (a.type.pk() != b.type.pk() && a.type.id != TypeId::Null && b.type.id != TypeId::Null)
        throw EngineError(B200_ERR_UNSUPPORTED, "comparison between " + a.type.str() + " and " + b.type.str());
      t = VK_STR;
    } else if (a.type.pk() == PK::F64 || b.type.pk() == PK::F64) {
      ColRef x = to_f64(a), y = to_f64(b);
      if (x.op.kind == OPD_REG && !(x.op.idx == a.op.idx && a.op.kind == OPD_REG)) temps.push_back(x);
      if (y.op.kind == OPD_REG && !(y.op.idx == b.op.idx && b.op.kind == OPD_REG)) temps.push_back(y);
      a = x;
      b = y;
      t = VK_F64;
    } else if (a.type.is_decimal() || b.type.is_decimal()) {
      for (ColRef* x : {&a, &b}) {
        ColRef w = widen_u64(*x);
        if (w.op.kind == OPD_REG && !(x->op.kind == OPD_REG && x->op.idx == w.op.idx)) temps.push_back(w);
        *x = w;
      }
      int sa = scale_of(a.type), sb = scale_of(b.type), s = std::max(sa, sb);
      int pa = precision_of(a.type) + (s - sa), pb = precision_of(b.type) + (s - sb);
      DataType ta = DataType::decimal(std::min(38, pa), s), tb = DataType::decimal(std::min(38, pb), s);
      ColRef x = rescale_up(a, s - sa, ta), y = rescale_up(b, s - sb, tb);
      if (x.op.kind == OPD_REG && (s - sa) > 0) temps.push_back(x);
      if (y.op.kind == OPD_REG && (s - sb) > 0) temps.push_back(y);
      a = x;
      b = y;
      // both sides provably fit 64 bits: compare the low words only
      t = (pa <= 18 && pb <= 18) ? VK_I64 : VK_I128;
    } else {
      t = VK_I64;
      if (a.type.id == TypeId::UInt64 && b.type.id == TypeId::UInt64) aux = PH_U64;
    }
    ColRef r = new_reg(DataType(TypeId::Bool), a.nullable || b.nullable);
    uint8_t vop = OP_CMP_EQ;
    switch (op) {
      case BinOp::Eq: vop = OP_CMP_EQ; break;
      case BinOp::Ne: vop = OP_CMP_NE; break;
      case BinOp::Lt: vop = OP_CMP_LT; break;
      case BinOp::Le: vop = OP_CMP_LE; break;
      case BinOp::Gt: vop = OP_CMP_GT; break;
      default: vop = OP_CMP_GE;
    }
    VInstr ins = blank(vop, t);
    ins.a = resolve(a);
    ins.b = resolve(b);
    if (t == VK_I64 && a.type.is_decimal()) {
      ins.a.vk = VK_I64;  // narrow view of a decimal operand
      ins.b.vk = VK_I64;
    }
    ins.dst = r.op;
    ins.aux = aux;
    if (a.nullable || b.nullable) ins.flags |= IF_NULLCHK;
    emit(ins);
    for (auto& tmp : temps) release(tmp);
    return r;
  }

  ColRef compile_bin(const Expr& e) {
    if (is_logic(e.op)) {
      ColRef a = compile(*e.args[0]);
      pin(a);
      ColRef b = compile(*e.args[1]);
      unpin(a);
      ColRef r = logic(e.op == BinOp::And ? OP_AND : OP_OR, a, b);
      release(a);
      release(b);
      return r;
    }
    if (is_compare(e.op)) {
      ColRef a = compile(*e.args[0]);
      pin(a);
      ColRef b = compile(*e.args[1]);
      unpin(a);
      ColRef r = compare(e.op, a, b);
      release(a);
      release(b);
      return r;
    }
    if (is_bitwise(e.op)) {
      // integer operands of the result's type (plan.hpp); only << can leave the type's range
      ColRef a = compile(*e.args[0]);
      pin(a);
      ColRef b = compile(*e.args[1]);
      unpin(a);
      static const uint8_t vops[] = {OP_BIT_AND, OP_BIT_OR, OP_BIT_XOR, OP_SHL, OP_SHR};
      ColRef r = new_reg(e.type, a.nullable || b.nullable);
      VInstr ins = blank(vops[(int)e.op - (int)BinOp::BitAnd], VK_I64);
      ins.a = resolve(a);
      ins.b = resolve(b);
      ins.dst = r.op;
      ins.aux = phys_of(e.type);
      if (a.nullable || b.nullable) ins.flags |= IF_NULLCHK;
      emit(ins);
      release(a);
      release(b);
      return e.op == BinOp::Shl ? wrap_int(r, e.type) : r;
    }
    const DataType rt = e.type;
    // fused decimal shape  a * (lit +/- b)
    if (rt.is_decimal() && e.op == BinOp::Mul) {
      for (int side = 0; side < 2; side++) {
        const Expr& inner = *e.args[(size_t)(1 - side)];
        const Expr& other = *e.args[(size_t)side];
        if (inner.kind == Expr::Bin && (inner.op == BinOp::Sub || inner.op == BinOp::Add) && inner.type.is_decimal() &&
            inner.args[0]->kind == Expr::Lit && !inner.args[0]->lit.is_null && inner.args[1]->type.is_decimal() &&
            other.type.is_decimal()) {
          const Expr& lit = *inner.args[0];
          int sl = scale_of(lit.type), sb = inner.args[1]->type.scale;
          if (inner.type.scale == sb && sl <= sb) {
            ColRef a = compile(other);
            pin(a);
            ColRef b = compile(*inner.args[1]);
            unpin(a);
            i128 lv = (lit.type.is_decimal() ? lit.lit.d : (i128)lit.lit.i) * pow10_i128(sb - sl);
            ColRef lc = dec_literal(lv, inner.type);
            ColRef r = new_reg(rt, a.nullable || b.nullable);
            VInstr ins = blank(inner.op == BinOp::Sub ? OP_DEC_MUL_LIT_MINUS : OP_DEC_MUL_LIT_PLUS, VK_I128);
            ins.a = resolve(a);
            ins.b = resolve(b);
            ins.dst = r.op;
            ins.imm = lc.op.idx;
            ins.flags = IF_CHECKED | ((a.nullable || b.nullable) ? IF_NULLCHK : 0);
            emit(ins);
            release(a);
            release(b);
            return r;
          }
        }
      }
    }
    ColRef a = compile(*e.args[0]);
    pin(a);
    ColRef b = compile(*e.args[1]);
    unpin(a);
    ColRef r;
    uint8_t vop = OP_ADD;
    switch (e.op) {
      case BinOp::Add: vop = OP_ADD; break;
      case BinOp::Sub: vop = OP_SUB; break;
      case BinOp::Mul: vop = OP_MUL; break;
      case BinOp::Div: vop = OP_DIV; break;
      default: vop = OP_MOD;
    }
    const bool nullable = a.nullable || b.nullable;
    if (rt.is_float()) {
      ColRef x = to_f64(a), y = to_f64(b);
      r = new_reg(rt, nullable);
      VInstr ins = blank(vop, VK_F64);
      ins.a = resolve(x);
      ins.b = resolve(y);
      ins.dst = r.op;
      ins.aux = rt.id == TypeId::Float32 ? PH_F32 : 0;
      if (nullable) ins.flags |= IF_NULLCHK;
      emit(ins);
      if (x.op.kind == OPD_REG && !(a.op.kind == OPD_REG && a.op.idx == x.op.idx)) release(x);
      if (y.op.kind == OPD_REG && !(b.op.kind == OPD_REG && b.op.idx == y.op.idx)) release(y);
    } else if (rt.is_decimal()) {
      for (ColRef* x : {&a, &b}) {
        ColRef w = widen_u64(*x);
        if (w.op.kind == OPD_REG && !(x->op.kind == OPD_REG && x->op.idx == w.op.idx)) release(*x);
        *x = w;
      }
      int s1 = scale_of(a.type), s2 = scale_of(b.type);
      ColRef x = a, y = b;
      int imm = 0;
      if (e.op == BinOp::Add || e.op == BinOp::Sub) {
        x = rescale_up(a, rt.scale - s1, DataType::decimal(38, rt.scale));
        y = rescale_up(b, rt.scale - s2, DataType::decimal(38, rt.scale));
      } else if (e.op == BinOp::Div) {
        imm = rt.scale - s1 + s2;
      } else if (e.op == BinOp::Mod) {
        int s = std::max(s1, s2);
        x = rescale_up(a, s - s1, DataType::decimal(38, s));
        y = rescale_up(b, s - s2, DataType::decimal(38, s));
      }
      r = new_reg(rt, nullable || e.op == BinOp::Div || e.op == BinOp::Mod);
      VInstr ins = blank(vop, VK_I128);
      ins.a = resolve(x);
      ins.b = resolve(y);
      ins.dst = r.op;
      ins.imm = imm;
      ins.flags = IF_CHECKED | (nullable ? IF_NULLCHK : 0);
      emit(ins);
      if (x.op.kind == OPD_REG && !(a.op.kind == OPD_REG && a.op.idx == x.op.idx)) release(x);
      if (y.op.kind == OPD_REG && !(b.op.kind == OPD_REG && b.op.idx == y.op.idx)) release(y);
    } else {
      r = new_reg(rt, nullable);
      VInstr ins = blank(vop, VK_I64);
      ins.a = resolve(a);
      ins.b = resolve(b);
      ins.dst = r.op;
      if (vop == OP_DIV || vop == OP_MOD) ins.aux = phys_of(rt);  // unsigned division, the minimum / -1 overflow
      ins.flags = IF_CHECKED | (nullable ? IF_NULLCHK : 0);
      emit(ins);
      r = wrap_int(r, rt);
    }
    release(a);
    release(b);
    return r;
  }

  // CASE WHEN c1 THEN v1 ... [ELSE e] END, as lazily as DataFusion's CaseExpr evaluates it (evaluate_selection): each WHEN
  // runs for the rows no earlier WHEN took, each THEN for the rows its WHEN took, the ELSE for the rest.  OP_ACTIVE
  // narrows the active rows around each part and restores them after the last, so an operation that can fail (a division,
  // a checked decimal operation, a cast to a decimal) fails only for a row its part is evaluated for.
  ColRef compile_case(const Expr& e) {
    const size_t npairs = (e.args.size() - (e.has_else ? 1 : 0)) / 2;
    const uint8_t vk = vk_of(e.type);
    ColRef dst = new_reg(e.type, true);
    pin(dst);
    {
      LitValue l;
      l.is_null = true;
      VInstr ins = blank(OP_MOV, vk);
      ins.a = resolve(literal(e.type, l));
      ins.dst = dst.op;
      ins.flags = IF_NULLCHK;
      emit(ins);
    }
    auto mask = [&](const ColRef* a, const ColRef* b, uint8_t negate, const ColRef* out) {
      VInstr ins = blank(OP_ACTIVE, VK_BOOL);
      if (a) ins.a = resolve(*a);
      if (b) ins.b = resolve(*b);
      if (out) ins.dst = out->op;
      ins.aux = negate;
      emit(ins);
    };
    ColRef entry = new_reg(DataType(TypeId::Bool), false);
    pin(entry);
    ColRef rem = new_reg(DataType(TypeId::Bool), false);
    pin(rem);
    ColRef sel = new_reg(DataType(TypeId::Bool), false);
    pin(sel);
    mask(nullptr, nullptr, 0, &entry);
    mask(nullptr, nullptr, 0, &rem);
    auto select = [&](const ColRef& cond, const Expr& value) {
      ColRef v = cast_to(compile(value), e.type);
      VInstr ins = blank(OP_SELECT, vk);
      ins.a = resolve(cond);
      ins.b = resolve(v);
      ins.dst = dst.op;
      ins.flags = IF_NULLCHK;
      emit(ins);
      dst.keep.insert(dst.keep.end(), v.keep.begin(), v.keep.end());
      release(v);
    };
    for (size_t w = 0; w < npairs; w++) {
      ColRef c = compile(*e.args[2 * w]);  // for the remaining rows
      pin(c);
      mask(&rem, &c, 0, &sel);             // its THEN: for the remaining rows where it is TRUE
      select(sel, *e.args[2 * w + 1]);
      mask(&rem, &c, 1, &rem);             // the rows left for the next WHEN / the ELSE
      unpin(c);
      release(c);
    }
    if (e.has_else) select(rem, *e.args.back());
    mask(&entry, nullptr, 0, nullptr);
    for (ColRef* r : {&entry, &rem, &sel}) {
      unpin(*r);
      release(*r);
    }
    unpin(dst);
    return dst;
  }

 public:
  ColRef cast_to(const ColRef& a, const DataType& to) {
    if (a.type == to) return a;
    PK from = a.type.pk(), dst = to.pk();
    auto simple = [&](uint8_t op, uint8_t t, int imm, uint8_t aux, bool may_null) {
      ColRef r = new_reg(to, a.nullable || may_null);
      r.keep = a.keep;
      VInstr ins = blank(op, t);
      ins.a = resolve(a);
      ins.dst = r.op;
      ins.imm = imm;
      ins.aux = aux;
      if (a.nullable) ins.flags |= IF_NULLCHK;
      emit(ins);
      release(a);
      return r;
    };
    if (a.type.id == TypeId::Null) {
      LitValue l;
      l.is_null = true;
      return literal(to, l);
    }
    if (dst == PK::I64 && (from == PK::I64 || from == PK::Bool)) {
      if (from == PK::Bool) return simple(OP_MOV, VK_I64, 0, 0, false);
      // a value of a signed type going to UInt64, or a UInt64 going to any other type: a negative 64-bit image is out
      // of range (a negative value, or one at or above 2^63)
      const bool sign_check = (to.id == TypeId::UInt64 && a.type.is_signed_int()) || (a.type.id == TypeId::UInt64 && to.is_integer() && to.id != TypeId::UInt64);
      if (!sign_check && (to.width() >= 8 || (a.type.width() <= to.width() && a.type.is_signed_int() == to.is_signed_int()))) {
        ColRef o = a;
        o.type = to;
        return o;
      }
      return simple(OP_NARROW_I64, VK_I64, sign_check ? 1 : 0, phys_of(to), true);
    }
    if (dst == PK::Bool && from == PK::I64) {
      ColRef zero = literal(a.type, LitValue());
      ColRef r = compare(BinOp::Ne, a, zero);
      release(a);
      return r;
    }
    if (dst == PK::F64 && from == PK::I64) return simple(OP_CAST_I64_F64, VK_F64, to.id == TypeId::Float32 ? 1 : 0, a.type.id == TypeId::UInt64 ? PH_U64 : 0, false);
    if (dst == PK::F64 && from == PK::I128) return simple(OP_CAST_I128_F64, VK_F64, a.type.scale, 0, false);
    if (dst == PK::F64 && from == PK::F64) {
      ColRef o = a;
      o.type = to;
      return o;
    }
    if (dst == PK::I64 && from == PK::F64) {
      ColRef r = simple(OP_CAST_F64_I64, VK_I64, 0, to.id == TypeId::UInt64 ? PH_U64 : 0, true);
      if (to.width() < 8) {
        ColRef n = new_reg(to, true);
        VInstr ins = blank(OP_NARROW_I64, VK_I64);
        ins.a = resolve(r);
        ins.dst = n.op;
        ins.aux = phys_of(to);
        ins.flags = IF_NULLCHK;
        emit(ins);
        release(r);
        return n;
      }
      return r;
    }
    if (dst == PK::I128 && from == PK::I64) {
      ColRef r = simple(OP_CAST_I64_I128, VK_I128, to.scale, a.type.id == TypeId::UInt64 ? PH_U64 : 0, false);
      prog.code[prog.n_instr - 1].flags |= IF_CHECKED;
      // value must fit the target precision (error, like arrow's cast of ints to decimal) [EXT]
      VInstr chk = blank(OP_CHECK_PRECISION, VK_I128);
      chk.a = r.op;
      chk.dst = r.op;
      chk.aux = to.precision;
      chk.flags = IF_CHECKED | (r.nullable ? IF_NULLCHK : 0);
      emit(chk);
      return r;
    }
    if (dst == PK::I128 && from == PK::I128) {
      int ds = to.scale - a.type.scale;
      ColRef r = simple(ds >= 0 ? OP_CAST_I128_I128_UP : OP_CAST_I128_I128_DOWN, VK_I128, ds >= 0 ? ds : -ds, 0, true);
      if (ds > 0) prog.code[prog.n_instr - 1].flags |= IF_CHECKED;
      VInstr chk = blank(OP_CHECK_PRECISION, VK_I128);
      chk.a = r.op;
      chk.dst = r.op;
      chk.aux = to.precision;
      chk.flags = IF_NULLCHK;
      emit(chk);
      return r;
    }
    if (dst == PK::I128 && from == PK::F64) {
      ColRef r = simple(OP_CAST_F64_I128, VK_I128, to.scale, 0, true);
      VInstr chk = blank(OP_CHECK_PRECISION, VK_I128);  // beyond the precision: NULL (safe cast)
      chk.a = r.op;
      chk.dst = r.op;
      chk.aux = to.precision;
      chk.flags = IF_NULLCHK;
      emit(chk);
      return r;
    }
    if (dst == PK::I64 && from == PK::I128) {
      ColRef r = simple(OP_CAST_I128_I64, VK_I64, a.type.scale, to.id == TypeId::UInt64 ? PH_U64 : 0, true);
      if (to.width() < 8) {
        ColRef n = new_reg(to, true);
        VInstr ins = blank(OP_NARROW_I64, VK_I64);
        ins.a = resolve(r);
        ins.dst = n.op;
        ins.aux = phys_of(to);
        ins.flags = IF_NULLCHK;
        emit(ins);
        release(r);
        return n;
      }
      return r;
    }
    if (dst == PK::Str && from == PK::Str) {
      ColRef o = a;
      o.type = to;
      return o;
    }
    if (to.id == TypeId::Utf8) return cast_to_utf8(a);
    throw EngineError(B200_ERR_UNSUPPORTED, "cast " + a.type.str() + " -> " + to.str());
  }
};

}  // namespace b200
