// Canonical text of a typed stage plan: the PlanNode tree plan.hpp built, written back as IR JSON with every column
// reference resolved to an index and every node annotated with its output schema.  Two IR texts describe the same plan
// exactly when their canonical texts are equal -- what tests/test_plan_proto.py compares (IR written by the harness vs IR
// decoded from protobuf plan bytes), and what the fixture generator reads to encode a plan as the reference's protobuf
// (it needs the resolved indices and the intermediate schemas).  Diagnostic / test surface only.
#pragma once
#include <string>

#include "plan.hpp"
#include "plan_proto.hpp"

namespace b200 {

inline std::string dump_schema(const Schema& s) {
  std::string o = "[";
  for (size_t i = 0; i < s.size(); i++)
    o += std::string(i ? "," : "") + "{\"name\":" + pbp::jstr(s[i].name) + ",\"type\":" + type_json(s[i].type) + ",\"nullable\":" + (s[i].nullable ? "true" : "false") + "}";
  return o + "]";
}

inline std::string dump_expr(const ExprPtr& e) {
  static const char* ops[] = {"+", "-", "*", "/", "%", "=", "!=", "<", "<=", ">", ">=", "and", "or", "&", "|", "^", "<<", ">>", "~", "~*", "!~", "!~*", "||"};
  auto list = [&](size_t from) {
    std::string o = "[";
    for (size_t i = from; i < e->args.size(); i++) o += (i > from ? "," : "") + dump_expr(e->args[i]);
    return o + "]";
  };
  const std::string ty = ",\"type\":" + type_json(e->type);
  switch (e->kind) {
    case Expr::Col: return "{\"col\":" + std::to_string(e->col) + ",\"name\":" + pbp::jstr(e->name) + ty + "}";
    case Expr::Lit: {
      std::string v = "null";
      if (!e->lit.is_null) {
        switch (e->type.pk()) {
          case PK::Bool: v = e->lit.i ? "true" : "false"; break;
          case PK::I64: v = std::to_string(e->lit.i); break;
          case PK::F64: {
            char b[64];
            snprintf(b, sizeof b, "%.17g", e->lit.f);
            v = b;
            break;
          }
          case PK::I128: v = "\"" + pbp::i128_to_string(e->lit.d) + "\""; break;
          case PK::Str: v = pbp::jstr(e->lit.s); break;
        }
      }
      return "{\"lit\":{\"t\":" + type_json(e->type) + ",\"v\":" + v + "}}";
    }
    case Expr::Bin: return std::string("{\"bin\":\"") + ops[(int)e->op] + "\",\"l\":" + dump_expr(e->args[0]) + ",\"r\":" + dump_expr(e->args[1]) + ty + "}";
    case Expr::Not: return "{\"not\":" + dump_expr(e->args[0]) + "}";
    case Expr::Neg: return "{\"neg\":" + dump_expr(e->args[0]) + ty + "}";
    case Expr::IsNull: return "{\"is_null\":" + dump_expr(e->args[0]) + "}";
    case Expr::IsNotNull: return "{\"is_not_null\":" + dump_expr(e->args[0]) + "}";
    case Expr::Cast: return "{\"cast\":" + dump_expr(e->args[0]) + ",\"to\":" + type_json(e->type) + "}";
    case Expr::Case: {
      const size_t pairs = (e->args.size() - (e->has_else ? 1 : 0)) / 2;
      std::string o = "{\"case\":{\"when\":[";
      for (size_t i = 0; i < pairs; i++) o += std::string(i ? "," : "") + "[" + dump_expr(e->args[2 * i]) + "," + dump_expr(e->args[2 * i + 1]) + "]";
      o += "]";
      if (e->has_else) o += ",\"else\":" + dump_expr(e->args.back());
      return o + "}" + ty + "}";
    }
    case Expr::InList: return "{\"in\":" + dump_expr(e->args[0]) + ",\"list\":" + list(1) + ",\"negated\":" + (e->negated ? "true" : "false") + "}";
    case Expr::Like: return "{\"like\":" + dump_expr(e->args[0]) + ",\"pattern\":" + pbp::jstr(e->pattern) + ",\"negated\":" + (e->negated ? "true" : "false") +
                                  (e->case_insensitive ? ",\"case_insensitive\":true" : "") + "}";
    case Expr::Fn: return "{\"fn\":" + pbp::jstr(e->fn) + ",\"args\":" + list(0) + ty + "}";
  }
  return "null";
}

inline std::string dump_ints(const std::vector<int>& v) {
  std::string o = "[";
  for (size_t i = 0; i < v.size(); i++) o += (i ? "," : "") + std::to_string(v[i]);
  return o + "]";
}

inline std::string dump_sort_keys(const std::vector<SortKey>& ks) {
  std::string o = "[";
  for (size_t i = 0; i < ks.size(); i++)
    o += std::string(i ? "," : "") + "{\"expr\":" + dump_expr(ks[i].expr) + ",\"asc\":" + (ks[i].asc ? "true" : "false") + ",\"nulls_first\":" + (ks[i].nulls_first ? "true" : "false") + "}";
  return o + "]";
}

inline std::string dump_plan(const PlanNode& n) {
  static const char* join_types[] = {"Inner", "Left", "Right", "Full", "LeftSemi", "RightSemi", "LeftAnti", "RightAnti"};
  static const char* agg_modes[] = {"Partial", "Final", "FinalPartitioned", "Single", "SinglePartitioned"};
  static const char* agg_fns[] = {"sum", "min", "max", "count", "avg", "var_samp", "var_pop", "stddev_samp", "stddev_pop", "covar_samp", "covar_pop", "corr",
                                  "regr_slope", "regr_intercept", "regr_count", "regr_r2", "regr_avgx", "regr_avgy", "regr_sxx", "regr_syy", "regr_sxy",
                                  "bool_and", "bool_or", "bit_and", "bit_or", "bit_xor", "first_value", "last_value"};
  std::string o = "{\"op\":" + pbp::jstr(n.op_name);
  auto child = [&](size_t i) { return dump_plan(*n.children[i]); };
  switch (n.op) {
    case PlanNode::Scan: o += ",\"table\":" + pbp::jstr(n.table) + ",\"projection\":" + dump_ints(n.scan_projection); break;
    case PlanNode::ShuffleReader: o += ",\"stage_id\":" + std::to_string(n.reader_stage_id) + ",\"broadcast\":" + (n.broadcast ? "true" : "false"); break;
    case PlanNode::Filter:
      o += ",\"predicate\":" + dump_expr(n.predicate);
      if (n.has_projection) o += ",\"projection\":" + dump_ints(n.projection);
      if (n.fetch >= 0) o += ",\"fetch\":" + std::to_string(n.fetch);
      o += ",\"input\":" + child(0);
      break;
    case PlanNode::Projection: {
      o += ",\"exprs\":[";
      for (size_t i = 0; i < n.exprs.size(); i++) o += std::string(i ? "," : "") + "{\"expr\":" + dump_expr(n.exprs[i].expr) + ",\"name\":" + pbp::jstr(n.exprs[i].name) + "}";
      o += "],\"input\":" + child(0);
      break;
    }
    case PlanNode::Aggregate: {
      o += std::string(",\"mode\":\"") + agg_modes[(int)n.agg_mode] + "\",\"group_by\":[";
      for (size_t i = 0; i < n.group_by.size(); i++)
        o += std::string(i ? "," : "") + "{\"expr\":" + dump_expr(n.group_by[i].expr) + ",\"name\":" + pbp::jstr(n.group_by[i].name) + "}";
      if (!n.grouping_sets.empty()) {
        o += "],\"grouping_sets\":[";
        for (size_t s = 0; s < n.grouping_sets.size(); s++) {
          o += s ? ",[" : "[";
          for (size_t k = 0; k < n.group_by.size(); k++) o += std::string(k ? "," : "") + (((n.grouping_sets[s] >> k) & 1u) ? "true" : "false");
          o += "]";
        }
      }
      o += "],\"aggr\":[";
      for (size_t i = 0; i < n.aggs.size(); i++) {
        const AggExpr& a = n.aggs[i];
        o += std::string(i ? "," : "") + "{\"fn\":\"" + agg_fns[(int)a.fn] + "\",\"name\":" + pbp::jstr(a.name) + ",\"args\":[" + (a.arg ? dump_expr(a.arg) : std::string()) + (a.arg2 ? "," + dump_expr(a.arg2) : std::string()) +
             "],\"input_type\":" + type_json(a.input_type) + ",\"sum_type\":" + type_json(a.sum_type) + ",\"result_type\":" + type_json(a.result_type) +
             (agg_is_first_last(a.fn) ? ",\"order_by\":" + dump_sort_keys(a.order_by) + ",\"ignore_nulls\":" + (a.ignore_nulls ? "true" : "false") : std::string()) + "}";
      }
      o += "],\"input\":" + child(0);
      break;
    }
    case PlanNode::HashJoin: {
      o += std::string(",\"join_type\":\"") + join_types[(int)n.join_type] + "\"";
      if (!n.nested_loop) {  // a nested-loop join has neither a partition mode of its own nor keys
        o += ",\"mode\":" + pbp::jstr(n.partition_mode) + ",\"on\":[";
        for (size_t i = 0; i < n.on.size(); i++) o += std::string(i ? "," : "") + "[" + dump_expr(n.on[i].first) + "," + dump_expr(n.on[i].second) + "]";
        o += "]";
        if (n.null_equals_null) o += ",\"null_equals_null\":true";
      }
      if (n.join_filter) o += ",\"filter\":" + dump_expr(n.join_filter);
      if (n.has_projection) o += ",\"projection\":" + dump_ints(n.projection);
      if (!n.sort_keys.empty()) o += ",\"sort_keys\":" + dump_sort_keys(n.sort_keys);
      o += ",\"left\":" + child(0) + ",\"right\":" + child(1);
      break;
    }
    case PlanNode::Sort:
    case PlanNode::SortPreservingMerge:
      o += ",\"expr\":" + dump_sort_keys(n.sort_keys) + ",\"preserve_partitioning\":" + (n.preserve_partitioning ? "true" : "false");
      if (n.fetch >= 0) o += ",\"fetch\":" + std::to_string(n.fetch);
      o += ",\"input\":" + child(0);
      break;
    case PlanNode::Passthrough: o += ",\"input\":" + child(0); break;
    case PlanNode::Window: {
      static const char* bounds[] = {"unbounded_preceding", "preceding", "current_row", "following", "unbounded_following"};
      auto bound = [&](const WindowBound& b) {
        return std::string("{\"kind\":\"") + bounds[b.kind] + "\"" + (b.kind == 1 || b.kind == 3 ? ",\"n\":" + std::to_string(b.n) : std::string()) + "}";
      };
      o += std::string(",\"mode\":") + (n.window_sorted ? "\"sorted\"" : "null") + ",\"partition_keys\":[";
      for (size_t i = 0; i < n.window_partition.size(); i++) o += (i ? "," : "") + dump_expr(n.window_partition[i]);
      o += "],\"order_by\":" + dump_sort_keys(n.window_order) + ",\"window_expr\":[";
      for (size_t i = 0; i < n.window_exprs.size(); i++) {
        const WindowExpr& w = n.window_exprs[i];
        o += std::string(i ? "," : "") + "{\"fn\":" + pbp::jstr(w.fn_name) + ",\"name\":" + pbp::jstr(w.name) + ",\"args\":[";
        for (size_t k = 0; k < w.args.size(); k++) o += (k ? "," : "") + dump_expr(w.args[k]);
        o += "],\"n\":" + std::to_string(w.n);
        if (w.default_value) o += ",\"default\":" + dump_expr(w.default_value);
        o += std::string(",\"frame\":{\"units\":\"") + (w.frame.range ? "range" : "rows") + "\",\"start\":" + bound(w.frame.start) + ",\"end\":" + bound(w.frame.end) + "}";
        o += ",\"result_type\":" + type_json(w.result_type) + "}";
      }
      o += "],\"input\":" + child(0);
      break;
    }
    case PlanNode::Limit: o += ",\"fetch\":" + std::to_string(n.fetch) + ",\"skip\":" + std::to_string(n.skip) + ",\"input\":" + child(0); break;
    case PlanNode::ShuffleWriter: {
      o += ",\"job_id\":" + pbp::jstr(n.job_id) + ",\"stage_id\":" + std::to_string(n.stage_id) + ",\"sort_shuffle\":" + (n.sort_shuffle ? "true" : "false");
      if (n.n_out_partitions > 0) {
        o += ",\"partitioning\":{\"hash\":[";
        for (size_t i = 0; i < n.part_exprs.size(); i++) o += (i ? "," : "") + dump_expr(n.part_exprs[i]);
        o += "],\"n\":" + std::to_string(n.n_out_partitions) + "}";
      }
      o += ",\"input\":" + child(0);
      break;
    }
  }
  return o + ",\"schema\":" + dump_schema(n.schema) + "}";
}

}  // namespace b200
