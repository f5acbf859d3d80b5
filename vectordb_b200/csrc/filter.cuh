// Device-side filter evaluation (SURVEY.md §8a row A12).
//
// Semantics follow query::expr::ExprEvaluator::LogicalEvaluate / NumEvaluate
// (engine/query/expr/expr_evaluator.cpp:170-258, :127-164) for numeric / bool predicates:
//  * ints are widened to int64 then double, floats to double, comparisons in double;
//  * a BoolAttr is "non-zero byte" (:56-59 casts the byte VALUE to a pointer);
//  * NOT / AND / OR / bool-typed EQ,NE evaluate their children through the two-argument overload,
//    i.e. with distance 0 (:166-168,:184,:204-211) — "@distance" only sees the real distance when
//    the ROOT is a numeric comparison.  Hence one effective distance per evaluation (root_dist()).
//  * strings (SURVEY.md §8f-4): a string column is mirrored as DICTIONARY CODES (int32 per row, one dictionary per
//    table so codes compare across columns); StringAttr reads the row's code, StringConst carries the literal's
//    code (-1: literal absent from the dictionary, equal to no row), and string EQ / NE (:186-190) compare codes.
//    IN (:176-185) is lowered by the caller to an OR of EQs; string concatenation stays out of scope.
//  * LIKE (:229-241): the strings behind the codes are mirrored as a dictionary (StrDict), and the match kernel
//    (like.cu) evaluates every LIKE node of a call once, before the search kernels, into a bitmap: one bit per
//    dictionary code when one side is a constant, one bit per row when both sides are columns, one bit when both are
//    constants.  prog_run only reads the bit: FNode.pad is the node's word offset in FilterProg.like_bits and
//    FNode.field_offset says which bit (kLikeByRow: bit `row`; kLikeConst: bit 0; otherwise the index of the child
//    whose value is the code to read).
// The parser emits children before parents, so one forward pass over the node array evaluates the
// tree without recursion.
#pragma once
#include "common.cuh"

namespace eps {

constexpr int kMaxFilterNodes = 64;
constexpr int kMaxStringCols = 8;
constexpr int kLikeByRow = -1;  // FNode.field_offset of a LIKE whose two sides are columns
constexpr int kLikeConst = -2;  // ... whose two sides are constants

enum NodeType : int {  // query/expr/expr_types.hpp:11-48
  NT_Invalid, NT_IntConst, NT_StringConst, NT_DoubleConst, NT_BoolConst, NT_Int1Attr, NT_Int2Attr, NT_Int4Attr,
  NT_Int8Attr, NT_StringAttr, NT_DoubleAttr, NT_FloatAttr, NT_BoolAttr, NT_GeoPointAttr, NT_Add, NT_Subtract,
  NT_Multiply, NT_Divide, NT_Module, NT_LT, NT_LTE, NT_EQ, NT_GT, NT_GTE, NT_NE, NT_AND, NT_OR, NT_NOT,
  NT_FunctionCall, NT_LIKE, NT_SumAgg, NT_MinAgg, NT_MaxAgg, NT_CountAgg, NT_IN, NT_ListString
};
enum ValueType : int { VT_STRING, VT_INT, VT_DOUBLE, VT_BOOL, VT_GEO_POINT, VT_LIST_STRING };

// Compact device form of eps_filter_node.
struct FNode {
  int16_t type;
  int16_t vtype;
  int16_t left, right;
  int32_t field_offset;
  int32_t pad;    // LIKE: word offset of the node's bits in FilterProg.like_bits
  double value;  // IntConst (as double, like NumEvaluate's static_cast), DoubleConst, BoolConst(0/1)
};

struct FilterProg {
  int n;              // 0 = no filter (root index -1 => true, expr_evaluator.cpp:171-173)
  int uses_distance;  // any node reads "@distance"
  int root_uses_dist; // root is a numeric comparison (the only place the real distance is visible)
  int pad;
  const int32_t* str_col[kMaxStringCols];  // device columns of dictionary codes (filled when the program is lowered)
  const uint32_t* like_bits;               // LIKE bitmaps of this program (filled by bind_like)
  FNode nodes[kMaxFilterNodes];
};

// Host: validate + lower eps_filter_node[] to FilterProg.  Returns EPS_* code.
int lower_filter(const eps_filter_node* nodes, int64_t n, FilterProg* out);

// One forward pass over the program; the root's numeric and logical values come back through *num_out / *bool_out.
// `dist` is what "@distance" reads.
__device__ __forceinline__ void prog_run(const FilterProg& p, const char* __restrict__ attrs, int64_t stride, int64_t row,
                                         double dist, double* num_out, bool* bool_out) {
  double num[kMaxFilterNodes];
  bool bl[kMaxFilterNodes];
  const char* base = attrs + row * stride;
  for (int i = 0; i < p.n; ++i) {
    const FNode& nd = p.nodes[i];
    double v = 0.0;
    bool b = false;
    switch (nd.type) {
      case NT_IntConst:
      case NT_StringConst:
      case NT_DoubleConst: v = nd.value; break;
      case NT_StringAttr: v = static_cast<double>(p.str_col[nd.field_offset][row]); break;
      case NT_BoolConst: b = nd.value != 0.0; break;
      case NT_Int1Attr: v = static_cast<double>(*reinterpret_cast<const int8_t*>(base + nd.field_offset)); break;
      case NT_Int2Attr: { int16_t x; memcpy(&x, base + nd.field_offset, 2); v = static_cast<double>(x); break; }
      case NT_Int4Attr: { int32_t x; memcpy(&x, base + nd.field_offset, 4); v = static_cast<double>(x); break; }
      case NT_Int8Attr: { int64_t x; memcpy(&x, base + nd.field_offset, 8); v = static_cast<double>(x); break; }
      case NT_DoubleAttr:
        if (nd.field_offset == -2) v = dist;
        else { double x; memcpy(&x, base + nd.field_offset, 8); v = x; }
        break;
      case NT_FloatAttr:
        if (nd.field_offset == -2) v = dist;
        else { float x; memcpy(&x, base + nd.field_offset, 4); v = static_cast<double>(x); }
        break;
      case NT_BoolAttr: b = *(base + nd.field_offset) != 0; break;
      case NT_NOT: b = !bl[nd.left]; break;
      case NT_Add: v = num[nd.left] + num[nd.right]; break;
      case NT_Subtract: v = num[nd.left] - num[nd.right]; break;
      case NT_Multiply: v = num[nd.left] * num[nd.right]; break;
      case NT_Divide: v = num[nd.left] / num[nd.right]; break;
      case NT_Module: v = fmod(num[nd.left], num[nd.right]); break;
      case NT_AND: b = bl[nd.left] && bl[nd.right]; break;
      case NT_OR: b = bl[nd.left] || bl[nd.right]; break;
      case NT_EQ:
      case NT_NE:
        if (p.nodes[nd.left].vtype == VT_BOOL) b = (bl[nd.left] == bl[nd.right]);
        else b = (num[nd.left] == num[nd.right]);
        if (nd.type == NT_NE) b = !b;
        break;
      case NT_GT: b = num[nd.left] > num[nd.right]; break;
      case NT_GTE: b = num[nd.left] >= num[nd.right]; break;
      case NT_LT: b = num[nd.left] < num[nd.right]; break;
      case NT_LTE: b = num[nd.left] <= num[nd.right]; break;
      case NT_LIKE: {
        const int64_t bit = nd.field_offset >= 0 ? static_cast<int64_t>(num[nd.field_offset])
                                                 : (nd.field_offset == kLikeByRow ? row : 0);
        b = (p.like_bits[nd.pad + (bit >> 5)] >> (bit & 31)) & 1u;
        break;
      }
      default: break;
    }
    num[i] = v;
    bl[i] = b;
  }
  *num_out = num[p.n - 1];
  *bool_out = bl[p.n - 1];
}

// LogicalEvaluate(root, row, distance) (:170-258): the distance is visible only when the root is a numeric comparison.
__device__ __forceinline__ bool filter_eval(const FilterProg& p, const char* __restrict__ attrs, int64_t stride,
                                            int64_t row, float distance) {
  if (p.n == 0) return true;
  double nv;
  bool bv;
  prog_run(p, attrs, stride, row, p.root_uses_dist ? static_cast<double>(distance) : 0.0, &nv, &bv);
  return bv;
}

// NumEvaluate(root, row, distance) (:127-164): the distance reaches "@distance" at any depth of the arithmetic.
__device__ __forceinline__ double value_eval(const FilterProg& p, const char* __restrict__ attrs, int64_t stride, int64_t row,
                                             double distance) {
  double nv = 0.0;
  bool bv = false;
  if (p.n > 0) prog_run(p, attrs, stride, row, distance, &nv, &bv);
  return nv;
}

}  // namespace eps
