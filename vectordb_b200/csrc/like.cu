// LIKE filters on the device (DESIGN.md §K3): the string dictionary mirror and the wildcard-match kernel.
//
// Reference: ExprEvaluator::LogicalEvaluate, NodeType::LIKE (engine/query/expr/expr_evaluator.cpp:229-241, :14-35).
// An empty pattern matches only the empty subject and the pattern "%" matches every subject.  Otherwise the pattern is
// regex-escaped, '%' becomes ".*", '_' becomes "." and std::regex_match runs (ECMAScript, on bytes).  So every byte but
// '%' and '_' is a literal, the match is case-sensitive and covers the whole subject, and since '.' of libstdc++'s
// ECMAScript mode matches any byte except '\n' and '\r', neither wildcard crosses a line terminator.
//
// Matcher: every '\n' / '\r' of the subject must line up, in order, with the same byte of the pattern.  Split both
// there; each segment pair is then a plain wildcard match, done greedily with one backtrack point (the last '%'):
// O(|s| |p|) time, O(1) space, no recursion, no length limit.
//
// Kernel: one thread per item, the bits of a warp's 32 items gathered with one ballot.  An item takes its subject and
// its pattern each from a constant code, from its own index (bit per dictionary code) or from a column's code of
// its row (bit per row).  Every LIKE node of a call is one job of the same launch.
#include <algorithm>
#include <climits>

#include "internal.h"

namespace eps {

enum LikeSrc : int32_t { LK_CONST, LK_ITEM, LK_COL };

struct LikeJob {
  int64_t item_base;  // first item of the job in the launch (a multiple of 32)
  int64_t n_items;
  int64_t word;       // first word of the job's bits in the call's bitmap buffer
  uint32_t* out;      // = that buffer + word: ceil(n_items / 32) words
  const int32_t* col_s;
  const int32_t* col_p;
  int32_t s_code, p_code;
  int32_t s_src, p_src;
};

__device__ __forceinline__ bool is_line_end(uint8_t c) { return c == '\n' || c == '\r'; }

// Wildcard match of one segment pair (no line terminator in either).
__device__ __forceinline__ bool segment_match(const uint8_t* __restrict__ s, int64_t ns, const uint8_t* __restrict__ p,
                                              int64_t np) {
  int64_t i = 0, j = 0, star = -1, mark = 0;
  while (i < ns) {
    const uint8_t c = j < np ? p[j] : 0;
    if (j < np && c == '%') {
      star = j++;
      mark = i;
    } else if (j < np && (c == '_' || c == s[i])) {
      ++i;
      ++j;
    } else if (star >= 0) {
      j = star + 1;
      i = ++mark;
    } else {
      return false;
    }
  }
  while (j < np && p[j] == '%') ++j;
  return j == np;
}

__device__ bool like_match(const uint8_t* __restrict__ s, int64_t ns, const uint8_t* __restrict__ p, int64_t np) {
  if (np == 0) return ns == 0;
  if (np == 1 && p[0] == '%') return true;
  int64_t i = 0, j = 0;
  for (;;) {
    int64_t ie = i, je = j;
    while (ie < ns && !is_line_end(s[ie])) ++ie;
    while (je < np && !is_line_end(p[je])) ++je;
    if (!segment_match(s + i, ie - i, p + j, je - j)) return false;
    if (ie == ns || je == np) return ie == ns && je == np;
    if (s[ie] != p[je]) return false;
    i = ie + 1;
    j = je + 1;
  }
}

__global__ void like_kernel(const LikeJob* __restrict__ jobs, int n_jobs, int64_t n_total, const int64_t* __restrict__ off,
                            const uint8_t* __restrict__ bytes) {
  const int64_t t = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (t >= n_total) return;  // n_total is a multiple of 32: whole warps leave
  int j = 0;
  while (j + 1 < n_jobs && jobs[j + 1].item_base <= t) ++j;
  const LikeJob& jb = jobs[j];
  const int64_t item = t - jb.item_base;
  bool m = false;
  if (item < jb.n_items) {
    const int64_t sc = jb.s_src == LK_CONST ? jb.s_code : (jb.s_src == LK_ITEM ? item : jb.col_s[item]);
    const int64_t pc = jb.p_src == LK_CONST ? jb.p_code : (jb.p_src == LK_ITEM ? item : jb.col_p[item]);
    const int64_t s0 = off[sc], p0 = off[pc];
    m = like_match(bytes + s0, off[sc + 1] - s0, bytes + p0, off[pc + 1] - p0);
  }
  const unsigned w = __ballot_sync(kFull, m);
  if ((threadIdx.x & 31) == 0 && item < jb.n_items) jb.out[item >> 5] = w;
}

int dict_append(Index* ix, int64_t first_code, int64_t count, const int64_t* offsets, const char* bytes) {
  StrDict& d = ix->dict;
  if (count < 0) return fail(EPS_ERR_INVALID_ARGUMENT, "negative string count");
  if (first_code != d.n)
    return fail(EPS_ERR_INVALID_ARGUMENT, "dictionary strings must be appended without gaps: first_code must equal the " +
                                              std::to_string(d.n) + " codes already mirrored");
  if (count == 0) return EPS_OK;
  if (!offsets || !bytes) return fail(EPS_ERR_INVALID_ARGUMENT, "null offsets / bytes");
  for (int64_t i = 0; i < count; ++i)
    if (offsets[i + 1] < offsets[i]) return fail(EPS_ERR_INVALID_ARGUMENT, "string offsets go backwards");
  if (offsets[0] < 0) return fail(EPS_ERR_INVALID_ARGUMENT, "negative string offset");
  if (d.n + count > INT32_MAX) return fail(EPS_ERR_UNSUPPORTED, "more than 2^31 - 1 dictionary codes (codes are int32)");
  const int64_t span = offsets[count] - offsets[0];
  // room for `need` elements, keeping the first `keep`: doubling, at least 256 (allocated on the first append)
  auto room = [&](Mem& m, size_t elem, int64_t need, int64_t keep) {
    const int64_t cap = static_cast<int64_t>(m.cap / elem);
    if (need <= cap && m.p) return EPS_OK;
    const int64_t want = std::max<int64_t>(need, std::max<int64_t>(2 * cap, 256));
    return m.grow(static_cast<size_t>(want) * elem, static_cast<size_t>(keep) * elem, ix->stream);
  };
  EPS_TRY(room(d.d_off, 8, d.n + count + 1, d.n + 1));
  EPS_TRY(room(d.d_bytes, 1, d.bytes + span, d.bytes));
  std::vector<int64_t> off(static_cast<size_t>(count) + (d.n == 0 ? 1 : 0));
  size_t k = 0;
  if (d.n == 0) off[k++] = 0;
  for (int64_t i = 1; i <= count; ++i) off[k++] = d.bytes + (offsets[i] - offsets[0]);
  EPS_CUDA(cudaMemcpyAsync(d.d_off + (d.n == 0 ? 0 : d.n + 1), off.data(), off.size() * 8, cudaMemcpyHostToDevice, ix->stream));
  if (span > 0)
    EPS_CUDA(cudaMemcpyAsync(d.d_bytes + d.bytes, bytes + offsets[0], static_cast<size_t>(span), cudaMemcpyHostToDevice, ix->stream));
  EPS_CUDA(cudaStreamSynchronize(ix->stream));
  d.n += count;
  d.bytes += span;
  return EPS_OK;
}

int check_like(const Index* ix, const FilterProg& prog) {
  for (int i = 0; i < prog.n; ++i) {
    const FNode& nd = prog.nodes[i];
    if (nd.type != NT_LIKE) continue;
    for (const int c : {static_cast<int>(nd.left), static_cast<int>(nd.right)}) {
      const FNode& ch = prog.nodes[c];
      if (ch.type == NT_StringConst) {
        if (!(ch.value >= 0.0 && ch.value < static_cast<double>(ix->dict.n)))
          return fail(EPS_ERR_INVALID_ARGUMENT, "LIKE literal code outside the mirrored string dictionary "
                                                "(append the literal with eps_index_append_string_dictionary)");
      } else {
        const StrCol& sc = ix->str_cols[ch.field_offset];
        if (sc.any_negative || sc.max_code >= ix->dict.n)
          return fail(EPS_ERR_INVALID_ARGUMENT, "LIKE reads a string column with codes outside the mirrored string dictionary");
      }
    }
  }
  return EPS_OK;
}

int bind_like(Index* ix, FilterProg* progs, int n, uint64_t* launches) {
  std::vector<LikeJob> jobs;
  std::vector<int64_t> base(static_cast<size_t>(n), -1);
  int64_t words = 0, items = 0;
  for (int p = 0; p < n; ++p) {
    FilterProg& pr = progs[p];
    for (int i = 0; i < pr.n; ++i) {
      FNode& nd = pr.nodes[i];
      if (nd.type != NT_LIKE) continue;
      if (base[p] < 0) base[p] = words;
      const FNode& l = pr.nodes[nd.left];
      const FNode& r = pr.nodes[nd.right];
      LikeJob jb{};
      jb.s_src = l.type == NT_StringConst ? LK_CONST : LK_ITEM;
      jb.p_src = r.type == NT_StringConst ? LK_CONST : LK_ITEM;
      jb.s_code = l.type == NT_StringConst ? static_cast<int32_t>(l.value) : 0;
      jb.p_code = r.type == NT_StringConst ? static_cast<int32_t>(r.value) : 0;
      if (jb.s_src == LK_CONST && jb.p_src == LK_CONST) {
        jb.n_items = 1;
      } else if (jb.s_src == LK_ITEM && jb.p_src == LK_ITEM) {  // both columns: one bit per row
        jb.s_src = jb.p_src = LK_COL;
        jb.col_s = ix->str_cols[l.field_offset].d_codes;
        jb.col_p = ix->str_cols[r.field_offset].d_codes;
        jb.n_items = ix->n_rows;
      } else {  // one column: one bit per dictionary code
        jb.n_items = ix->dict.n;
      }
      const int64_t w = (jb.n_items + 31) / 32;
      if (words - base[p] + w > INT32_MAX)
        return fail(EPS_ERR_UNSUPPORTED, "the LIKE bitmaps of one expression exceed 2^31 words");
      nd.pad = static_cast<int32_t>(words - base[p]);
      jb.word = words;
      jb.item_base = items;
      items += w * 32;
      words += w;
      if (jb.n_items > 0) jobs.push_back(jb);
    }
  }
  if (words == 0) return EPS_OK;
  EPS_TRY(ix->s_like.reserve(static_cast<size_t>(words) * 4));
  uint32_t* bits = ix->s_like.as<uint32_t>();
  for (int p = 0; p < n; ++p)
    if (base[p] >= 0) progs[p].like_bits = bits + base[p];
  if (jobs.empty()) return EPS_OK;
  for (auto& jb : jobs) jb.out = bits + jb.word;
  EPS_TRY(ix->s_like_jobs.reserve(jobs.size() * sizeof(LikeJob)));
  // pageable source: the runtime stages it before returning, so `jobs` may go out of scope
  EPS_CUDA(cudaMemcpyAsync(ix->s_like_jobs.p, jobs.data(), jobs.size() * sizeof(LikeJob), cudaMemcpyHostToDevice, ix->stream));
  constexpr int kThreads = 256;
  like_kernel<<<static_cast<unsigned>((items + kThreads - 1) / kThreads), kThreads, 0, ix->stream>>>(
      ix->s_like_jobs.as<LikeJob>(), static_cast<int>(jobs.size()), items, ix->dict.d_off,
      ix->dict.d_bytes.as<const uint8_t>());
  EPS_CUDA(cudaGetLastError());
  if (launches) *launches += 1;
  return EPS_OK;
}

}  // namespace eps
