// Reference-side binding: the drop-in for Epsilla's vector-search hot path.
//
// This translation unit is compiled against the reference's UNMODIFIED headers and provides strong
// definitions of exactly three reference symbols, which replace the engine's own (weakened at link time,
// see integration/Makefile) — no reference source file is edited:
//
//   vectordb::engine::execution::VecSearchExecutor::VecSearchExecutor(...)   engine/db/execution/vec_search_executor.cpp:29-73
//   vectordb::engine::execution::VecSearchExecutor::Search(...)              engine/db/execution/vec_search_executor.cpp:833-935
//   vectordb::engine::ANNGraphSegment::BuildFromVectorTable(...)             engine/db/ann_graph_segment.cpp:201-242
//
// Everything else of the class (SearchByAttribute, the public result arrays search_result_ / distance_ /
// dimension_ that TableMVP::Search reads after the call — engine/db/table_mvp.cpp:365-394) stays the
// reference's.  TableMVP, ExecutorPool, DBServer and the filter parser therefore run unchanged; the dense
// vector search and the graph build run on the GPU through include/epsilla_b200.h.
//
// State: one device mirror (eps_index) per (vector table, graph, executor parameters), shared by the
// NumExecutorPerField executors TableMVP creates for a field (engine/db/table_mvp.cpp:72-89) and destroyed
// with the last of them — ownership rides on the executor's own ann_index_ shared_ptr (aliasing
// constructor), so the reference's inline destructor needs no hook.  Calls on a mirror are serialised by a
// mutex; concurrent unfiltered single-query calls from the executors of a pool are COALESCED into one batched
// launch by a leader/follower batch former (SURVEY.md §8f-2) — the reference API stays one query per call.
//
// Scope limits, reported as a non-OK Status instead of silently computing on the CPU: sparse-vector fields
// and string / IN / LIKE / NEARBY filter nodes (SURVEY.md §2 rows 9, 17).
#include <cstdlib>
#include <atomic>
#include <condition_variable>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "db/ann_graph_segment.hpp"
#include "db/execution/vec_search_executor.hpp"
#include "db/index/index.hpp"
#include "epsilla_b200.h"

namespace vectordb {
namespace engine {

namespace b200 {

struct Mirror {
  std::shared_ptr<ANNGraphSegment> ann;  // keeps the graph alive, like the reference member does
  eps_index* ix = nullptr;
  std::mutex mu;
  int metric = EPS_METRIC_L2;
  int64_t dim = 0;
  float* host_vectors = nullptr;
  int64_t capacity = 0;
  int64_t attr_rows = 0;
  const char* attr_ptr = nullptr;
  int64_t L_master = 500, L_local = 500;
  bool prefilter = false;
  int64_t nav = 0;
  int64_t* offsets = nullptr;
  int64_t* nbrs = nullptr;
  // Coalescing of concurrent single-query calls (SURVEY.md 8f-2): unfiltered searches that arrive while
  // another executor's call is in flight are gathered and served by ONE batched launch.
  struct Pending {
    const float* query;
    size_t limit;
    const std::vector<query::expr::ExprNodePtr>* filter;  // the caller's parsed filter (empty = none)
    std::string key;                  // serialised filter: requests with equal keys (and limits) share a launch
    TableSegmentMVP* segment;
    int64_t total;                    // record_number_ snapshot of the caller (:839)
    int64_t n_indexed;
    int num_threads;
    int64_t* ids;
    double* dists;
    int64_t count = 0;
    int rc = EPS_OK;
    bool unsupported = false;         // report NOT_IMPLEMENTED_ERROR instead of DB_UNEXPECTED_ERROR
    std::string err;  // eps_last_error() is thread-local: the leader copies the text for its followers
    bool done = false;
  };
  std::mutex qmu;
  std::condition_variable qcv;
  std::vector<Pending*> waiting;
  bool leader_active = false;
  uint64_t calls = 0, launches = 0;  // Search() calls served / eps_search_batch launches made (coalescing evidence)
  // String columns are mirrored as dictionary codes (SURVEY.md 8f-4): one string -> code dictionary per table,
  // rows encoded incrementally (append-only) the first time a filter reads the column.
  std::unordered_map<std::string, int32_t> dict;
  std::vector<int64_t> str_rows;  // per string column: rows whose codes are on the device
  ~Mirror() {
    if (ix) eps_index_destroy(ix);
  }
};

// The executor's own ann_index_ member owns the mirror: it is an ALIAS of the mirror's shared_ptr that still points
// at the graph.  std::get_deleter on that alias reaches the control block's deleter, which remembers the mirror.
struct MirrorDeleter {
  Mirror* self = nullptr;
  void operator()(Mirror* p) const { delete p; }
};
static Mirror* MirrorOf(const std::shared_ptr<ANNGraphSegment>& alias) {
  const MirrorDeleter* d = std::get_deleter<MirrorDeleter>(alias);
  return d ? d->self : nullptr;
}

// process-wide coalescing evidence (tests): Search() calls served and eps_search_batch launches made
static std::atomic<int64_t> g_calls{0}, g_launches{0};

using Key = std::tuple<const float*, const ANNGraphSegment*, int64_t, int64_t, bool, int, int>;
static std::mutex g_mu;
static std::map<Key, std::weak_ptr<Mirror>> g_mirrors;

static int MetricOf(const DistFunc& f) {
  if (!std::holds_alternative<DenseVecDistFunc<float>>(f)) return -1;
  auto fp = std::get<DenseVecDistFunc<float>>(f);
  auto is = [&](meta::MetricType m) {
    return fp == std::get<DenseVecDistFunc<float>>(GetDistFunc(meta::FieldType::VECTOR_FLOAT, m));
  };
  if (is(meta::MetricType::EUCLIDEAN)) return EPS_METRIC_L2;
  if (is(meta::MetricType::COSINE)) return EPS_METRIC_COSINE;
  if (is(meta::MetricType::DOT_PRODUCT)) return EPS_METRIC_IP;
  return -1;  // a DistFunc the library does not know (e.g. a test wrapper)
}

// Device ordinal of the mirrors: EPSILLA_B200_DEVICE (the reference has no GPU setting to read it from).
static int DeviceOrdinal() {
  static const int dev = [] { const char* e = std::getenv("EPSILLA_B200_DEVICE"); return e ? std::atoi(e) : 0; }();
  return dev;
}

// Byte-exact serialisation of a parsed filter: equal strings <=> the same program on the same columns.
static std::string FilterKey(const std::vector<query::expr::ExprNodePtr>& nodes) {
  std::string k;
  auto put = [&](const void* p, size_t n) { k.append(static_cast<const char*>(p), n); };
  for (const auto& np : nodes) {
    const auto& n = *np;
    const int64_t head[5] = {static_cast<int64_t>(n.node_type), static_cast<int64_t>(n.value_type), static_cast<int64_t>(n.left),
                             static_cast<int64_t>(n.right), n.int_value};
    put(head, sizeof(head));
    put(&n.double_value, sizeof(double));
    k.push_back(n.bool_value ? 1 : 0);
    for (const std::string* sp : {&n.field_name, &n.str_value, &n.function_name}) {
      const uint32_t len = static_cast<uint32_t>(sp->size());
      put(&len, 4);
      k.append(*sp);
    }
    const uint32_t na = static_cast<uint32_t>(n.arguments.size());
    put(&na, 4);
    for (size_t a : n.arguments) { const int64_t v = static_cast<int64_t>(a); put(&v, 8); }
  }
  return k;
}

// Segment state -> device mirror, once per launch (caller holds m->mu): lazily create the index, upload appended
// rows, ship the dirty span of the deleted bitset.
static int Prepare(Mirror* m, TableSegmentMVP* seg, int64_t total, int64_t n_indexed, int num_threads) {
  if (m->ix == nullptr) {
    m->capacity = static_cast<int64_t>(seg->size_limit_);
    if (eps_index_create(&m->ix, m->metric, m->dim, m->host_vectors, m->capacity, DeviceOrdinal()) != EPS_OK) return -1;
    if (eps_index_sync_rows(m->ix, std::max<int64_t>(total, n_indexed)) != EPS_OK) return -1;
    if (n_indexed > 0 && eps_index_set_graph(m->ix, n_indexed, m->offsets, m->nbrs, m->nav) != EPS_OK) return -1;
    if (eps_index_config(m->ix, m->L_master, m->L_local, m->prefilter ? 1 : 0, 0) != EPS_OK) return -1;
    // IntraQueryThreads (config.hpp:18, default 4): 1 = the sequential order, > 1 = that many candidates expanded
    // concurrently (the reference's parallel mode is itself not a pure function of its inputs)
    const int width = num_threads >= 8 ? 8 : num_threads >= 4 ? 4 : num_threads >= 2 ? 2 : 1;
    if (eps_index_set_search_width(m->ix, width) != EPS_OK) return -1;
  }
  if (total > eps_index_rows(m->ix) && eps_index_sync_rows(m->ix, total) != EPS_OK) return -1;
  ConcurrentBitset& deleted = *(seg->deleted_);  // (:840)
  const int64_t rows = eps_index_rows(m->ix);
  if (eps_index_set_deleted(m->ix, deleted.data(), (rows + 7) / 8) != EPS_OK) return -1;
  return 0;
}

// filter nodes -> PODs (:841-848), caller holds m->mu: field names resolved through the segment's offset map; string
// work happens here, on the host — new rows of the string columns a filter reads are dictionary-encoded and appended
// to the device mirror, literals become codes, `x IN (a, b, ..)` becomes `x = a OR x = b ..`.
// Returns 0, -1 (library error, text in eps_last_error) or -2 (out of scope, text in *why).
static int LowerFilter(Mirror* m, TableSegmentMVP* seg, const std::vector<query::expr::ExprNodePtr>& src,
                       std::vector<eps_filter_node>* out, std::string* why) {
  using query::expr::NodeType;
  using query::expr::ValueType;
  out->clear();
  if (src.empty()) return 0;
  const int64_t rows = eps_index_rows(m->ix);
  if (m->attr_rows != rows || m->attr_ptr != seg->attribute_table_) {
    if (eps_index_set_attrs(m->ix, seg->attribute_table_, seg->primitive_offset_, rows) != EPS_OK) return -1;
    m->attr_rows = rows;
    m->attr_ptr = seg->attribute_table_;
  }
  for (const auto& np : src) {
    if (np->node_type != NodeType::StringAttr) continue;
    auto it = seg->field_name_mem_offset_map_.find(np->field_name);
    if (it == seg->field_name_mem_offset_map_.end()) continue;
    const size_t col = it->second;
    if (col >= 8 || col >= seg->var_len_attr_table_.size()) { *why = "more than 8 string columns are out of scope of the GPU path"; return -2; }
    if (m->str_rows.size() <= col) m->str_rows.resize(col + 1, 0);
    if (m->str_rows[col] < rows) {
      std::vector<int32_t> codes;
      codes.reserve(static_cast<size_t>(rows - m->str_rows[col]));
      auto& column = seg->var_len_attr_table_[col];
      for (int64_t r = m->str_rows[col]; r < rows; ++r) {
        const std::string* sv = std::get_if<std::string>(&column[r]);
        auto ins = m->dict.emplace(sv ? *sv : std::string(), static_cast<int32_t>(m->dict.size()));
        codes.push_back(ins.first->second);
      }
      if (eps_index_set_string_codes(m->ix, static_cast<int>(col), m->str_rows[col], codes.data(), static_cast<int64_t>(codes.size())) != EPS_OK)
        return -1;
      m->str_rows[col] = rows;
    }
  }
  std::vector<int64_t> remap(src.size(), -1);  // parser index -> index of the POD holding the node's value
  auto pod = [](NodeType t, ValueType v) {
    eps_filter_node d;
    std::memset(&d, 0, sizeof(d));
    d.node_type = static_cast<int64_t>(t);
    d.value_type = static_cast<int64_t>(v);
    d.left = d.right = -1;
    d.field_offset = -1;
    return d;
  };
  for (size_t i = 0; i < src.size(); ++i) {
    const auto& sn = *src[i];
    if (sn.node_type == NodeType::IN) {  // expr_evaluator.cpp:176-185: last argument is the attribute
      const size_t len = sn.arguments.size();
      if (len < 2) { *why = "malformed IN node"; return -2; }
      const int64_t attr = remap[sn.arguments[len - 1]];
      int64_t acc = -1;
      for (size_t j = 0; j + 1 < len; ++j) {
        eps_filter_node eq = pod(NodeType::EQ, ValueType::BOOL);
        eq.left = attr;
        eq.right = remap[sn.arguments[j]];
        out->push_back(eq);
        const int64_t eq_at = static_cast<int64_t>(out->size()) - 1;
        if (acc < 0) { acc = eq_at; continue; }
        eps_filter_node o = pod(NodeType::OR, ValueType::BOOL);
        o.left = acc;
        o.right = eq_at;
        out->push_back(o);
        acc = static_cast<int64_t>(out->size()) - 1;
      }
      remap[i] = acc;
      continue;
    }
    if (sn.node_type == NodeType::Add && sn.value_type == ValueType::STRING) { *why = "string concatenation in filters is out of scope of the GPU path"; return -2; }
    eps_filter_node d = pod(sn.node_type, sn.value_type);
    const bool unary = sn.node_type == NodeType::NOT;
    const bool leaf = sn.node_type <= NodeType::GeoPointAttr;
    if (!leaf) {
      d.left = sn.left < src.size() ? remap[sn.left] : -1;
      d.right = (!unary && sn.right < src.size()) ? remap[sn.right] : -1;
    }
    d.int_value = sn.int_value;
    d.double_value = sn.double_value;
    d.bool_value = sn.bool_value ? 1 : 0;
    if (sn.node_type == NodeType::StringConst) {
      auto it = m->dict.find(sn.str_value);
      d.int_value = it == m->dict.end() ? -1 : it->second;  // a literal no row carries equals nothing
    }
    if (!sn.field_name.empty()) {
      if (sn.field_name == "@distance") d.field_offset = -2;
      else {
        auto it = seg->field_name_mem_offset_map_.find(sn.field_name);
        if (it != seg->field_name_mem_offset_map_.end()) d.field_offset = static_cast<int64_t>(it->second);
      }
    }
    out->push_back(d);
    remap[i] = static_cast<int64_t>(out->size()) - 1;
  }
  return 0;
}

// Leader/follower batch former.  A caller only enqueues its request (no device work, no mirror lock); the first
// caller becomes the leader and serves, in ONE eps_search_batch call, every request queued at that moment with the
// same limit and the same filter — mirroring the segment (appended rows, dirty delete bytes, new string codes) and
// lowering the filter once per launch.  Requests that arrive while a launch is in flight queue up and form the next
// batch, so a lone caller never waits and concurrent callers are batched by the device's own service time.
// Requests keep their per-call semantics (one query, own result arrays); only the launch is shared.
static void SearchCoalesced(Mirror* m, Mirror::Pending* me) {
  std::unique_lock<std::mutex> q(m->qmu);
  m->waiting.push_back(me);
  if (m->leader_active) {
    m->qcv.wait(q, [&] { return me->done || !m->leader_active; });
    if (me->done) return;
    // the leader left before taking this request: fall through and lead
  }
  m->leader_active = true;
  while (!me->done) {
    std::vector<Mirror::Pending*> batch;
    std::vector<Mirror::Pending*> rest;
    Mirror::Pending* head = m->waiting.front();
    for (auto* p : m->waiting)
      ((p->limit == head->limit && p->segment == head->segment && p->key == head->key) ? batch : rest).push_back(p);
    m->waiting.swap(rest);
    q.unlock();
    const size_t lim = head->limit;
    const int64_t nq = static_cast<int64_t>(batch.size());
    int rc = EPS_OK;
    bool unsupported = false;
    std::string text;
    {
      std::lock_guard<std::mutex> lk(m->mu);  // the index itself is single-threaded
      int64_t total = 0;
      for (auto* p : batch) total = std::max(total, p->total);
      std::vector<eps_filter_node> nodes;
      if (Prepare(m, head->segment, total, head->n_indexed, head->num_threads) != 0) { rc = EPS_ERR_CUDA; text = eps_last_error(); }
      if (rc == EPS_OK) {
        const int lr = LowerFilter(m, head->segment, *head->filter, &nodes, &text);
        if (lr == -1) { rc = EPS_ERR_CUDA; text = eps_last_error(); }
        if (lr == -2) { rc = EPS_ERR_UNSUPPORTED; unsupported = true; }
      }
      if (rc == EPS_OK) {
        const eps_filter_node* fp = nodes.empty() ? nullptr : nodes.data();
        if (nq == 1) {  // no copy through staging buffers for a lone request
          rc = eps_search_batch(m->ix, head->query, 1, static_cast<int64_t>(lim), fp, static_cast<int64_t>(nodes.size()), head->ids, head->dists,
                                &head->count, nullptr);
        } else {
          std::vector<float> qbuf(static_cast<size_t>(nq) * m->dim);
          for (int64_t i = 0; i < nq; ++i) std::memcpy(qbuf.data() + i * m->dim, batch[i]->query, sizeof(float) * m->dim);
          std::vector<int64_t> oi(static_cast<size_t>(nq) * lim), oc(static_cast<size_t>(nq));
          std::vector<double> od(static_cast<size_t>(nq) * lim);
          rc = eps_search_batch(m->ix, qbuf.data(), nq, static_cast<int64_t>(lim), fp, static_cast<int64_t>(nodes.size()), oi.data(), od.data(),
                                oc.data(), nullptr);
          if (rc == EPS_OK) {
            for (int64_t i = 0; i < nq; ++i) {
              batch[i]->count = oc[i];
              std::memcpy(batch[i]->ids, oi.data() + i * lim, sizeof(int64_t) * lim);
              std::memcpy(batch[i]->dists, od.data() + i * lim, sizeof(double) * lim);
            }
          }
        }
        if (rc != EPS_OK) { text = eps_last_error(); unsupported = rc == EPS_ERR_UNSUPPORTED; }
        ++m->launches; ++g_launches;
      }
    }
    q.lock();
    m->calls += static_cast<uint64_t>(nq);
    g_calls += nq;
    for (auto* p : batch) { p->rc = rc; p->unsupported = unsupported; p->err = text; p->done = true; }
    m->qcv.notify_all();
  }
  m->leader_active = false;
  m->qcv.notify_all();  // a queued follower (if any) takes over as leader
}

}  // namespace b200

namespace execution {

// Same signature and member initialisation as the reference constructor; the per-query CPU scratch
// (is_visited_, set_L_, brute_force_queue_) is left empty because the search runs on the device.
VecSearchExecutor::VecSearchExecutor(const int64_t dimension, const int64_t start_search_point,
                                     std::shared_ptr<ANNGraphSegment> ann_index, int64_t* offset_table,
                                     int64_t* neighbor_list,
                                     std::variant<DenseVectorColumnDataContainer, VariableLenAttrColumnContainer*> vector_column,
                                     DistFunc fstdistfunc, void* dist_func_param, int num_threads, int64_t L_master,
                                     int64_t L_local, int64_t subsearch_iterations, bool prefilter_enabled)
    : total_indexed_vector_(ann_index->record_number_),
      dimension_(dimension),
      start_search_point_(start_search_point),
      offset_table_(offset_table),
      neighbor_list_(neighbor_list),
      vector_column_(vector_column),
      fstdistfunc_(fstdistfunc),
      dist_func_param_(dist_func_param),
      num_threads_(num_threads),
      L_master_(L_master),
      L_local_(L_local),
      subsearch_iterations_(subsearch_iterations),
      search_result_(L_master),
      distance_(L_master),
      init_ids_(1, 0),
      local_queues_sizes_(num_threads, 0),
      local_queues_starts_(num_threads),
      brute_force_search_(ann_index->record_number_ < BruteforceThreshold),
      prefilter_enabled_(prefilter_enabled) {
  const int metric = b200::MetricOf(fstdistfunc);
  if (metric < 0 || !std::holds_alternative<DenseVectorColumnDataContainer>(vector_column)) {
    ann_index_ = ann_index;  // sparse / unknown metric: Search() reports NOT_IMPLEMENTED
    return;
  }
  float* table = std::get<DenseVectorColumnDataContainer>(vector_column);
  b200::Key key(table, ann_index.get(), L_master, L_local, prefilter_enabled, metric, num_threads);
  std::shared_ptr<b200::Mirror> m;
  {
    std::lock_guard<std::mutex> lk(b200::g_mu);
    auto it = b200::g_mirrors.find(key);
    if (it != b200::g_mirrors.end()) m = it->second.lock();
    if (!m) {
      b200::Mirror* raw = new b200::Mirror();
      m = std::shared_ptr<b200::Mirror>(raw, b200::MirrorDeleter{raw});
      m->ann = ann_index;
      m->metric = metric;
      m->dim = dimension;
      m->host_vectors = table;
      m->L_master = L_master;
      m->L_local = L_local;
      m->prefilter = prefilter_enabled;
      m->nav = start_search_point;
      m->offsets = offset_table;
      m->nbrs = neighbor_list;
      b200::g_mirrors[key] = m;
    }
  }
  // the executor's own ann_index_ owns the mirror (aliasing constructor) and still points at the graph
  ann_index_ = std::shared_ptr<ANNGraphSegment>(m, ann_index.get());
}

Status VecSearchExecutor::Search(const VectorPtr query_data, vectordb::engine::TableSegmentMVP* table_segment,
                                 const size_t limit, std::vector<vectordb::query::expr::ExprNodePtr>& filter_nodes,
                                 int64_t& result_size) {
  result_size = 0;
  b200::Mirror* m = b200::MirrorOf(ann_index_);
  if (m == nullptr || !std::holds_alternative<DenseVectorPtr>(query_data))
    return Status(NOT_IMPLEMENTED_ERROR, "epsilla_b200: sparse-vector search is out of scope of the GPU path");
  if (search_result_.size() < limit) {  // the reference overruns here when limit > L_master (SURVEY Q2)
    search_result_.resize(limit);
    distance_.resize(limit);
  }
  b200::Mirror::Pending me;
  me.query = std::get<DenseVectorPtr>(query_data);
  me.limit = limit;
  me.filter = &filter_nodes;
  me.key = b200::FilterKey(filter_nodes);
  me.segment = table_segment;
  me.total = table_segment->record_number_;  // snapshot (:839)
  me.n_indexed = total_indexed_vector_;
  me.num_threads = num_threads_;
  me.ids = search_result_.data();
  me.dists = distance_.data();
  b200::SearchCoalesced(m, &me);
  if (me.unsupported) return Status(NOT_IMPLEMENTED_ERROR, "epsilla_b200: " + me.err);
  if (me.rc != EPS_OK) return Status(DB_UNEXPECTED_ERROR, "epsilla_b200: search: " + me.err);
  result_size = me.count;
  return Status::OK();  // (:934)
}

}  // namespace execution

// Graph build on the device, emitting the reference's own CSR members so SaveANNGraph / the loader
// (engine/db/ann_graph_segment.cpp:39-98,156-199) and every executor keep working unchanged.
void ANNGraphSegment::BuildFromVectorTable(VectorColumnData vector_column, int64_t n, int64_t dim,
                                           meta::MetricType metricType) {
  if (!std::holds_alternative<DenseVectorColumnDataContainer>(vector_column))
    throw std::runtime_error("epsilla_b200: sparse-vector graph build is out of scope of the GPU path");
  int metric = EPS_METRIC_L2;
  if (metricType == meta::MetricType::COSINE) metric = EPS_METRIC_COSINE;
  if (metricType == meta::MetricType::DOT_PRODUCT) metric = EPS_METRIC_IP;
  eps_index* ix = nullptr;
  auto die = [&](const char* what) {
    std::string msg = std::string("epsilla_b200 build: ") + what + ": " + eps_last_error();
    if (ix) eps_index_destroy(ix);
    throw std::runtime_error(msg);
  };
  // Rows already mirrored for an executor of this table are reused in place (no second upload of the table): the
  // build index adopts the device rows of a live mirror, which stays pinned until the build is done.
  float* table = std::get<DenseVectorColumnDataContainer>(vector_column);
  std::shared_ptr<b200::Mirror> donor;
  {
    std::lock_guard<std::mutex> lk(b200::g_mu);
    for (auto& kv : b200::g_mirrors) {
      if (std::get<0>(kv.first) != table) continue;
      auto sp = kv.second.lock();
      if (sp && sp->ix && sp->capacity >= n) { donor = sp; break; }
    }
  }
  const float* d_rows = nullptr;
  if (donor) {
    std::lock_guard<std::mutex> lk(donor->mu);
    if (eps_index_sync_rows(donor->ix, std::max<int64_t>(n, eps_index_rows(donor->ix))) == EPS_OK) d_rows = eps_index_device_rows(donor->ix);
  }
  if (d_rows) {
    if (eps_index_create(&ix, metric, dim, nullptr, n, b200::DeviceOrdinal()) != EPS_OK) die("create");
    if (eps_index_adopt_device_rows(ix, d_rows, n) != EPS_OK) die("adopt_device_rows");
  } else {
    if (eps_index_create(&ix, metric, dim, table, n, b200::DeviceOrdinal()) != EPS_OK) die("create");
    if (eps_index_sync_rows(ix, n) != EPS_OK) die("sync_rows");
  }
  if (eps_index_build(ix, n, nullptr) != EPS_OK) die("build");
  int64_t ni = 0, ne = 0, nav = 0;
  if (eps_index_get_graph(ix, &ni, &ne, nullptr, nullptr, &nav) != EPS_OK) die("get_graph");
  int64_t* off = new int64_t[ni + 1];
  int64_t* nb = new int64_t[ne > 0 ? ne : 1];
  if (eps_index_get_graph(ix, nullptr, nullptr, off, nb, nullptr) != EPS_OK) { delete[] off; delete[] nb; die("get_graph"); }
  eps_index_destroy(ix);
  record_number_ = n;
  if (offset_table_ != nullptr) delete[] offset_table_;
  if (neighbor_list_ != nullptr) delete[] neighbor_list_;
  offset_table_ = off;
  neighbor_list_ = nb;
  navigation_point_ = nav;
}

}  // namespace engine
}  // namespace vectordb

// Coalescing counters of this process (Search() calls served, launches made), for the integration tests.
extern "C" __attribute__((visibility("default"))) void eps_dropin_counters(int64_t* calls, int64_t* launches) {
  if (calls) *calls = vectordb::engine::b200::g_calls.load();
  if (launches) *launches = vectordb::engine::b200::g_launches.load();
}
