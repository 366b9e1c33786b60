// group.cu — several GPUs behind ONE process: the database is uploaded once, copied peer to peer
// (NVLink / NVSwitch) to every other device, indexed on each, and queries / all-pairs rows are sharded
// across the devices with no data-path collective (SURVEY.md §8e).  The reference is a single process
// (LIBRARY_API.md:138-156): this is what lets a drop-in of search_batch() use all the GPUs of a box
// (shim/search_batch_vsg.cpp with VSG_DEVICES=0,1,...).  bench.py's multi-GPU runs keep one process per
// GPU with an NCCL broadcast, as its contract asks; both end in the same per-device calls.
#include "vsg_internal.h"
#include "workers.h"

#include <algorithm>
#include <chrono>
#include <cstring>

using namespace vsg;

struct vsg_group {
  std::vector<int> devices;
  std::vector<vsg_ctx *> ctx;
  std::vector<vsg_seqset *> db;
  std::vector<vsg_index *> index;
  int wordlength = 8, mask_lower = 0;
  double upload_ms = 0.0, broadcast_ms = 0.0, index_ms = 0.0;
  int64_t broadcast_bytes = 0;
  vsg_fallback_fn fallback = nullptr;   // the application's routine; query indices are those of the whole call
  void * fallback_user = nullptr;
};

namespace {

double now_ms()
{
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// a copy of `src` (resident on another device) in ctx's HBM: packed symbols, offsets and lengths travel
// device to device; the small host-side metadata is shared as is
int clone_seqset(vsg_ctx * c, const vsg_seqset * src, vsg_seqset ** out)
{
  *out = nullptr;
  VSG_CUDA_OK(cudaSetDevice(c->device));
  vsg_seqset * s = new (std::nothrow) vsg_seqset();
  if (s == nullptr) { Error::set("out of host memory"); return VSG_ENOMEM; }
  s->device = c->device;
  s->h_len = src->h_len;
  s->h_nonacgt = src->h_nonacgt;
  s->h_off = src->h_off;
  s->total = src->total;
  int64_t const n = src->d.n;
  int rc;
  if ((rc = s->b_sym.reserve(static_cast<size_t>(src->total) + 64)) != VSG_OK ||
      (rc = s->b_off.reserve(sizeof(int64_t) * static_cast<size_t>(n) + 8)) != VSG_OK ||
      (rc = s->b_len.reserve(sizeof(int32_t) * static_cast<size_t>(n) + 8)) != VSG_OK) {
    vsg_seqset_destroy(s);
    return rc;
  }
  if (src->total > 0) {
    VSG_CUDA_OK(cudaMemcpyPeerAsync(s->b_sym.p, c->device, src->d.sym, src->device, static_cast<size_t>(src->total), c->stream));
  }
  if (n > 0) {
    VSG_CUDA_OK(cudaMemcpyPeerAsync(s->b_off.p, c->device, src->d.off, src->device, sizeof(int64_t) * static_cast<size_t>(n), c->stream));
    VSG_CUDA_OK(cudaMemcpyPeerAsync(s->b_len.p, c->device, src->d.len, src->device, sizeof(int32_t) * static_cast<size_t>(n), c->stream));
  }
  s->d.sym = static_cast<uint8_t *>(s->b_sym.p);
  s->d.off = static_cast<int64_t *>(s->b_off.p);
  s->d.len = static_cast<int32_t *>(s->b_len.p);
  s->d.n = n;
  *out = s;
  return VSG_OK;
}

}  // namespace

extern "C" int vsg_group_create(const int * devices, int ndev, const vsg_scoring * scoring, const char * cat,
                                const int64_t * off, const int32_t * len, int64_t n, int wordlength, int mask_lower,
                                int dust_db, vsg_group ** out)
{
  if (devices == nullptr || ndev < 1 || scoring == nullptr || out == nullptr) { Error::set("vsg_group_create: bad argument"); return VSG_EINVAL; }
  *out = nullptr;
  vsg_group * g = new (std::nothrow) vsg_group();
  if (g == nullptr) { Error::set("out of host memory"); return VSG_ENOMEM; }
  g->wordlength = wordlength;
  g->mask_lower = (mask_lower != 0 || dust_db != 0) ? 1 : 0;
  int rc = VSG_OK;
  for (int i = 0; i < ndev && rc == VSG_OK; i++) {
    vsg_ctx * c = nullptr;
    rc = vsg_ctx_create(devices[i], scoring, &c);
    if (rc == VSG_OK) { g->devices.push_back(devices[i]); g->ctx.push_back(c); }
  }
  if (rc != VSG_OK) { vsg_group_destroy(g); return rc; }
  g->db.assign(static_cast<size_t>(ndev), nullptr);
  g->index.assign(static_cast<size_t>(ndev), nullptr);
  // 1. one upload (+ optional DUST) on the first device
  double t0 = now_ms();
  rc = vsg_seqset_create(g->ctx[0], cat, off, len, n, 1, &g->db[0]);
  if (rc == VSG_OK && dust_db != 0) { rc = vsg_seqset_dust(g->ctx[0], g->db[0]); }
  if (rc != VSG_OK) { vsg_group_destroy(g); return rc; }
  g->upload_ms = now_ms() - t0;
  // 2. device-to-device copies to the others, all in flight together
  t0 = now_ms();
  for (int i = 1; i < ndev; i++) {
    // direct peer access where the topology offers it (cudaMemcpyPeer stages through the host otherwise)
    int can = 0;
    cudaDeviceCanAccessPeer(&can, devices[i], devices[0]);
    if (can != 0) {
      cudaSetDevice(devices[i]);
      cudaError_t const e = cudaDeviceEnablePeerAccess(devices[0], 0);
      if (e != cudaSuccess) { cudaGetLastError(); }   // already enabled
    }
    rc = clone_seqset(g->ctx[static_cast<size_t>(i)], g->db[0], &g->db[static_cast<size_t>(i)]);
    if (rc != VSG_OK) { vsg_group_destroy(g); return rc; }
    g->broadcast_bytes += g->db[0]->total + static_cast<int64_t>(12) * n;
  }
  for (int i = 1; i < ndev; i++) {
    if ((rc = vsg_ctx_sync(g->ctx[static_cast<size_t>(i)])) != VSG_OK) { vsg_group_destroy(g); return rc; }
  }
  g->broadcast_ms = now_ms() - t0;
  // 3. every device builds its own index (a few ms; cheaper than shipping 2 B per posting)
  t0 = now_ms();
  rc = run_parallel(ndev, [&](int i) {
    return vsg_index_create(g->ctx[static_cast<size_t>(i)], g->db[static_cast<size_t>(i)], wordlength, g->mask_lower,
                            &g->index[static_cast<size_t>(i)]);
  });
  g->index_ms = now_ms() - t0;
  if (rc != VSG_OK) { vsg_group_destroy(g); return rc; }
  *out = g;
  return VSG_OK;
}

extern "C" void vsg_group_destroy(vsg_group * g)
{
  if (g == nullptr) { return; }
  for (auto * ix : g->index) { if (ix != nullptr) { vsg_index_destroy(ix); } }
  for (auto * s : g->db) { if (s != nullptr) { vsg_seqset_destroy(s); } }
  for (auto * c : g->ctx) { if (c != nullptr) { vsg_ctx_destroy(c); } }
  delete g;
}

extern "C" int vsg_group_size(const vsg_group * g) { return g != nullptr ? static_cast<int>(g->ctx.size()) : 0; }
extern "C" vsg_ctx * vsg_group_ctx(vsg_group * g, int i) { return (g != nullptr && i >= 0 && i < static_cast<int>(g->ctx.size())) ? g->ctx[static_cast<size_t>(i)] : nullptr; }
extern "C" vsg_seqset * vsg_group_db(vsg_group * g, int i) { return (g != nullptr && i >= 0 && i < static_cast<int>(g->db.size())) ? g->db[static_cast<size_t>(i)] : nullptr; }
extern "C" vsg_index * vsg_group_index(vsg_group * g, int i) { return (g != nullptr && i >= 0 && i < static_cast<int>(g->index.size())) ? g->index[static_cast<size_t>(i)] : nullptr; }

extern "C" int vsg_group_stats(const vsg_group * g, double * ms3, int64_t * broadcast_bytes)
{
  if (g == nullptr || ms3 == nullptr) { return VSG_EINVAL; }
  ms3[0] = g->upload_ms; ms3[1] = g->broadcast_ms; ms3[2] = g->index_ms;
  if (broadcast_bytes != nullptr) { *broadcast_bytes = g->broadcast_bytes; }
  return VSG_OK;
}

extern "C" int vsg_group_set_fallback(vsg_group * g, vsg_fallback_fn fn, void * user)
{
  if (g == nullptr) { return VSG_EINVAL; }
  g->fallback = fn; g->fallback_user = user;
  for (auto * c : g->ctx) { vsg_ctx_set_fallback(c, fn, user); }   // vsg_group_allpairs: indices are global already
  return VSG_OK;
}

namespace {
// a device sees its slice of the queries: hand the application the index within the whole call
struct SliceFallback { vsg_fallback_fn fn; void * user; int64_t base; };
int slice_fallback(void * u, int64_t query, int32_t strand, int64_t target, int64_t * out)
{
  SliceFallback const * w = static_cast<SliceFallback *>(u);
  return w->fn(w->user, query + w->base, strand, target, out);
}

// The queries of a group call sharded over the devices: fn(d, ctx, slice, b0, b1, opts, work4) searches queries
// [b0, b1) of the call, uploaded (and DUST-masked) on device d as `slice`, with opts rebased to the slice.
template <class Fn>
int group_run(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq, int dust_queries,
              const vsg_search_opts * opts, int64_t * work, Fn && fn)
{
  int const nd = static_cast<int>(g->ctx.size());
  if (work != nullptr) { work[0] = work[1] = work[2] = work[3] = 0; }
  if (nq == 0) { return VSG_OK; }
  // contiguous query ranges of equal nucleotide count (the DP work per query is proportional to its length)
  std::vector<int64_t> bounds(static_cast<size_t>(nd) + 1, nq);
  {
    double total = 0.0;
    for (int64_t i = 0; i < nq; i++) { total += qlen[i]; }
    bounds[0] = 0;
    double acc = 0.0;
    int p = 1;
    for (int64_t i = 0; i < nq && p < nd; i++) {
      acc += qlen[i];
      while (p < nd && acc >= total * p / nd) { bounds[static_cast<size_t>(p++)] = i + 1; }
    }
  }
  std::vector<int64_t> w(static_cast<size_t>(nd) * 4, 0);
  int const rc = run_parallel(nd, [&](int d) -> int {
    int64_t const b0 = bounds[static_cast<size_t>(d)], b1 = bounds[static_cast<size_t>(d) + 1];
    if (b1 <= b0) { return VSG_OK; }
    vsg_ctx * c = g->ctx[static_cast<size_t>(d)];
    // this device's slice, rebased: offsets relative to its first sequence
    int64_t const base = qoff[b0];
    std::vector<int64_t> off(static_cast<size_t>(b1 - b0));
    for (int64_t i = b0; i < b1; i++) { off[static_cast<size_t>(i - b0)] = qoff[i] - base; }
    vsg_seqset * q = nullptr;
    int rc = vsg_seqset_create(c, qcat + base, off.data(), qlen + b0, b1 - b0, 1, &q);
    if (rc == VSG_OK && dust_queries != 0) { rc = vsg_seqset_dust(c, q); }
    SliceFallback sf{g->fallback, g->fallback_user, b0};
    if (g->fallback != nullptr) { vsg_ctx_set_fallback(c, slice_fallback, &sf); }
    vsg_search_opts o = *opts;
    if (o.query_sizes != nullptr) { o.query_sizes += b0; }
    if (o.query_labels != nullptr) { o.query_labels += b0; }
    if (rc == VSG_OK) { rc = fn(d, c, q, b0, b1, o, w.data() + 4 * d); }
    if (g->fallback != nullptr) { vsg_ctx_set_fallback(c, g->fallback, g->fallback_user); }
    if (q != nullptr) { vsg_seqset_destroy(q); }
    return rc;
  });
  if (rc != VSG_OK) { return rc; }
  for (int d = 0; d < nd && work != nullptr; d++) {
    for (int z = 0; z < 4; z++) { work[z] += w[static_cast<size_t>(4 * d + z)]; }
  }
  return VSG_OK;
}

}  // namespace

extern "C" int vsg_group_search(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq,
                                int dust_queries, const vsg_search_opts * opts, vsg_search_result * results, int max_results,
                                int32_t * counts, int64_t * work)
{
  if (g == nullptr || opts == nullptr || results == nullptr || counts == nullptr || nq < 0 ||
      (nq > 0 && (qcat == nullptr || qoff == nullptr || qlen == nullptr))) { Error::set("vsg_group_search: bad argument"); return VSG_EINVAL; }
  return group_run(g, qcat, qoff, qlen, nq, dust_queries, opts, work,
                   [&](int d, vsg_ctx * c, const vsg_seqset * q, int64_t b0, int64_t b1, const vsg_search_opts & o, int64_t * w) {
    return vsg_search_batch(c, g->index[static_cast<size_t>(d)], g->db[static_cast<size_t>(d)], q, 0, b1 - b0, &o,
                            results + static_cast<size_t>(b0) * max_results, max_results, counts + b0, w);
  });
}

namespace vsg {

int group_search_rows(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq, int dust_queries,
                      const vsg_search_opts * opts, int64_t maxhits, std::vector<vsg_search_result> & rows,
                      std::vector<int64_t> & first, int64_t * work)
{
  if (g == nullptr || opts == nullptr || nq < 0 || maxhits < 0 || (nq > 0 && (qcat == nullptr || qoff == nullptr || qlen == nullptr))) {
    Error::set("vsg_group_search_hits: bad argument");
    return VSG_EINVAL;
  }
  int const nd = static_cast<int>(g->ctx.size());
  std::vector<std::vector<vsg_search_result>> drows(static_cast<size_t>(nd));
  std::vector<std::vector<int64_t>> dfirst(static_cast<size_t>(nd));
  int const rc = group_run(g, qcat, qoff, qlen, nq, dust_queries, opts, work,
                           [&](int d, vsg_ctx * c, const vsg_seqset * q, int64_t b0, int64_t b1, const vsg_search_opts & o, int64_t * w) {
    return search_hits_host(c, g->index[static_cast<size_t>(d)], g->db[static_cast<size_t>(d)], q, 0, b1 - b0, &o, maxhits,
                            drows[static_cast<size_t>(d)], dfirst[static_cast<size_t>(d)], w);
  });
  if (rc != VSG_OK) { return rc; }
  // the devices' slices are consecutive query ranges: concatenate them in device order
  rows.clear();
  first.assign(1, 0);
  for (int d = 0; d < nd; d++) {
    auto const & fd = dfirst[static_cast<size_t>(d)];
    for (size_t i = 1; i < fd.size(); i++) { first.push_back(static_cast<int64_t>(rows.size()) + fd[i]); }
    rows.insert(rows.end(), drows[static_cast<size_t>(d)].begin(), drows[static_cast<size_t>(d)].end());
    std::vector<vsg_search_result>().swap(drows[static_cast<size_t>(d)]);
  }
  first.resize(static_cast<size_t>(nq) + 1, static_cast<int64_t>(rows.size()));
  return VSG_OK;
}

int group_sintax(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq,
                 const vsg_sintax_opts * opts, vsg_sintax_result * out)
{
  vsg_search_opts const none{};   // group_run's search options: no per-query arrays to rebase
  return group_run(g, qcat, qoff, qlen, nq, 0, &none, nullptr,
                   [&](int d, vsg_ctx * c, const vsg_seqset * q, int64_t b0, int64_t b1, const vsg_search_opts &, int64_t *) {
    vsg_sintax_opts o = *opts;
    o.query_number0 += b0;   // this device's first query keeps its input number
    return vsg_sintax(c, g->index[static_cast<size_t>(d)], q, 0, b1 - b0, &o, out + b0);
  });
}

int group_orient(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq, int query_mask_lower,
                 vsg_orient_result * out)
{
  vsg_search_opts const none{};   // group_run's search options: no per-query arrays to rebase
  return group_run(g, qcat, qoff, qlen, nq, 0, &none, nullptr,
                   [&](int d, vsg_ctx * c, const vsg_seqset * q, int64_t b0, int64_t b1, const vsg_search_opts &, int64_t *) {
    return vsg_orient(c, g->index[static_cast<size_t>(d)], q, 0, b1 - b0, query_mask_lower, out + b0);
  });
}

}  // namespace vsg

extern "C" int vsg_group_search_hits(vsg_group * g, const char * qcat, const int64_t * qoff, const int32_t * qlen, int64_t nq,
                                     int dust_queries, const vsg_search_opts * opts, int64_t maxhits, vsg_search_result * hits,
                                     int64_t cap, int64_t * first, int64_t * nhits, int64_t * work)
{
  if (first == nullptr || nhits == nullptr || cap < 0 || (cap > 0 && hits == nullptr)) { Error::set("vsg_group_search_hits: bad argument"); return VSG_EINVAL; }
  *nhits = 0;
  std::vector<vsg_search_result> rows;
  std::vector<int64_t> f;
  int const rc = group_search_rows(g, qcat, qoff, qlen, nq, dust_queries, opts, maxhits, rows, f, work);
  if (rc != VSG_OK) { return rc; }
  return hits_out(rows, f, "vsg_group_search_hits", hits, cap, first, nhits);
}

extern "C" int vsg_group_allpairs(vsg_group * g, const vsg_search_opts * opts, vsg_pair_hit * hits, int64_t cap,
                                  int64_t * nhits, int64_t * work)
{
  if (g == nullptr || opts == nullptr || nhits == nullptr || (cap > 0 && hits == nullptr)) { Error::set("vsg_group_allpairs: bad argument"); return VSG_EINVAL; }
  int const nd = static_cast<int>(g->ctx.size());
  const vsg_seqset * set = g->db[0];
  int64_t const n = set->d.n;
  *nhits = 0;
  if (work != nullptr) { work[0] = work[1] = 0; }
  // row ranges of equal DP work (triangle balancing), one per device
  std::vector<int64_t> bounds(static_cast<size_t>(nd) + 1, 0);
  int rc = vsg_allpairs_partition(set->h_len.data(), n, nd, bounds.data());
  if (rc != VSG_OK) { return rc; }
  // every device writes into its own stretch of the caller's buffer, sized by its share of the pairs
  std::vector<int64_t> cap_off(static_cast<size_t>(nd) + 1, 0);
  {
    double total_pairs = 0.0;
    std::vector<double> pr(static_cast<size_t>(nd));
    for (int d = 0; d < nd; d++) {
      double p = 0.0;
      for (int64_t i = bounds[static_cast<size_t>(d)]; i < bounds[static_cast<size_t>(d) + 1]; i++) { p += static_cast<double>(n - i - 1); }
      pr[static_cast<size_t>(d)] = p; total_pairs += p;
    }
    for (int d = 0; d < nd; d++) {
      int64_t const share = total_pairs > 0 ? static_cast<int64_t>(static_cast<double>(cap) * pr[static_cast<size_t>(d)] / total_pairs) : 0;
      cap_off[static_cast<size_t>(d) + 1] = std::min<int64_t>(cap, cap_off[static_cast<size_t>(d)] + share);
    }
    cap_off[static_cast<size_t>(nd)] = cap;
  }
  std::vector<int64_t> got(static_cast<size_t>(nd), 0), w(static_cast<size_t>(nd) * 2, 0);
  rc = run_parallel(nd, [&](int d) -> int {
    int64_t const r0 = bounds[static_cast<size_t>(d)], r1 = bounds[static_cast<size_t>(d) + 1];
    if (r1 <= r0) { return VSG_OK; }
    return vsg_allpairs(g->ctx[static_cast<size_t>(d)], g->db[static_cast<size_t>(d)], r0, r1 - r0, opts,
                        hits + cap_off[static_cast<size_t>(d)], cap_off[static_cast<size_t>(d) + 1] - cap_off[static_cast<size_t>(d)],
                        &got[static_cast<size_t>(d)], w.data() + 2 * d);
  });
  if (rc != VSG_OK) { return rc; }
  int64_t pos = 0;
  for (int d = 0; d < nd; d++) {
    // compact the per-device stretches into one list in row order
    if (cap_off[static_cast<size_t>(d)] != pos && got[static_cast<size_t>(d)] > 0) {
      std::memmove(hits + pos, hits + cap_off[static_cast<size_t>(d)], sizeof(vsg_pair_hit) * static_cast<size_t>(got[static_cast<size_t>(d)]));
    }
    pos += got[static_cast<size_t>(d)];
    if (work != nullptr) { work[0] += w[static_cast<size_t>(2 * d)]; work[1] += w[static_cast<size_t>(2 * d + 1)]; }
  }
  *nhits = pos;
  return VSG_OK;
}
