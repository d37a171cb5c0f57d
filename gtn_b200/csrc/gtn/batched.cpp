/*
 * gtn/batched.cpp -- the list forms of the hot-path ops as ONE packed launch each.
 *
 * The reference's Python bindings give every function a list overload that maps the single-graph
 * function over the batch with parallelMap (bindings/python/gtn/_functions.cpp:69-135,
 * gtn/parallel/parallel_map.h:153-188); its CTC benchmark and its PyTorch example drive a whole
 * minibatch through exactly these calls (benchmarks/ctc.cpp:150-165).  On a GPU "B threads, one graph
 * each" means B contexts, B batch-of-one lattices and ~10 launches plus a synchronising read-back per
 * utterance.  Here a list call whose graphs qualify becomes one C-ABI call on a B-entry lattice:
 *
 *   compose / intersect (list, list)   every pair = (host graph without epsilon on the matched side,
 *                                      gtn::linearGraph): the emissions are gathered into one device
 *                                      buffer [B][T_max * C] (or found there already), ONE
 *                                      gtnb_compose_linear builds the B lattices
 *   forwardScore / viterbiScore (list) the B entries of such a lattice, each once: ONE gtnb_forward;
 *                                      or B linear graphs (the CTC normaliser): ONE gtnb_linear_forward
 *   viterbiPath (list)                 the B entries of such a lattice, each once: ONE gtnb_viterbi_path
 *   backward (list)                    the entries' gradFuncs only RECORD their seeds (detail::BatchState);
 *                                      the first read of a resulting gradient runs gtnb_backward +
 *                                      gtnb_compose_grad (or the normaliser's gradient pass) once for the
 *                                      whole batch, and every entry's gradient is a lazy slice of it
 *
 * Anything else (mixed shapes, epsilons, device-resident operands, size-1 broadcasts) falls back to
 * parallelMap of the single-graph op, i.e. the reference's own semantics.  Results are identical either
 * way: the batched lattices are the same kernels run on B entries instead of one.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <stdexcept>

#include "gtn/autograd.h"
#include "gtn/device.h"
#include "gtn/functions.h"
#include "gtn/parallel.h"

namespace gtn {

namespace detail {
bool matchedSideHasEpsilon(const Graph& g, bool useIlabel);
}

namespace {

using detail::BatchState;
using detail::check;
using detail::Context;
using detail::DeviceBuffer;
using detail::LatticeHandle;

using Binary = Graph (*)(const Graph&, const Graph&);
Binary single2(Binary f) {
  return f;
}

cudaStream_t streamOf(const std::shared_ptr<Context>& c) {
  return (cudaStream_t)gtnb_ctx_stream(c->ctx);
}

/*
 * The emissions of B linear graphs in one device buffer, entry i at float offset i * stride.  Reuses a
 * buffer an earlier list op gathered (every graph holds the slice i * stride of the same buffer);
 * otherwise copies every graph's weights in -- device to device where setWeights got a device pointer,
 * host to device else -- and remembers the slices.
 */
std::shared_ptr<DeviceBuffer> gatherEmissions(
    const std::vector<const Graph*>& lin, size_t stride, const std::shared_ptr<Context>& c) {
  const size_t B = lin.size();
  {
    size_t off = 0;
    auto first = lin[0]->batchSlice(&off);
    bool same = first && off == 0 && first->owner == c && first->count >= B * stride;
    for (size_t i = 1; same && i < B; i++) {
      auto bi = lin[i]->batchSlice(&off);
      same = bi == first && off == i * stride;
    }
    if (same) return first;
  }
  auto buf = std::make_shared<DeviceBuffer>(c, B * stride);
  // device copies owned by other threads' streams must be complete before this stream reads them
  std::vector<std::shared_ptr<Context>> drained;
  for (size_t i = 0; i < B; i++) {
    auto dev = lin[i]->deviceWeights();
    if (dev && dev->owner != c && std::find(drained.begin(), drained.end(), dev->owner) == drained.end()) {
      std::lock_guard<std::mutex> lo(dev->owner->lock);
      check(dev->owner, gtnb_ctx_synchronize(dev->owner->ctx));
      drained.push_back(dev->owner);
    }
  }
  std::lock_guard<std::mutex> l(c->lock);
  for (size_t i = 0; i < B; i++) {
    const size_t n = (size_t)lin[i]->linearFrames() * (size_t)lin[i]->linearLabels();
    if (n == 0) continue;
    auto dev = lin[i]->deviceWeights();
    cudaError_t e;
    if (dev && dev->count == n)
      e = cudaMemcpyAsync(buf->ptr + i * stride, dev->ptr, sizeof(float) * n, cudaMemcpyDeviceToDevice, streamOf(c));
    else
      e = cudaMemcpyAsync(buf->ptr + i * stride, lin[i]->weights(), sizeof(float) * n, cudaMemcpyHostToDevice, streamOf(c));
    if (e != cudaSuccess) throw std::runtime_error("[gtn] gathering the emissions of a batch failed");
  }
  // pageable sources: the copies above have consumed them when the calls return; nothing to wait for
  for (size_t i = 0; i < B; i++) lin[i]->cacheBatchSlice(buf, i * stride);
  return buf;
}

/* the gradients of a whole batch come back in ONE copy through a pinned block of the context (caller holds
 * c->lock); a per-entry read-back would pay a synchronous copy per utterance */
void readBack(const std::shared_ptr<Context>& c, int slot, const void* owner, const float* dev, size_t n) {
  if (c->pinnedCount[slot] < n) {
    if (c->pinned[slot]) gtnb_host_free(c->ctx, c->pinned[slot]);
    c->pinned[slot] = nullptr;
    c->pinnedCount[slot] = 0;
    c->pinnedOwner[slot] = nullptr;
    void* p = nullptr;
    if (gtnb_host_alloc(c->ctx, sizeof(float) * n, &p) == GTNB_OK) {
      c->pinned[slot] = static_cast<float*>(p);
      c->pinnedCount[slot] = n;
    }
  }
  if (c->pinned[slot] && n) {
    check(c, gtnb_memcpy_d2h(c->ctx, c->pinned[slot], dev, sizeof(float) * n));
    check(c, gtnb_ctx_synchronize(c->ctx));
    c->pinnedOwner[slot] = owner;
  }
}

/* the B entries' arc gradients, as the lattice holds them now, into bs.arcGrads; na: the entries' arc counts
 * (h->sizes(), read before the caller took bs.m and c->lock) */
void copyArcGrads(const std::shared_ptr<LatticeHandle>& h, const std::vector<int32_t>& na, BatchState& bs) {
  auto& c = h->owner;
  bs.arcGrads.resize((size_t)h->B);
  for (int b = 0; b < h->B; b++) {
    bs.arcGrads[b].resize((size_t)na[b]);
    if (na[b]) check(c, gtnb_lattice_arc_grads(c->ctx, h->lat, b, bs.arcGrads[b].data()));
  }
}

/* run the pending backward of a batched lattice once: shortestDistanceGrad for the recorded seeds
 * (shortest.cpp:33-82), host-provided arc gradients added on top, then compose's gradFunc (compose.cpp:496-518)
 * for all entries into bs.dLinear / bs.dGraph */
void flushLattice(const std::shared_ptr<LatticeHandle>& h) {
  BatchState& bs = *h->batch;
  std::lock_guard<std::mutex> lk(bs.m);
  if (bs.flushed) return;
  auto& c = h->owner;
  const size_t B = (size_t)h->B;
  size_t graphTotal = 0;
  for (size_t b = 0; b < B; b++) graphTotal = std::max(graphTotal, bs.graphOff[b + 1]);
  bs.dLinear = std::make_shared<DeviceBuffer>(c, std::max<size_t>(B * bs.stride, 1));
  bs.dGraph = std::make_shared<DeviceBuffer>(c, std::max<size_t>(graphTotal, 1));
  bool hostDeltas = false;
  for (size_t b = 0; b < B; b++) hostDeltas = hostDeltas || !bs.hostDeltas[b].empty();
  const auto& na = h->sizes().second;
  std::lock_guard<std::mutex> l(c->lock);
  if (bs.mode >= 0) {
    if (h->scoreMode != bs.mode) { // the lattice was re-scored in the other semiring since: restore
      check(c, gtnb_forward(c->ctx, h->lat, bs.mode, nullptr, nullptr));
      h->scoreMode = bs.mode;
    }
    check(c, gtnb_backward(c->ctx, h->lat, bs.mode, bs.sdDelta.data()));
    // the entries' own gradients are the seeds' alone: keep them before the host deltas are added in
    if (hostDeltas) copyArcGrads(h, na, bs);
  }
  for (size_t b = 0; b < B; b++) {
    if (bs.hostDeltas[b].empty()) continue;
    std::vector<float>& d = bs.hostDeltas[b];
    if (bs.mode >= 0)
      for (size_t i = 0; i < d.size() && i < bs.arcGrads[b].size(); i++) d[i] += bs.arcGrads[b][i];
    check(c, gtnb_lattice_set_arc_grads(c->ctx, h->lat, (int)b, d.data()));
  }
  check(c, gtnb_memset(c->ctx, bs.dLinear->ptr, 0, sizeof(float) * std::max<size_t>(B * bs.stride, 1)));
  check(c, gtnb_memset(c->ctx, bs.dGraph->ptr, 0, sizeof(float) * std::max<size_t>(graphTotal, 1)));
  check(c, gtnb_compose_grad(c->ctx, h->lat, bs.dGraph->ptr, bs.dLinear->ptr, (int64_t)bs.stride));
  readBack(c, 0, &bs, bs.dLinear->ptr, B * bs.stride);
  bs.flushed = true;
}

/* one slice of a batch's gradient: a host copy while the context's pinned block still holds that batch's
 * read-back, a device read otherwise */
void fetchBatchSlice(const std::shared_ptr<Context>& c, int slot, const void* owner, const float* dev, size_t off,
                     size_t n, std::vector<float>& out);
bool addBatchSlice(const std::shared_ptr<Context>& c, int slot, const void* owner, size_t off, size_t n, float* dst, size_t dn);

void fetchSlice(const std::shared_ptr<Context>& c, const float* dev, size_t n, std::vector<float>& out) {
  out.resize(n);
  if (n == 0) return;
  std::lock_guard<std::mutex> l(c->lock);
  check(c, gtnb_memcpy_d2h(c->ctx, out.data(), dev, sizeof(float) * n));
  check(c, gtnb_ctx_synchronize(c->ctx));
}

/* all pairs qualify for one frame-synchronous device composition?  which side is linear */
bool batchComposable(const std::vector<Graph>& a, const std::vector<Graph>& b, bool* linearFirst) {
  if (a.size() != b.size() || a.size() < 2) return false;
  const bool lf = a[0].isLinear() && !b[0].isLinear();
  const bool ls = b[0].isLinear();
  if (!lf && !ls) return false;
  const bool linFirst = lf && !ls;
  const int C = (linFirst ? a[0] : b[0]).linearLabels();
  if (C <= 0) return false;
  for (size_t i = 0; i < a.size(); i++) {
    const Graph& lin = linFirst ? a[i] : b[i];
    const Graph& g = linFirst ? b[i] : a[i];
    if (!lin.isLinear() || lin.linearLabels() != C || lin.isDeviceResident()) return false;
    if (g.isDeviceResident()) return false;
    if (detail::matchedSideHasEpsilon(g, linFirst)) return false;
  }
  *linearFirst = linFirst;
  return true;
}

std::vector<Graph> composeBatch(const std::vector<Graph>& a, const std::vector<Graph>& b, bool intersectMode) {
  bool linearFirst = false;
  if (!batchComposable(a, b, &linearFirst)) {
    // B arbitrary pairs (no emissions chain among them): one launch of k_gcompose.cu, one CTA per pair
    const size_t n = std::max(a.size(), b.size());
    const int policy = detail::composeDevicePolicy();
    bool general = n >= 2 && policy != 2 && detail::deviceCount() > 0 && (a.size() == n || a.size() == 1) &&
                   (b.size() == n || b.size() == 1);
    double states = 0.0;
    for (size_t i = 0; general && i < n; i++) {
      const Graph& x = a[a.size() == 1 ? 0 : i];
      const Graph& y = b[b.size() == 1 ? 0 : i];
      general = !x.isDeviceResident() && !y.isDeviceResident();
      states += (double)x.numNodes() * (double)y.numNodes();
    }
    // (the rule of the single-pair dispatch, functions.cpp generalOnDevice, with the per-pair threshold of a list)
    if (general && (policy == 1 || states >= detail::kComposeDeviceListStates * (double)n)) {
      std::vector<const Graph*> pa(a.size()), pb(b.size());
      for (size_t i = 0; i < a.size(); i++) pa[i] = &a[i];
      for (size_t i = 0; i < b.size(); i++) pb[i] = &b[i];
      std::vector<Graph> out;
      if (detail::composeGraphsDevice(pa, pb, intersectMode, out)) return out;
    }
    return parallelMap(intersectMode ? single2(intersect) : single2(compose), a, b);
  }
  const size_t B = a.size();
  auto c = detail::threadContext();
  std::vector<const Graph*> lin(B), gr(B);
  std::vector<int32_t> T(B);
  const int C = (linearFirst ? a[0] : b[0]).linearLabels();
  int maxT = 0;
  for (size_t i = 0; i < B; i++) {
    lin[i] = linearFirst ? &a[i] : &b[i];
    gr[i] = linearFirst ? &b[i] : &a[i];
    T[i] = lin[i]->linearFrames();
    maxT = std::max(maxT, T[i]);
  }
  const size_t stride = (size_t)std::max(maxT, 1) * C;
  auto emis = gatherEmissions(lin, stride, c);
  std::vector<detail::ViewStorage> vs(B);
  std::vector<gtnb_graph_view> views(B);
  {
    // the host views of the B graphs, on the reference's own worker threads
    std::vector<int> idx(B);
    for (size_t i = 0; i < B; i++) idx[i] = (int)i;
    parallelMap(
        [&](int i) {
          detail::makeView(*gr[i], vs[i]);
          return 0;
        },
        idx);
    for (size_t i = 0; i < B; i++) views[i] = vs[i].view;
  }
  gtnb_lattice* lat = nullptr;
  int rc;
  {
    std::lock_guard<std::mutex> l(c->lock);
    rc = gtnb_compose_linear(c->ctx, (int)B, views.data(), (int)B, linearFirst ? 1 : 0, T.data(), C, emis->ptr,
                             (int64_t)stride, &lat);
  }
  if (rc == GTNB_ERR_UNSUPPORTED) return parallelMap(intersectMode ? single2(intersect) : single2(compose), a, b);
  check(c, rc);
  auto handle = std::make_shared<LatticeHandle>();
  handle->owner = c;
  handle->lat = lat;
  handle->B = (int)B;
  handle->composed = true;
  handle->emissions = emis;
  handle->frames.assign(T.begin(), T.end());
  handle->labels = C;
  handle->linearFirst = linearFirst;
  auto bs = std::make_shared<BatchState>();
  bs->sdDelta.assign(B, 0.0f);
  bs->hostDeltas.resize(B);
  bs->stride = stride;
  bs->graphOff.assign(B + 1, 0);
  for (size_t i = 0; i < B; i++) bs->graphOff[i + 1] = bs->graphOff[i] + gr[i]->numArcs();
  handle->batch = bs;

  std::vector<Graph> out;
  out.reserve(B);
  for (size_t i = 0; i < B; i++) {
    const size_t graphArcs = gr[i]->numArcs(), emisArcs = (size_t)T[i] * C;
    const int bi = (int)i;
    // compose's gradFunc (compose.cpp:496-518), deferred: the scatter runs once for the batch
    auto gradFunc = [handle, bi, linearFirst, graphArcs, emisArcs](std::vector<Graph>& inputs, Graph& deltas) {
      BatchState& bs = *handle->batch;
      {
        std::lock_guard<std::mutex> lk(bs.m);
        if (bs.flushed)
          throw std::logic_error("[gtn::compose] the batched backward of this lattice has already run "
                                 "(backward the whole list before reading gradients, or retain and recompose)");
        // arc gradients still parked on the device come from the batched shortest-distance backward and are
        // there when it runs; keep a copy of those produced on the host
        deltas.hostContributions(bs.hostDeltas[bi]);
      }
      auto c = handle->owner;
      Graph& gGraph = inputs[linearFirst ? 1 : 0];
      Graph& gLinear = inputs[linearFirst ? 0 : 1];
      // compose.cpp:516-517 adds to both inputs unconditionally (addGrad ignores calcGrad == false)
      gGraph.addLazyGrad(graphArcs, [handle, bi, graphArcs, c](std::vector<float>& v) {
        flushLattice(handle);
        fetchSlice(c, handle->batch->dGraph->ptr + handle->batch->graphOff[bi], graphArcs, v);
      });
      gLinear.addLazyGrad(
          emisArcs,
          [handle, bi, emisArcs, c](std::vector<float>& v) {
            flushLattice(handle);
            BatchState& bs = *handle->batch;
            fetchBatchSlice(c, 0, &bs, bs.dLinear->ptr, (size_t)bi * bs.stride, emisArcs, v);
          },
          [handle, bi, emisArcs, c](float* dst, size_t dn) {
            flushLattice(handle);
            BatchState& bs = *handle->batch;
            return addBatchSlice(c, 0, &bs, (size_t)bi * bs.stride, emisArcs, dst, dn);
          });
    };
    out.push_back(Graph::fromLattice(handle, bi, gradFunc, {a[i], b[i]}));
  }
  return out;
}

void fetchBatchSlice(const std::shared_ptr<Context>& c, int slot, const void* owner, const float* dev, size_t off,
                     size_t n, std::vector<float>& out) {
  {
    std::lock_guard<std::mutex> l(c->lock);
    if (c->pinnedOwner[slot] == owner && c->pinned[slot]) {
      out.assign(c->pinned[slot] + off, c->pinned[slot] + off + n);
      return;
    }
  }
  fetchSlice(c, dev + off, n, out);
}

/* adds a batch's slice into dst when the context's pinned block still holds that batch's read-back */
bool addBatchSlice(const std::shared_ptr<Context>& c, int slot, const void* owner, size_t off, size_t n, float* dst, size_t dn) {
  std::lock_guard<std::mutex> l(c->lock);
  if (c->pinnedOwner[slot] != owner || !c->pinned[slot]) return false;
  const float* src = c->pinned[slot] + off;
  for (size_t i = 0; i < n && i < dn; i++) dst[i] += src[i];
  return true;
}

Graph scalarResult(Graph::GradFunc gradFunc, const Graph& input, float score) {
  Graph result(std::move(gradFunc), {input});
  result.addNode(true);
  result.addNode(false, true);
  result.addArc(0, 1, 0, 0, score);
  return result;
}

/* state of a batched forwardScore over B emission chains (the CTC normaliser, benchmarks/ctc.cpp:157) */
struct LinearBatch {
  std::mutex m;
  std::shared_ptr<Context> c;
  std::shared_ptr<DeviceBuffer> emis, grad;
  std::vector<int32_t> T;
  int C{0};
  size_t stride{0};
  bool tropical{false};
  std::vector<float> delta;
  bool flushed{false};
};

void flushLinear(const std::shared_ptr<LinearBatch>& lb) {
  std::lock_guard<std::mutex> lk(lb->m);
  if (lb->flushed) return;
  auto& c = lb->c;
  const size_t B = lb->T.size();
  lb->grad = std::make_shared<DeviceBuffer>(c, std::max<size_t>(B * lb->stride, 1));
  DeviceBuffer sdev(c, B + 4), ddev(c, B + 4);
  std::lock_guard<std::mutex> l(c->lock);
  check(c, gtnb_memset(c->ctx, lb->grad->ptr, 0, sizeof(float) * std::max<size_t>(B * lb->stride, 1)));
  check(c, gtnb_memcpy_h2d(c->ctx, ddev.ptr, lb->delta.data(), sizeof(float) * B));
  check(c, gtnb_linear_forward(c->ctx, (int)B, lb->T.data(), lb->C, lb->emis->ptr, (int64_t)lb->stride,
                               lb->tropical ? 1 : 0, sdev.ptr, lb->grad->ptr, (int64_t)lb->stride, ddev.ptr, 1.0f));
  check(c, gtnb_ctx_synchronize(c->ctx)); // ddev / sdev go out of scope
  readBack(c, 1, lb.get(), lb->grad->ptr, B * lb->stride);
  lb->flushed = true;
}

/* the batched lattice whose B entries gs are, each exactly once (in any order); null otherwise */
std::shared_ptr<LatticeHandle> entriesOfOneBatch(const std::vector<Graph>& gs) {
  const size_t B = gs.size();
  auto h = B >= 2 ? gs[0].scoringLattice() : nullptr;
  if (!h || !h->batch || (size_t)h->B != B) return nullptr;
  std::vector<char> seen(B, 0);
  for (size_t i = 0; i < B; i++) {
    const int bi = gs[i].latticeIndex();
    if (gs[i].scoringLattice() != h || bi < 0 || bi >= (int)B || seen[bi]) return nullptr;
    seen[bi] = 1;
  }
  return h;
}

std::vector<Graph> scoreBatch(const std::vector<Graph>& gs, bool tropical) {
  const size_t B = gs.size();
  Graph (*single)(const Graph&) = tropical ? static_cast<Graph (*)(const Graph&)>(viterbiScore)
                                           : static_cast<Graph (*)(const Graph&)>(forwardScore);
  if (B < 2) return parallelMap(single, gs);
  // (1) the B entries of one batched lattice, each exactly once
  {
    auto h = entriesOfOneBatch(gs);
    if (h) {
      auto& c = h->owner;
      std::vector<float> scores(B);
      {
        std::lock_guard<std::mutex> l(c->lock);
        check(c, gtnb_forward(c->ctx, h->lat, tropical ? 1 : 0, scores.data(), nullptr));
        h->scoreMode = tropical ? 1 : 0;
      }
      const auto& na = h->sizes().second;
      std::vector<Graph> out;
      out.reserve(B);
      for (size_t i = 0; i < B; i++) {
        const int bi = gs[i].latticeIndex();
        const size_t numArcs = (size_t)na[bi];
        auto gradFunc = [h, bi, tropical, numArcs](std::vector<Graph>& inputs, Graph& deltas) {
          BatchState& bs = *h->batch;
          {
            std::lock_guard<std::mutex> lk(bs.m);
            if (bs.flushed)
              throw std::logic_error("[gtn::forwardScore] the batched backward of this lattice has already run");
            if (bs.mode >= 0 && bs.mode != (tropical ? 1 : 0))
              throw std::logic_error("[gtn] forwardScore and viterbiScore of one batched lattice cannot both be "
                                     "differentiated in one backward pass; use the single-graph functions");
            bs.mode = tropical ? 1 : 0;
            bs.sdDelta[bi] += deltas.item();
          }
          // the lattice entry's own gradient: its arc gradients, still on the device
          inputs[0].addLazyGrad(numArcs, [h, bi, numArcs](std::vector<float>& v) {
            flushLattice(h);
            {
              BatchState& bs = *h->batch;
              std::lock_guard<std::mutex> lk(bs.m);
              if (!bs.arcGrads.empty()) {
                v = bs.arcGrads[bi];
                return;
              }
            }
            auto& c = h->owner;
            v.resize(numArcs);
            if (numArcs == 0) return;
            std::lock_guard<std::mutex> l(c->lock);
            check(c, gtnb_lattice_arc_grads(c->ctx, h->lat, bi, v.data()));
          });
        };
        out.push_back(scalarResult(gradFunc, gs[i], scores[bi]));
      }
      return out;
    }
  }
  // (2) B emission chains: the per-frame reductions of all of them in one launch
  {
    bool ok = gs[0].isLinear() && gs[0].linearLabels() > 0;
    const int C = gs[0].linearLabels();
    for (size_t i = 0; ok && i < B; i++) ok = gs[i].isLinear() && gs[i].linearLabels() == C && !gs[i].isDeviceResident();
    if (ok) {
      auto lb = std::make_shared<LinearBatch>();
      lb->c = detail::threadContext();
      lb->C = C;
      lb->tropical = tropical;
      lb->T.resize(B);
      int maxT = 0;
      std::vector<const Graph*> lin(B);
      for (size_t i = 0; i < B; i++) {
        lin[i] = &gs[i];
        lb->T[i] = gs[i].linearFrames();
        maxT = std::max(maxT, lb->T[i]);
      }
      lb->stride = (size_t)std::max(maxT, 1) * C;
      lb->emis = gatherEmissions(lin, lb->stride, lb->c);
      lb->delta.assign(B, 0.0f);
      std::vector<float> scores(B);
      {
        DeviceBuffer sdev(lb->c, B + 4);
        std::lock_guard<std::mutex> l(lb->c->lock);
        check(lb->c, gtnb_linear_forward(lb->c->ctx, (int)B, lb->T.data(), C, lb->emis->ptr, (int64_t)lb->stride,
                                         tropical ? 1 : 0, sdev.ptr, nullptr, 0, nullptr, 1.0f));
        check(lb->c, gtnb_memcpy_d2h(lb->c->ctx, scores.data(), sdev.ptr, sizeof(float) * B));
        check(lb->c, gtnb_ctx_synchronize(lb->c->ctx));
      }
      std::vector<Graph> out;
      out.reserve(B);
      for (size_t i = 0; i < B; i++) {
        const size_t n = (size_t)lb->T[i] * C;
        const int bi = (int)i;
        auto gradFunc = [lb, bi, n](std::vector<Graph>& inputs, Graph& deltas) {
          {
            std::lock_guard<std::mutex> lk(lb->m);
            if (lb->flushed) throw std::logic_error("[gtn::forwardScore] the batched backward of this list has already run");
            lb->delta[bi] += deltas.item();
          }
          inputs[0].addLazyGrad(
              n,
              [lb, bi, n](std::vector<float>& v) {
                flushLinear(lb);
                fetchBatchSlice(lb->c, 1, lb.get(), lb->grad->ptr, (size_t)bi * lb->stride, n, v);
              },
              [lb, bi, n](float* dst, size_t dn) {
                flushLinear(lb);
                return addBatchSlice(lb->c, 1, lb.get(), (size_t)bi * lb->stride, n, dst, dn);
              });
        };
        out.push_back(scalarResult(gradFunc, gs[i], scores[i]));
      }
      return out;
    }
  }
  return parallelMap(single, gs);
}

/* does the autograd tape behind g contain an entry of a batched op? */
bool tapeHasBatch(const Graph& g, int depth = 0) {
  if (g.lattice() && g.lattice()->batch) return true;
  if (depth > 6) return false;
  for (auto& in : g.inputs())
    if (tapeHasBatch(in, depth + 1)) return true;
  return false;
}

} // namespace

namespace detail {

void keepBatchArcGrads(const std::shared_ptr<LatticeHandle>& h) {
  BatchState& bs = *h->batch;
  std::lock_guard<std::mutex> lk(bs.m);
  // not flushed: the flush re-runs the batch's own backward before any of its lazy gradients reads; no seed: no
  // lazy gradient reads the entries' arc gradients
  if (!bs.flushed || bs.mode < 0 || !bs.arcGrads.empty()) return;
  const auto& na = h->sizes().second;
  std::lock_guard<std::mutex> l(h->owner->lock);
  copyArcGrads(h, na, bs);
}

} // namespace detail

std::vector<Graph> compose(const std::vector<Graph>& a, const std::vector<Graph>& b) {
  return composeBatch(a, b, false);
}
std::vector<Graph> intersect(const std::vector<Graph>& a, const std::vector<Graph>& b) {
  return composeBatch(a, b, true);
}
std::vector<Graph> forwardScore(const std::vector<Graph>& gs) {
  return scoreBatch(gs, false);
}
std::vector<Graph> viterbiScore(const std::vector<Graph>& gs) {
  return scoreBatch(gs, true);
}
std::vector<Graph> viterbiPath(const std::vector<Graph>& gs) {
  // the B entries of one batched lattice, each once: ONE gtnb_viterbi_path, split into B paths
  auto h = entriesOfOneBatch(gs);
  if (!h) return parallelMap(static_cast<Graph (*)(const Graph&)>(viterbiPath), gs);
  auto p = detail::latticePaths(h);
  std::vector<Graph> out;
  out.reserve(gs.size());
  for (auto& g : gs) out.push_back(detail::pathGraph(g, p, g.latticeIndex()));
  return out;
}

void backward(const std::vector<Graph>& gs, bool retainGraph) {
  // The batched ops only record seeds in their gradFuncs: walking the B tapes is host pointer chasing, done
  // in this thread.  Tapes without batched entries keep the reference's thread-per-graph map
  // (bindings/python/gtn/_autograd.cpp:19-62).
  bool batched = false;
  for (size_t i = 0; !batched && i < gs.size() && i < 2; i++) batched = tapeHasBatch(gs[i]);
  if (batched) {
    for (auto g : gs) backward(g, retainGraph);
    return;
  }
  auto fn = [retainGraph](const Graph& g) {
    backward(g, retainGraph);
    return 0;
  };
  parallelMap(fn, gs);
}

} // namespace gtn
