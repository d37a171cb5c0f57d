/*
 * gtn/graph.cpp -- gtn::Graph (reference: /root/reference/gtn/graph.cpp) plus the
 * lazy host view of device-resident lattices.  Written against the reference's
 * documented behaviour; error messages match the ones its tests pin.
 */
#include "gtn/graph.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <utility>

#include "gtn/device.h"

namespace gtn {

/* ---- detail: contexts, buffers, views -------------------------------- */

namespace detail {

Context::~Context() {
  for (float* p : pinned)
    if (p && ctx) gtnb_host_free(ctx, p);
  if (ctx) gtnb_ctx_destroy(ctx);
}

std::shared_ptr<Context> threadContext() {
  thread_local std::shared_ptr<Context> tls;
  if (!tls) {
    auto c = std::make_shared<Context>();
    int dev = 0;
    cudaGetDevice(&dev);
    int rc = gtnb_ctx_create(dev, nullptr, &c->ctx);
    if (rc != GTNB_OK) {
      throw std::runtime_error(std::string(gtnb_last_error(nullptr)));
    }
    tls = c;
  }
  return tls;
}

void check(const std::shared_ptr<Context>& c, int status) {
  if (status == GTNB_OK) return;
  std::string msg = gtnb_last_error(c ? c->ctx : nullptr);
  switch (status) {
    case GTNB_ERR_INVALID_ARGUMENT:
      throw std::invalid_argument(msg);
    case GTNB_ERR_LOGIC:
      throw std::logic_error(msg);
    default:
      throw std::runtime_error(msg);
  }
}

DeviceBuffer::DeviceBuffer(std::shared_ptr<Context> c, size_t n) : owner(std::move(c)), count(n) {
  void* p = nullptr;
  std::lock_guard<std::mutex> l(owner->lock);
  check(owner, gtnb_device_alloc(owner->ctx, sizeof(float) * std::max<size_t>(n, 4), &p));
  ptr = static_cast<float*>(p);
}

DeviceBuffer::~DeviceBuffer() {
  if (ptr && owner && owner->ctx) {
    std::lock_guard<std::mutex> l(owner->lock);
    gtnb_device_free(owner->ctx, ptr);
  }
}

/* node / arc counts of every entry, read back once per lattice (a batch of B entries answers B numArcs()
 * calls with one device round trip) */
std::pair<const std::vector<int32_t>&, const std::vector<int32_t>&> LatticeHandle::sizes() {
  std::lock_guard<std::mutex> l(sizesLock);
  if (nn.empty()) {
    nn.assign(std::max(B, 1), 0);
    na.assign(std::max(B, 1), 0);
    std::lock_guard<std::mutex> cl(owner->lock);
    check(owner, gtnb_lattice_sizes(owner->ctx, lat, nn.data(), na.data()));
  }
  return {nn, na};
}

LatticeHandle::~LatticeHandle() {
  if (lat && owner && owner->ctx) {
    std::lock_guard<std::mutex> l(owner->lock);
    gtnb_lattice_destroy(owner->ctx, lat);
  }
}

bool isDevicePointer(const void* p, int* device) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  if (device) *device = attr.device;
  return attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
}

void makeView(const Graph& g, ViewStorage& s) {
  const int N = (int)g.numNodes(), A = (int)g.numArcs();
  s.flags.resize(N);
  s.src.resize(A);
  s.dst.resize(A);
  s.il.resize(A);
  s.ol.resize(A);
  s.w.resize(A);
  s.inPtr.assign(N + 1, 0);
  s.outPtr.assign(N + 1, 0);
  s.inArcs.clear();
  s.outArcs.clear();
  for (int n = 0; n < N; n++) {
    s.flags[n] = (g.isStart(n) ? 1 : 0) | (g.isAccept(n) ? 2 : 0);
    for (auto a : g.in(n)) s.inArcs.push_back(a);
    for (auto a : g.out(n)) s.outArcs.push_back(a);
    s.inPtr[n + 1] = (int)s.inArcs.size();
    s.outPtr[n + 1] = (int)s.outArcs.size();
  }
  const float* w = A ? g.weights() : nullptr;
  for (int a = 0; a < A; a++) {
    s.src[a] = g.srcNode(a);
    s.dst[a] = g.dstNode(a);
    s.il[a] = g.ilabel(a);
    s.ol[a] = g.olabel(a);
    s.w[a] = w[a];
  }
  s.start.assign(g.start().begin(), g.start().end());
  s.accept.assign(g.accept().begin(), g.accept().end());
  std::memset(&s.view, 0, sizeof(s.view));
  s.view.num_nodes = N;
  s.view.num_arcs = A;
  s.view.node_flags = s.flags.data();
  s.view.arc_src = s.src.data();
  s.view.arc_dst = s.dst.data();
  s.view.arc_ilabel = s.il.data();
  s.view.arc_olabel = s.ol.data();
  s.view.weights = s.w.data();
  s.view.in_ptr = s.inPtr.data();
  s.view.in_arcs = s.inArcs.data();
  s.view.out_ptr = s.outPtr.data();
  s.view.out_arcs = s.outArcs.data();
  s.view.start = s.start.data();
  s.view.num_start = (int)s.start.size();
  s.view.accept = s.accept.data();
  s.view.num_accept = (int)s.accept.size();
}

} // namespace detail

/* ---- construction ------------------------------------------------------ */

Graph::Graph(GradFunc gradFunc, std::vector<Graph> inputs) {
  sharedGrad_->calcGrad = false;
  // a graph computes a gradient if any of its inputs does (graph.cpp:16-27)
  for (auto& g : inputs) {
    sharedGrad_->calcGrad |= g.calcGrad();
  }
  if (calcGrad()) {
    sharedGrad_->gradFunc = std::move(gradFunc);
    sharedGrad_->inputs = std::move(inputs);
  }
}

Graph::Graph(bool calcGrad /* = true */) {
  sharedGrad_->calcGrad = calcGrad;
}

Graph Graph::fromLattice(
    std::shared_ptr<detail::LatticeHandle> lattice,
    int index,
    GradFunc gradFunc,
    std::vector<Graph> inputs) {
  Graph g(std::move(gradFunc), std::move(inputs));
  g.sharedGraph_->lattice = std::move(lattice);
  g.sharedGraph_->latticeIndex = index;
  g.sharedGraph_->hostReady = false;
  // The arc weights belong to THIS handle's SharedWeights only: gradient graphs share sharedGraph_
  // (addGrad) but own their weights, so materialising the topology through one of them must never
  // write the lattice's forward weights over a gradient (round-1 advisor finding).
  auto lat = g.sharedGraph_->lattice;
  g.sharedWeights_->latticeWeights = true;
  g.sharedWeights_->lazyFetch = [lat, index](std::vector<float>& host) {
    std::vector<int32_t> nn(lat->B), na(lat->B);
    std::lock_guard<std::mutex> cl(lat->owner->lock);
    detail::check(lat->owner, gtnb_lattice_sizes(lat->owner->ctx, lat->lat, nn.data(), na.data()));
    host.assign(std::max(na[index], 1), 0.0f);
    detail::check(
        lat->owner,
        gtnb_lattice_download(
            lat->owner->ctx, lat->lat, index, nullptr, nullptr, nullptr, nullptr, nullptr, host.data(),
            nullptr, nullptr));
    host.resize(na[index]);
  };
  return g;
}

/* ---- lazy host view ---------------------------------------------------- */

const Graph::SharedGraph& Graph::host() const {
  if (!sharedGraph_->hostReady) materialize();
  return *sharedGraph_;
}

Graph::SharedGraph& Graph::host() {
  if (!sharedGraph_->hostReady) materialize();
  return *sharedGraph_;
}

void Graph::materialize() const {
  auto& sg = *sharedGraph_;
  std::lock_guard<std::mutex> l(sg.materialize_lock);
  if (sg.hostReady) return;
  if (!sg.lattice) {
    // a gtn::linearGraph that nobody has looked at yet (creations.cpp): build the chain now
    const int M = sg.linearFrames, N = sg.linearLabels;
    sg.nodes.clear();
    sg.arcs.clear();
    sg.start.assign(1, 0);
    sg.accept.assign(1, M);
    sg.nodes.reserve((size_t)M + 1);
    sg.arcs.reserve((size_t)M * N);
    sg.nodes.emplace_back(true, false);
    for (int m = 1; m <= M; m++) {
      sg.nodes.emplace_back(false, m == M);
      sg.nodes[m - 1].out.reserve(N);
      sg.nodes[m].in.reserve(N);
      for (int n = 0; n < N; n++) {
        const int idx = (m - 1) * N + n;
        sg.arcs.emplace_back(m - 1, m, n, n);
        sg.nodes[m - 1].out.push_back(idx);
        sg.nodes[m].in.push_back(idx);
      }
    }
    sg.hostReady = true;
    return;
  }
  auto lat = sg.lattice;
  std::vector<int32_t> nn(lat->B), na(lat->B);
  {
    std::lock_guard<std::mutex> cl(lat->owner->lock);
    detail::check(lat->owner, gtnb_lattice_sizes(lat->owner->ctx, lat->lat, nn.data(), na.data()));
  }
  const int N = nn[sg.latticeIndex], A = na[sg.latticeIndex];
  std::vector<uint8_t> flags(std::max(N, 1));
  std::vector<int32_t> src(std::max(A, 1)), dst(std::max(A, 1)), il(std::max(A, 1)), ol(std::max(A, 1));
  {
    // topology only: the weights are fetched by the owning handle's SharedWeights (fromLattice)
    std::lock_guard<std::mutex> cl(lat->owner->lock);
    detail::check(
        lat->owner,
        gtnb_lattice_download(
            lat->owner->ctx, lat->lat, sg.latticeIndex, flags.data(), src.data(), dst.data(),
            il.data(), ol.data(), nullptr, nullptr, nullptr));
  }
  sg.nodes.clear();
  sg.arcs.clear();
  sg.start.clear();
  sg.accept.clear();
  sg.nodes.reserve(N);
  sg.arcs.reserve(A);
  for (int n = 0; n < N; n++) {
    sg.nodes.emplace_back(flags[n] & 1, (flags[n] & 2) != 0);
    if (flags[n] & 1) sg.start.push_back(n);
    if (flags[n] & 2) sg.accept.push_back(n);
  }
  for (int a = 0; a < A; a++) {
    sg.arcs.emplace_back(src[a], dst[a], il[a], ol[a]);
    sg.nodes[src[a]].out.push_back(a);
    sg.nodes[dst[a]].in.push_back(a);
  }
  sg.hostReady = true;
}

size_t Graph::numArcs() const {
  auto& sg = *sharedGraph_;
  if (!sg.hostReady)
    return sg.lattice ? (size_t)sg.lattice->sizes().second[sg.latticeIndex]
                      : (size_t)sg.linearFrames * (size_t)sg.linearLabels; // a pending linearGraph
  return sg.arcs.size();
}

size_t Graph::numNodes() const {
  auto& sg = *sharedGraph_;
  if (!sg.hostReady)
    return sg.lattice ? (size_t)sg.lattice->sizes().first[sg.latticeIndex] : (size_t)sg.linearFrames + 1;
  return sg.nodes.size();
}

/* ---- topology edits ---------------------------------------------------- */

int Graph::addNode(bool start /* = false */, bool accept /* = false */) {
  auto& sg = host();
  int idx = static_cast<int>(sg.nodes.size());
  sg.nodes.emplace_back(start, accept);
  if (start) sg.start.push_back(idx);
  if (accept) sg.accept.push_back(idx);
  sg.ilabelSorted = false;
  sg.olabelSorted = false;
  topologyEdited();
  return idx;
}

size_t Graph::addArc(size_t srcNode, size_t dstNode, int label) {
  return addArc(srcNode, dstNode, label, label);
}

size_t Graph::addArc(size_t srcNode, size_t dstNode, int ilabel, int olabel, float weight /* = 0 */) {
  assert(ilabel >= epsilon && olabel >= epsilon);
  auto& sg = host();
  int idx = static_cast<int>(sg.arcs.size());
  sg.arcs.emplace_back(static_cast<int>(srcNode), static_cast<int>(dstNode), ilabel, olabel);
  hostWeights().push_back(weight);
  sg.nodes[srcNode].out.push_back(idx);
  sg.nodes[dstNode].in.push_back(idx);
  sg.ilabelSorted = false;
  sg.olabelSorted = false;
  topologyEdited();
  return idx;
}

float Graph::item() const {
  if (numArcs() != 1) {
    throw std::invalid_argument("[Graph::item] Cannot convert Graph with more than 1 arc to a scalar.");
  }
  return weight(0);
}

Graph Graph::deepCopy(const Graph& src) {
  Graph out(src.calcGrad());
  const auto& sg = src.host();
  out.sharedGraph_->arcs = sg.arcs;
  out.sharedGraph_->nodes = sg.nodes;
  out.sharedGraph_->start = sg.start;
  out.sharedGraph_->accept = sg.accept;
  out.sharedGraph_->linearFrames = sg.linearFrames;
  out.sharedGraph_->linearLabels = sg.linearLabels;
  out.sharedWeights_->host = src.hostWeights();
  return out;
}

void Graph::arcSort(bool olabel /* = false */) {
  auto& sg = host();
  if ((olabel && sg.olabelSorted) || (!olabel && sg.ilabelSorted)) {
    return;
  }
  sg.olabelSorted = olabel;
  sg.ilabelSorted = !olabel;
  auto less = [olabel, &arcs = sg.arcs](int a, int b) {
    return olabel ? arcs[a].olabel < arcs[b].olabel : arcs[a].ilabel < arcs[b].ilabel;
  };
  for (auto& n : sg.nodes) {
    std::sort(n.in.begin(), n.in.end(), less);
    std::sort(n.out.begin(), n.out.end(), less);
  }
}

/* ---- weights ----------------------------------------------------------- */

std::vector<float>& Graph::hostWeights() const {
  assert(sharedWeights_ != nullptr);
  auto& sw = *sharedWeights_;
  if (sw.lazyFetch) {
    std::lock_guard<std::mutex> l(sw.lock);
    if (sw.lazyFetch) {
      sw.lazyFetch(sw.host);
      sw.lazyFetch = nullptr;
    }
  }
  if (!sw.lazyAdds.empty()) {
    std::lock_guard<std::mutex> l(sw.lock);
    // (256 entries x 256 KB per minibatch come through here: no zero fill, no temporary where the source can add
    // in place, one scratch vector per thread otherwise)
    thread_local std::vector<float> part;
    for (auto& a : sw.lazyAdds) {
      if (!a.fetch) {
        for (size_t i = 0; i < sw.host.size() && i < a.host.size(); i++) sw.host[i] += a.host[i];
        continue;
      }
      if (a.acc && a.acc(sw.host.data(), sw.host.size())) continue;
      part.clear();
      a.fetch(part);
      for (size_t i = 0; i < sw.host.size() && i < part.size(); i++) sw.host[i] += part[i];
    }
    sw.lazyAdds.clear();
  }
  if (sw.hostStale) {
    std::lock_guard<std::mutex> l(sw.lock);
    if (sw.hostStale) {
      sw.host.resize(sw.device->count);
      auto& c = sw.device->owner;
      std::lock_guard<std::mutex> cl(c->lock);
      detail::check(c, gtnb_memcpy_d2h(c->ctx, sw.host.data(), sw.device->ptr, sizeof(float) * sw.device->count));
      detail::check(c, gtnb_ctx_synchronize(c->ctx));
      sw.hostStale = false;
    }
  }
  return sw.host;
}

float* Graph::weights() {
  // (no host(): the weights do not need the topology -- a pending linearGraph or a device-resident lattice
  // stays unmaterialised when only its weights or gradient are read)
  auto& hw = hostWeights();
  // the caller may write through the pointer: neither the device copy nor a device lattice built
  // from the old values can be trusted any longer
  sharedWeights_->device.reset();
  sharedWeights_->batch.reset();
  sharedWeights_->latticeWeights = false;
  return hw.data();
}

const float* Graph::weights() const {
  return hostWeights().data();
}

float Graph::weight(size_t i) const {
  return hostWeights()[i];
}

void Graph::setWeight(size_t i, float weight) {
  hostWeights()[i] = weight;
  sharedWeights_->device.reset();
  sharedWeights_->batch.reset();
  sharedWeights_->latticeWeights = false;
}

std::shared_ptr<detail::DeviceBuffer> Graph::deviceWeights() const {
  if (!sharedWeights_) return nullptr;
  std::lock_guard<std::mutex> l(sharedWeights_->lock);
  return sharedWeights_->device;
}

std::shared_ptr<detail::DeviceBuffer> Graph::batchSlice(size_t* offset) const {
  if (!sharedWeights_) return nullptr;
  std::lock_guard<std::mutex> l(sharedWeights_->lock);
  if (offset) *offset = sharedWeights_->batchOffset;
  return sharedWeights_->batch;
}

void Graph::cacheBatchSlice(std::shared_ptr<detail::DeviceBuffer> buf, size_t offset) const {
  if (!sharedWeights_) return;
  std::lock_guard<std::mutex> l(sharedWeights_->lock);
  sharedWeights_->batch = std::move(buf);
  sharedWeights_->batchOffset = offset;
}

void Graph::cacheDeviceWeights(std::shared_ptr<detail::DeviceBuffer> buf) const {
  if (!sharedWeights_) return;
  std::lock_guard<std::mutex> l(sharedWeights_->lock);
  if (!sharedWeights_->device) sharedWeights_->device = std::move(buf);
}

void Graph::setWeights(const float* weights) {
  const size_t n = numArcs();
  auto& sw = *sharedWeights_;
  int ptrDevice = -1;
  if (n > 0 && detail::isDevicePointer(weights, &ptrDevice)) {
    auto c = detail::threadContext();
    if (ptrDevice != gtnb_ctx_device(c->ctx))
      throw std::invalid_argument(
          "[Graph::setWeights] device pointer lives on GPU " + std::to_string(ptrDevice) +
          ", this thread's context on GPU " + std::to_string(gtnb_ctx_device(c->ctx)));
    auto buf = std::make_shared<detail::DeviceBuffer>(c, n);
    {
      std::lock_guard<std::mutex> cl(c->lock);
      cudaStream_t st = (cudaStream_t)gtnb_ctx_stream(c->ctx);
      // Order the copy after the producer of `weights`.  The context's stream is non-blocking, so
      // nothing orders it after e.g. a torch kernel still writing the tensor: wait for everything
      // queued so far on the legacy default stream (torch's default) and on the per-thread default
      // stream.  A producer on any other stream must synchronise before calling (INTEGRATION.md).
      cudaEvent_t ev;
      bool ok = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) == cudaSuccess;
      for (cudaStream_t prod : {cudaStreamLegacy, cudaStreamPerThread}) {
        ok = ok && cudaEventRecord(ev, prod) == cudaSuccess && cudaStreamWaitEvent(st, ev, 0) == cudaSuccess;
      }
      if (ok) cudaEventDestroy(ev);
      if (!ok ||
          cudaMemcpyAsync(buf->ptr, weights, sizeof(float) * n, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        throw std::runtime_error("[Graph::setWeights] device copy failed");
    }
    std::lock_guard<std::mutex> l(sw.lock);
    sw.device = buf;
    sw.batch.reset();
    sw.hostStale = true;
    sw.lazyFetch = nullptr;
    sw.latticeWeights = false;
    return;
  }
  std::lock_guard<std::mutex> l(sw.lock);
  sw.host.resize(n);
  std::copy(weights, weights + n, sw.host.data());
  sw.device.reset();
  sw.batch.reset();
  sw.hostStale = false;
  sw.lazyFetch = nullptr;
  sw.latticeWeights = false;
}

void Graph::labelsToArray(int* out, bool ilabel) {
  for (size_t i = 0; i < numArcs(); ++i) {
    out[i] = ilabel ? this->ilabel(i) : olabel(i);
  }
}

std::vector<int> Graph::labelsToVector(bool ilabel) {
  std::vector<int> out(numArcs());
  labelsToArray(out.data(), ilabel);
  return out;
}

/* ---- gradients --------------------------------------------------------- */

Graph& Graph::grad() {
  return const_cast<Graph&>(static_cast<const Graph&>(*this).grad());
}

const Graph& Graph::grad() const {
  if (!calcGrad()) {
    throw std::logic_error("[Graph::grad] Gradient calculation disabled.");
  }
  if (!sharedGrad_->grad) {
    throw std::logic_error("[Graph::grad] Gradient not calculated yet.");
  }
  return *sharedGrad_->grad;
}

void Graph::addGrad(std::vector<float>&& other) {
  if (calcGrad()) {
    if (other.size() != numArcs()) {
      throw std::logic_error("[Graph::addGrad] Invalid grad size.");
    }
    std::lock_guard<std::mutex> lock(sharedGraph_->grad_lock);
    if (isGradAvailable()) {
      auto& sw = *sharedGrad_->grad->sharedWeights_;
      if (sw.lazyFetch || !sw.lazyAdds.empty()) {
        // resolving a pending gradient here could run a batch's deferred backward before every seed is in
        std::lock_guard<std::mutex> l(sw.lock);
        sw.lazyAdds.push_back({nullptr, nullptr, std::move(other)});
        return;
      }
      auto& gw = sharedGrad_->grad->hostWeights();
      for (size_t i = 0; i < other.size(); i++) gw[i] += other[i];
    } else {
      // the gradient graph shares the topology (graph.cpp:102-104)
      sharedGrad_->grad = std::make_unique<Graph>(false);
      sharedGrad_->grad->sharedGraph_ = sharedGraph_;
      sharedGrad_->grad->sharedWeights_->host = std::move(other);
    }
  }
}

void Graph::addLazyGrad(
    size_t /* numArcs */, std::function<void(std::vector<float>&)> fetch, std::function<bool(float*, size_t)> acc) {
  if (!calcGrad()) return;
  std::lock_guard<std::mutex> lock(sharedGraph_->grad_lock);
  if (!isGradAvailable()) {
    sharedGrad_->grad = std::make_unique<Graph>(false);
    sharedGrad_->grad->sharedGraph_ = sharedGraph_;
    sharedGrad_->grad->sharedWeights_->lazyFetch = std::move(fetch);
    return;
  }
  // queue this contribution behind the gradient already present, on the host or not: fetching it now could
  // run its batch's deferred backward in the middle of backward(), before every seed is recorded (the batched
  // list ops park one per op and entry until somebody reads)
  auto& gw = *sharedGrad_->grad->sharedWeights_;
  std::lock_guard<std::mutex> l(gw.lock);
  gw.lazyAdds.push_back({std::move(fetch), std::move(acc), {}});
}

bool Graph::hostContributions(std::vector<float>& out) const {
  if (!sharedWeights_) return false;
  auto& sw = *sharedWeights_;
  if (!hasPendingWeights()) {
    out = hostWeights();
    return true;
  }
  std::lock_guard<std::mutex> l(sw.lock);
  bool any = !sw.lazyFetch; // then the host vector holds the first contribution
  for (auto& a : sw.lazyAdds) any = any || !a.fetch;
  if (!any) return false;
  const size_t n = numArcs();
  if (sw.lazyFetch)
    out.assign(n, 0.0f);
  else
    out = sw.host;
  out.resize(n, 0.0f);
  for (auto& a : sw.lazyAdds)
    if (!a.fetch)
      for (size_t i = 0; i < n && i < a.host.size(); i++) out[i] += a.host[i];
  return true;
}

void Graph::addGrad(const std::vector<float>& other) {
  addGrad(std::vector<float>(other));
}

void Graph::addGrad(const Graph& other) {
  addGrad(other.hostWeights());
}

void Graph::setCalcGrad(bool calcGrad) {
  sharedGrad_->calcGrad = calcGrad;
  if (!calcGrad) {
    sharedGrad_->gradFunc = nullptr;
    sharedGrad_->inputs.clear();
    sharedGrad_->grad.reset();
  }
}

void Graph::setInputs(std::vector<Graph> inputs) {
  sharedGrad_->inputs = std::move(inputs);
}

void Graph::zeroGrad() {
  sharedGrad_->grad.reset();
}

std::uintptr_t Graph::id() {
  return reinterpret_cast<std::uintptr_t>(sharedGrad_.get());
}

} // namespace gtn
