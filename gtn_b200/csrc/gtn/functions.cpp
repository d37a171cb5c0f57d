/*
 * gtn/functions.cpp -- hot-path functions on top of the C ABI.
 *
 *   compose / intersect    with a linearGraph operand -> gtnb_compose_linear (device);
 *                          otherwise host graph construction (detail::composeHost)
 *   forwardScore / viterbiScore -> gtnb_forward (+ gtnb_backward in the gradFunc)
 *   viterbiPath            -> gtnb_viterbi_path
 *
 * References: gtn/functions.cpp:18-64,225-251,320-330; gtn/functions/compose.cpp;
 * gtn/functions/shortest.cpp.
 */
#include "gtn/functions.h"

#include <algorithm>
#include <cstdlib>
#include <cmath>
#include <limits>
#include <queue>
#include <stdexcept>

#include <cuda_runtime_api.h>

#include "gtn/device.h"
#include "gtn/parallel.h"

namespace gtn {

/* ---- scalar glue --------------------------------------------------------- */

Graph negate(const Graph& g) {
  if (g.numArcs() != 1) {
    throw std::logic_error("[gtn::negate] input must have only one arc");
  }
  auto gradFunc = [](std::vector<Graph>& inputs, Graph& deltas) { inputs[0].addGrad(negate(deltas)); };
  Graph result(gradFunc, {g});
  result.addNode(true);
  result.addNode(false, true);
  result.addArc(0, 1, 0, 0, -g.item());
  return result;
}

Graph add(const Graph& g1, const Graph& g2) {
  if (g1.numArcs() != 1 || g2.numArcs() != 1) {
    throw std::logic_error("[gtn::add] inputs must have only one arc");
  }
  float weight = g1.item() + g2.item();
  auto gradFunc = [](std::vector<Graph>& inputs, Graph& deltas) {
    inputs[0].addGrad(deltas);
    inputs[1].addGrad(deltas);
  };
  Graph result(gradFunc, {g1, g2});
  result.addNode(true);
  result.addNode(false, true);
  result.addArc(0, 1, 0, 0, weight);
  return result;
}

Graph subtract(const Graph& g1, const Graph& g2) {
  if (g1.numArcs() != 1 || g2.numArcs() != 1) {
    throw std::logic_error("[gtn::subtract] inputs must have only one arc");
  }
  float weight = g1.item() - g2.item();
  auto gradFunc = [](std::vector<Graph>& inputs, Graph& deltas) {
    inputs[0].addGrad(deltas);
    if (inputs[1].calcGrad()) {
      inputs[1].addGrad(negate(deltas));
    }
  };
  Graph result(gradFunc, {g1, g2});
  result.addNode(true);
  result.addNode(false, true);
  result.addArc(0, 1, 0, 0, weight);
  return result;
}

Graph clone(const Graph& g, Projection projection /* = Projection::NONE */) {
  auto gradFunc = [](std::vector<Graph>& inputs, Graph& deltas) { inputs[0].addGrad(deltas); };
  Graph out(gradFunc, {g.withoutWeights()});
  for (size_t n = 0; n < g.numNodes(); ++n) {
    out.addNode(g.isStart(n), g.isAccept(n));
  }
  for (size_t a = 0; a < g.numArcs(); ++a) {
    out.addArc(
        g.srcNode(a),
        g.dstNode(a),
        projection == Projection::OUTPUT ? g.olabel(a) : g.ilabel(a),
        projection == Projection::INPUT ? g.ilabel(a) : g.olabel(a),
        g.weight(a));
  }
  return out;
}

Graph projectInput(const Graph& g) {
  return clone(g, Projection::INPUT);
}

Graph projectOutput(const Graph& g) {
  return clone(g, Projection::OUTPUT);
}

/* ---- host composition (general case) ------------------------------------- */

namespace detail {

namespace {

/*
 * Enumerates the arc pairs (i of g1, j of g2) leaving (or entering) a node pair whose
 * g1 output label equals the g2 input label, in the order the reference's matchers do
 * (compose.cpp:211-374): nested loops when nothing is sorted, binary search in the
 * sorted side otherwise (restarting from the previous hit when both are sorted).
 */
class Matcher {
 public:
  enum Kind { UNSORTED, SINGLY, DOUBLY };
  Matcher(const Graph& g1, const Graph& g2, Kind kind, bool searchG1)
      : g1_(g1), g2_(g2), kind_(kind), searchG1Cfg_(searchG1) {}

  void match(int lnode, int rnode, bool matchIn) {
    const auto& lv = matchIn ? g1_.in(lnode) : g1_.out(lnode);
    const auto& rv = matchIn ? g2_.in(rnode) : g2_.out(rnode);
    if (kind_ == UNSORTED) {
      lv_ = &lv;
      rv_ = &rv;
      li_ = ri_ = 0;
      return;
    }
    searchG1_ = kind_ == DOUBLY ? lv.size() > rv.size() : searchG1Cfg_;
    s_ = searchG1_ ? &lv : &rv;
    q_ = searchG1_ ? &rv : &lv;
    qi_ = si_ = sb_ = 0;
  }

  bool hasNext() {
    if (kind_ == UNSORTED) {
      for (; li_ < lv_->size(); ++li_) {
        for (; ri_ < rv_->size(); ++ri_) {
          if (g1_.olabel((*lv_)[li_]) == g2_.ilabel((*rv_)[ri_])) return true;
        }
        ri_ = 0;
      }
      return false;
    }
    if (qi_ == q_->size()) return false;
    if (si_ != s_->size() && qlabel((*q_)[qi_]) == slabel((*s_)[si_])) return true;
    if (si_ != sb_) ++qi_;
    for (; qi_ < q_->size(); ++qi_) {
      const int ql = qlabel((*q_)[qi_]);
      auto lb = std::lower_bound(
          s_->begin() + sb_, s_->end(), ql, [this](int arc, int val) { return slabel(arc) < val; });
      const size_t pos = lb - s_->begin();
      if (kind_ == SINGLY) {
        si_ = pos;
        if (si_ == s_->size()) continue;
        if (slabel((*s_)[si_]) == ql) return true;
      } else {
        sb_ = pos;
        if (sb_ == s_->size()) return false;
        if (slabel((*s_)[sb_]) == ql) {
          si_ = sb_;
          return true;
        }
      }
    }
    return false;
  }

  std::pair<int, int> next() {
    if (kind_ == UNSORTED) return {(*lv_)[li_], (*rv_)[ri_++]};
    if (searchG1_) return {(*s_)[si_++], (*q_)[qi_]};
    return {(*q_)[qi_], (*s_)[si_++]};
  }

 private:
  int qlabel(int arc) const {
    return searchG1_ ? g2_.ilabel(arc) : g1_.olabel(arc);
  }
  int slabel(int arc) const {
    return searchG1_ ? g1_.olabel(arc) : g2_.ilabel(arc);
  }
  const Graph& g1_;
  const Graph& g2_;
  Kind kind_;
  bool searchG1Cfg_;
  bool searchG1_{false};
  const std::vector<int>*lv_{nullptr}, *rv_{nullptr}, *s_{nullptr}, *q_{nullptr};
  size_t li_{0}, ri_{0}, qi_{0}, si_{0}, sb_{0};
};

} // namespace

Graph composeHost(const Graph& first, const Graph& second, bool intersectMode) {
  const bool s1 = intersectMode ? (first.ilabelSorted() || first.olabelSorted()) : first.olabelSorted();
  const bool s2 = intersectMode ? (second.ilabelSorted() || second.olabelSorted()) : second.ilabelSorted();
  Matcher matcher(
      first, second, (s1 && s2) ? Matcher::DOUBLY : ((s1 || s2) ? Matcher::SINGLY : Matcher::UNSORTED), s1);

  const size_t n1 = first.numNodes(), n2 = second.numNodes();
  auto index = [n1](int a, int b) { return (size_t)a + n1 * (size_t)b; };

  // states that can reach an accepting pair (compose.cpp:64-104)
  std::vector<bool> reachable(n1 * n2, false);
  std::queue<std::pair<int, int>> todo;
  for (auto f : first.accept()) {
    for (auto s : second.accept()) {
      todo.emplace(f, s);
      reachable[index(f, s)] = true;
    }
  }
  auto epsBack = [&](bool inSecond, std::pair<int, int> cur) {
    const auto& edges = inSecond ? second.in(cur.second) : first.in(cur.first);
    const bool sorted = inSecond ? second.ilabelSorted() : first.olabelSorted();
    for (auto i : edges) {
      const int label = inSecond ? second.ilabel(i) : first.olabel(i);
      if (label != epsilon) {
        if (sorted) break;
        continue;
      }
      const int un = inSecond ? second.srcNode(i) : first.srcNode(i);
      const size_t idx = inSecond ? index(cur.first, un) : index(un, cur.second);
      if (!reachable[idx]) {
        if (inSecond)
          todo.emplace(cur.first, un);
        else
          todo.emplace(un, cur.second);
      }
      reachable[idx] = true;
    }
  };
  while (!todo.empty()) {
    auto cur = todo.front();
    todo.pop();
    matcher.match(cur.first, cur.second, true);
    while (matcher.hasNext()) {
      auto ij = matcher.next();
      const int u1 = first.srcNode(ij.first), u2 = second.srcNode(ij.second);
      if (!reachable[index(u1, u2)]) todo.emplace(u1, u2);
      reachable[index(u1, u2)] = true;
    }
    epsBack(false, cur);
    epsBack(true, cur);
  }

  // forward construction (compose.cpp:389-489)
  Graph ngraph(nullptr, {first, second});
  std::vector<int> newNodes(n1 * n2, -1);
  for (auto a : first.start()) {
    for (auto b : second.start()) {
      if (reachable[index(a, b)]) {
        newNodes[index(a, b)] = ngraph.addNode(true, first.isAccept(a) && second.isAccept(b));
        todo.emplace(a, b);
      }
    }
  }
  std::vector<std::pair<int, int>> gradInfo;
  auto addArcTo = [&](int curNode, int d1, int d2, float w, int il, int ol) {
    const size_t idx = index(d1, d2);
    if (!reachable[idx]) return false;
    if (newNodes[idx] < 0) {
      newNodes[idx] = ngraph.addNode(
          first.isStart(d1) && second.isStart(d2), first.isAccept(d1) && second.isAccept(d2));
      todo.emplace(d1, d2);
    }
    ngraph.addArc(curNode, newNodes[idx], il, ol, w);
    return true;
  };
  auto epsForward = [&](bool inSecond, int curNode, std::pair<int, int> cur) {
    const auto& edges = inSecond ? second.out(cur.second) : first.out(cur.first);
    const bool sorted = inSecond ? second.ilabelSorted() : first.olabelSorted();
    for (auto i : edges) {
      const int label = inSecond ? second.ilabel(i) : first.olabel(i);
      if (label != epsilon) {
        if (sorted) break;
        continue;
      }
      const bool ok = addArcTo(
          curNode,
          inSecond ? cur.first : first.dstNode(i),
          inSecond ? second.dstNode(i) : cur.second,
          inSecond ? second.weight(i) : first.weight(i),
          inSecond ? epsilon : first.ilabel(i),
          inSecond ? second.olabel(i) : epsilon);
      if (ok) gradInfo.emplace_back(inSecond ? -1 : i, inSecond ? i : -1);
    }
  };
  while (!todo.empty()) {
    auto cur = todo.front();
    todo.pop();
    const int curNode = newNodes[index(cur.first, cur.second)];
    bool epsMatched = false;
    matcher.match(cur.first, cur.second, false);
    while (matcher.hasNext()) {
      auto ij = matcher.next();
      const int i = ij.first, j = ij.second;
      if (first.olabel(i) == epsilon) {
        epsMatched = true;
        continue;
      }
      if (addArcTo(
              curNode, first.dstNode(i), second.dstNode(j), first.weight(i) + second.weight(j),
              first.ilabel(i), second.olabel(j))) {
        gradInfo.emplace_back(i, j);
      }
    }
    if (!epsMatched || second.isAccept(cur.second) || !first.isAccept(cur.first)) {
      epsForward(false, curNode, cur);
    }
    if (!epsMatched || first.isAccept(cur.first)) {
      epsForward(true, curNode, cur);
    }
  }

  // gradFunc (compose.cpp:496-518)
  auto gradFunc = [gradInfo = std::move(gradInfo)](std::vector<Graph>& inputs, Graph& deltas) {
    const bool c1 = inputs[0].calcGrad(), c2 = inputs[1].calcGrad();
    std::vector<float> g1(c1 ? inputs[0].numArcs() : 0, 0.0f), g2(c2 ? inputs[1].numArcs() : 0, 0.0f);
    for (size_t k = 0; k < gradInfo.size(); k++) {
      const float d = deltas.weight(k);
      if (c1 && gradInfo[k].first >= 0) g1[gradInfo[k].first] += d;
      if (c2 && gradInfo[k].second >= 0) g2[gradInfo[k].second] += d;
    }
    inputs[0].addGrad(std::move(g1));
    inputs[1].addGrad(std::move(g2));
  };
  ngraph.setGradFunc(std::move(gradFunc));
  return ngraph;
}

bool matchedSideHasEpsilon(const Graph& g, bool useIlabel) {
  for (size_t a = 0; a < g.numArcs(); a++) {
    if ((useIlabel ? g.ilabel(a) : g.olabel(a)) == epsilon) return true;
  }
  return false;
}

namespace {

/* emissions of a linear graph on the device: reuse setWeights(device ptr), else upload */
std::shared_ptr<DeviceBuffer> emissionsOnDevice(const Graph& linear, const std::shared_ptr<Context>& c) {
  const size_t n = (size_t)linear.linearFrames() * (size_t)linear.linearLabels();
  auto dev = linear.deviceWeights();
  // a cached copy is only valid for work on the stream that owns it
  if (dev && dev->count == n && dev->owner == c) return dev;
  auto buf = std::make_shared<DeviceBuffer>(c, n);
  if (dev && dev->count == n && n) {
    // device weights owned by another thread's stream: drain it, then take a private copy so that
    // the stream-ordered free of either buffer can never race the other stream's kernels
    {
      std::lock_guard<std::mutex> lo(dev->owner->lock);
      check(dev->owner, gtnb_ctx_synchronize(dev->owner->ctx));
    }
    std::lock_guard<std::mutex> l(c->lock);
    if (cudaMemcpyAsync(buf->ptr, dev->ptr, sizeof(float) * n, cudaMemcpyDeviceToDevice,
                        (cudaStream_t)gtnb_ctx_stream(c->ctx)) != cudaSuccess)
      throw std::runtime_error("[gtn] device copy of the emissions failed");
    return buf;
  }
  if (n) {
    const float* w = linear.weights();
    std::lock_guard<std::mutex> l(c->lock);
    check(c, gtnb_memcpy_h2d(c->ctx, buf->ptr, w, sizeof(float) * n));
    check(c, gtnb_ctx_synchronize(c->ctx));
  }
  if (!dev) linear.cacheDeviceWeights(buf); // forwardScore(e) and intersect(ctc, e) share one upload
  return buf;
}

/* frame-synchronous device composition of `graph` with the emissions chain `linear` */
bool composeLinearDevice(const Graph& first, const Graph& second, bool linearFirst, Graph& out) {
  const Graph& linear = linearFirst ? first : second;
  const Graph& graph = linearFirst ? second : first;
  const int T = linear.linearFrames(), C = linear.linearLabels();
  if (C <= 0 || graph.isDeviceResident()) return false;
  if (matchedSideHasEpsilon(graph, linearFirst)) return false;
  auto c = threadContext();
  auto emis = emissionsOnDevice(linear, c);
  ViewStorage vs;
  makeView(graph, vs);
  gtnb_lattice* lat = nullptr;
  int rc;
  {
    std::lock_guard<std::mutex> l(c->lock);
    rc = gtnb_compose_linear(c->ctx, 1, &vs.view, 1, linearFirst ? 1 : 0, &T, C, emis->ptr, (int64_t)T * C, &lat);
  }
  if (rc == GTNB_ERR_UNSUPPORTED) return false; // e.g. too large to materialise: host path
  check(c, rc);
  auto handle = std::make_shared<LatticeHandle>();
  handle->owner = c;
  handle->lat = lat;
  handle->B = 1;
  handle->composed = true;
  handle->emissions = emis;
  handle->frames = {T};
  handle->labels = C;
  handle->linearFirst = linearFirst;

  const size_t graphArcs = graph.numArcs();
  const size_t emisArcs = (size_t)T * C;
  // compose's gradFunc (compose.cpp:496-518) as a device scatter
  auto gradFunc = [handle, linearFirst, graphArcs, emisArcs](std::vector<Graph>& inputs, Graph& deltas) {
    Graph& gGraph = inputs[linearFirst ? 1 : 0];
    Graph& gLinear = inputs[linearFirst ? 0 : 1];
    const bool needGraph = gGraph.calcGrad(), needLinear = gLinear.calcGrad();
    auto& c = handle->owner;
    std::vector<float> hostGraph(needGraph ? graphArcs : 0), hostLinear(needLinear ? emisArcs : 0);
    if (needGraph || needLinear) {
      // arc gradients: still on the device if they came straight from the
      // shortest-distance gradFunc, otherwise pushed up from the host deltas
      const bool onDevice = deltas.hasLazyWeights();
      const float* hostDeltas = onDevice ? nullptr : deltas.weights();
      DeviceBuffer dGraph(c, std::max<size_t>(graphArcs, 1)), dLinear(c, std::max<size_t>(emisArcs, 1));
      std::lock_guard<std::mutex> l(c->lock);
      if (!onDevice) check(c, gtnb_lattice_set_arc_grads(c->ctx, handle->lat, 0, hostDeltas));
      check(c, gtnb_memset(c->ctx, dGraph.ptr, 0, sizeof(float) * std::max<size_t>(graphArcs, 1)));
      check(c, gtnb_memset(c->ctx, dLinear.ptr, 0, sizeof(float) * std::max<size_t>(emisArcs, 1)));
      check(c, gtnb_compose_grad(
                   c->ctx, handle->lat, needGraph ? dGraph.ptr : nullptr,
                   needLinear ? dLinear.ptr : nullptr, (int64_t)emisArcs));
      if (needGraph && graphArcs)
        check(c, gtnb_memcpy_d2h(c->ctx, hostGraph.data(), dGraph.ptr, sizeof(float) * graphArcs));
      if (needLinear && emisArcs)
        check(c, gtnb_memcpy_d2h(c->ctx, hostLinear.data(), dLinear.ptr, sizeof(float) * emisArcs));
      check(c, gtnb_ctx_synchronize(c->ctx));
    }
    // compose.cpp:516-517 adds to both inputs unconditionally (addGrad ignores calcGrad == false)
    inputs[linearFirst ? 1 : 0].addGrad(std::move(hostGraph));
    inputs[linearFirst ? 0 : 1].addGrad(std::move(hostLinear));
  };
  out = Graph::fromLattice(handle, 0, gradFunc, {first, second});
  return true;
}

} // namespace

namespace {
int g_composePolicy = -1;
}

int deviceCount() {
  static const int n = [] {
    int c = 0;
    if (cudaGetDeviceCount(&c) != cudaSuccess) {
      cudaGetLastError();
      c = 0;
    }
    return c;
  }();
  return n;
}

int composeDevicePolicy() {
  if (g_composePolicy < 0) {
    const char* e = std::getenv("GTNB_COMPOSE_DEVICE");
    const std::string v = e ? e : "auto";
    g_composePolicy = v == "always" ? 1 : (v == "never" ? 2 : 0);
  }
  return g_composePolicy;
}

void setComposeDevicePolicy(int policy) {
  g_composePolicy = policy;
}

bool composeGraphsDevice(
    const std::vector<const Graph*>& first, const std::vector<const Graph*>& second, bool intersectMode,
    std::vector<Graph>& out) {
  const size_t B = std::max(first.size(), second.size());
  if (first.empty() || second.empty() || (first.size() != B && first.size() != 1) ||
      (second.size() != B && second.size() != 1))
    return false;
  auto c = threadContext();
  std::vector<ViewStorage> v1(first.size()), v2(second.size());
  std::vector<gtnb_graph_view> w1(first.size()), w2(second.size());
  {
    // the host views of all operands, on the reference's own worker threads (parallel_map.h)
    std::vector<int> idx(first.size() + second.size());
    for (size_t i = 0; i < idx.size(); i++) idx[i] = (int)i;
    auto one = [&](int i) {
      if ((size_t)i < first.size())
        makeView(*first[i], v1[i]);
      else
        makeView(*second[i - first.size()], v2[i - first.size()]);
      return 0;
    };
    if (idx.size() > 2)
      parallelMap(one, idx);
    else
      for (int i : idx) one(i);
    for (size_t i = 0; i < first.size(); i++) w1[i] = v1[i].view;
    for (size_t i = 0; i < second.size(); i++) w2[i] = v2[i].view;
  }
  // which matcher the reference would pick (functions.cpp:225-251)
  std::vector<int32_t> kind(B);
  for (size_t b = 0; b < B; b++) {
    const Graph& a = *first[first.size() == 1 ? 0 : b];
    const Graph& g = *second[second.size() == 1 ? 0 : b];
    const bool s1 = intersectMode ? (a.ilabelSorted() || a.olabelSorted()) : a.olabelSorted();
    const bool s2 = intersectMode ? (g.ilabelSorted() || g.olabelSorted()) : g.ilabelSorted();
    kind[b] = (s1 && s2) ? 3 : (s1 ? 1 : (s2 ? 2 : 0));
  }
  gtnb_composed* res = nullptr;
  int rc;
  {
    std::lock_guard<std::mutex> l(c->lock);
    rc = gtnb_compose_graphs(c->ctx, (int)B, w1.data(), (int)w1.size(), w2.data(), (int)w2.size(), kind.data(), &res);
  }
  if (rc == GTNB_ERR_UNSUPPORTED) return false;
  check(c, rc);
  struct Guard {
    std::shared_ptr<Context> c;
    gtnb_composed* r;
    ~Guard() {
      std::lock_guard<std::mutex> l(c->lock);
      gtnb_composed_destroy(c->ctx, r);
    }
  } guard{c, res};
  auto buildOne = [&](int bi) {
    const size_t b = (size_t)bi;
    int32_t N = 0, A = 0;
    gtnb_composed_sizes(res, (int)b, &N, &A);
    std::vector<uint8_t> fl(N);
    std::vector<int32_t> src(A), dst(A), il(A), ol(A), gi1(A), gi2(A);
    std::vector<float> w(A);
    {
      std::lock_guard<std::mutex> l(c->lock);
      check(c, gtnb_composed_download(c->ctx, res, (int)b, fl.data(), src.data(), dst.data(), il.data(), ol.data(),
                                      w.data(), gi1.data(), gi2.data()));
    }
    const Graph& a = *first[first.size() == 1 ? 0 : b];
    const Graph& g = *second[second.size() == 1 ? 0 : b];
    Graph ng(nullptr, {a, g});
    for (int n = 0; n < N; n++) ng.addNode(fl[n] & 1, fl[n] & 2);
    for (int k = 0; k < A; k++) ng.addArc(src[k], dst[k], il[k], ol[k], w[k]);
    // compose's gradFunc (compose.cpp:496-518)
    auto gradFunc = [gi1 = std::move(gi1), gi2 = std::move(gi2)](std::vector<Graph>& inputs, Graph& deltas) {
      const bool c1 = inputs[0].calcGrad(), c2 = inputs[1].calcGrad();
      std::vector<float> g1(c1 ? inputs[0].numArcs() : 0, 0.0f), g2(c2 ? inputs[1].numArcs() : 0, 0.0f);
      for (size_t k = 0; k < gi1.size(); k++) {
        const float d = deltas.weight(k);
        if (c1 && gi1[k] >= 0) g1[gi1[k]] += d;
        if (c2 && gi2[k] >= 0) g2[gi2[k]] += d;
      }
      inputs[0].addGrad(std::move(g1));
      inputs[1].addGrad(std::move(g2));
    };
    ng.setGradFunc(std::move(gradFunc));
    return ng;
  };
  // the B host Graphs: downloads one after the other (one stream), construction on the worker threads
  std::vector<int> idx(B);
  for (size_t b = 0; b < B; b++) idx[b] = (int)b;
  if (B > 1) {
    out = parallelMap(buildOne, idx);
  } else {
    out.clear();
    out.push_back(buildOne(0));
  }
  return true;
}

namespace {

/* does the device take this general pair?  (see composeDevicePolicy) */
bool generalOnDevice(const Graph& g1, const Graph& g2) {
  const int policy = composeDevicePolicy();
  if (policy == 2 || g1.isDeviceResident() || g2.isDeviceResident() || deviceCount() == 0) return false;
  if (policy == 1) return true;
  // the device beats the host construction once there are enough product states to search.  On an H100
  // (scripts/bench_gcompose.py, profiles/h100_gcompose.json) a single ctc x bigram pair stays faster on the host up
  // to 60 k states (13 vs 20 ms), every pair from 181 k on is 2.5-6x faster on the device (ctc x trigram, lexicon x
  // LM, an epsilon operand x the emissions chain)
  return (double)g1.numNodes() * (double)g2.numNodes() >= kComposeDeviceStates;
}

Graph composeDispatch(const Graph& g1, const Graph& g2, bool intersectMode) {
  Graph out;
  // the frame-synchronous device path needs one operand to be the emissions chain
  if (g2.isLinear() && !g1.isLinear() && composeLinearDevice(g1, g2, false, out)) return out;
  if (g1.isLinear() && composeLinearDevice(g1, g2, true, out)) return out;
  if (g2.isLinear() && composeLinearDevice(g1, g2, false, out)) return out;
  if (generalOnDevice(g1, g2)) {
    std::vector<Graph> res;
    if (composeGraphsDevice({&g1}, {&g2}, intersectMode, res)) return res[0];
  }
  return composeHost(g1, g2, intersectMode);
}

/* shortestDistance on the emissions chain itself (the CTC normaliser, benchmarks/ctc.cpp:157):
 * per-frame reductions, no lattice needed */
Graph shortestDistanceLinear(const Graph& g, bool tropical) {
  auto c = threadContext();
  const int T = g.linearFrames(), C = g.linearLabels();
  auto emis = emissionsOnDevice(g, c);
  float score = 0.0f;
  {
    DeviceBuffer sdev(c, 4);
    std::lock_guard<std::mutex> l(c->lock);
    check(c, gtnb_linear_forward(c->ctx, 1, &T, C, emis->ptr, (int64_t)T * C, tropical ? 1 : 0, sdev.ptr,
                                 nullptr, 0, nullptr, 1.0f));
    check(c, gtnb_memcpy_d2h(c->ctx, &score, sdev.ptr, sizeof(float)));
    check(c, gtnb_ctx_synchronize(c->ctx));
  }
  auto gradFunc = [emis, T, C, tropical](std::vector<Graph>& inputs, Graph& deltas) {
    auto& c = emis->owner;
    const size_t n = (size_t)T * C;
    std::vector<float> grad(n, 0.0f);
    if (n) {
      DeviceBuffer sdev(c, 4), gdev(c, n);
      std::lock_guard<std::mutex> l(c->lock);
      check(c, gtnb_memset(c->ctx, gdev.ptr, 0, sizeof(float) * n));
      check(c, gtnb_linear_forward(c->ctx, 1, &T, C, emis->ptr, (int64_t)n, tropical ? 1 : 0, sdev.ptr,
                                   gdev.ptr, (int64_t)n, nullptr, deltas.item()));
      check(c, gtnb_memcpy_d2h(c->ctx, grad.data(), gdev.ptr, sizeof(float) * n));
      check(c, gtnb_ctx_synchronize(c->ctx));
    }
    inputs[0].addGrad(std::move(grad));
  };
  Graph result(gradFunc, {g});
  result.addNode(true);
  result.addNode(false, true);
  result.addArc(0, 1, 0, 0, score);
  return result;
}

/* shortest distance over one graph on the device.  An entry of a batched lattice (a list intersect) is scored by a
 * launch over the whole batch: the forward and the backward run on all B entries, the backward with a one-hot
 * seed, and this entry's row is taken */
Graph shortestDistanceDevice(const Graph& g, bool tropical) {
  if (g.isLinear() && g.linearLabels() > 0 && !g.isDeviceResident()) return shortestDistanceLinear(g, tropical);
  std::shared_ptr<LatticeHandle> handle;
  bool latticeEntry = false;
  if (g.scoringLattice() && g.scoringLattice()->composed) {
    handle = g.scoringLattice();
    latticeEntry = true;
  } else {
    auto c = threadContext();
    ViewStorage vs;
    makeView(g, vs);
    gtnb_lattice* lat = nullptr;
    {
      std::lock_guard<std::mutex> l(c->lock);
      check(c, gtnb_pack(c->ctx, 1, &vs.view, &lat));
    }
    handle = std::make_shared<LatticeHandle>();
    handle->owner = c;
    handle->lat = lat;
    handle->B = 1;
  }
  auto& c = handle->owner;
  const int B = std::max(handle->B, 1);
  const int bi = latticeEntry ? g.latticeIndex() : 0;
  const bool batchEntry = B > 1;
  std::vector<float> scores(B);
  {
    std::lock_guard<std::mutex> l(c->lock);
    check(c, gtnb_forward(c->ctx, handle->lat, tropical ? 1 : 0, scores.data(), nullptr));
    handle->scoreMode = tropical ? 1 : 0;
  }
  const size_t numArcs = g.numArcs();
  auto gradFunc = [handle, tropical, latticeEntry, batchEntry, B, bi, numArcs](std::vector<Graph>& inputs,
                                                                                Graph& deltas) {
    auto& c = handle->owner;
    std::vector<float> delta(B, 0.0f);
    delta[bi] = deltas.item();
    if (batchEntry && handle->batch) {
      keepBatchArcGrads(handle);
    } else if (latticeEntry && inputs[0].isGradAvailable() && inputs[0].grad().hasPendingWeights()) {
      // a gradient of this lattice still parked on the device would be overwritten by this launch (no batch
      // behind it: resolving it reads the lattice and nothing else)
      inputs[0].grad().weights();
    }
    {
      std::lock_guard<std::mutex> l(c->lock);
      // the lattice may have been re-used by another score op since: restore the node scores
      if (handle->scoreMode != (tropical ? 1 : 0)) {
        check(c, gtnb_forward(c->ctx, handle->lat, tropical ? 1 : 0, nullptr, nullptr));
        handle->scoreMode = tropical ? 1 : 0;
      }
      check(c, gtnb_backward(c->ctx, handle->lat, tropical ? 1 : 0, delta.data()));
    }
    auto fetch = [handle, bi, numArcs](std::vector<float>& v) {
      auto& c = handle->owner;
      v.resize(numArcs);
      if (numArcs == 0) return;
      std::lock_guard<std::mutex> l(c->lock);
      check(c, gtnb_lattice_arc_grads(c->ctx, handle->lat, bi, v.data()));
    };
    if (latticeEntry && !batchEntry) {
      inputs[0].addLazyGrad(numArcs, fetch);
    } else {
      // the next launch on a shared lattice overwrites every entry's arc gradients: read this one now
      std::vector<float> v;
      fetch(v);
      inputs[0].addGrad(std::move(v));
    }
  };
  Graph result(gradFunc, {g});
  result.addNode(true);
  result.addNode(false, true);
  result.addArc(0, 1, 0, 0, scores[bi]);
  return result;
}

} // namespace
} // namespace detail

Graph compose(const Graph& g1, const Graph& g2) {
  return detail::composeDispatch(g1, g2, false);
}

Graph intersect(const Graph& g1, const Graph& g2) {
  return detail::composeDispatch(g1, g2, true);
}

Graph forwardScore(const Graph& g) {
  return detail::shortestDistanceDevice(g, false);
}

Graph viterbiScore(const Graph& g) {
  return detail::shortestDistanceDevice(g, true);
}

namespace detail {

LatticePaths latticePaths(const std::shared_ptr<LatticeHandle>& h, int maxNodes) {
  auto& c = h->owner;
  const int B = std::max(h->B, 1);
  if (maxNodes <= 0) // a path visits each node at most once: the largest entry bounds every row
    for (int b = 0; b < B; b++) maxNodes = std::max(maxNodes, (int)h->sizes().first[b]);
  maxNodes = std::max(maxNodes, 1);
  LatticePaths p;
  p.stride = maxNodes;
  const size_t n = (size_t)B * maxNodes;
  p.arcs.resize(n);
  p.il.resize(n);
  p.ol.resize(n);
  p.w.resize(n);
  p.len.assign(B, 0);
  std::lock_guard<std::mutex> l(c->lock);
  check(c, gtnb_viterbi_path(c->ctx, h->lat, maxNodes, p.arcs.data(), p.il.data(), p.ol.data(), p.w.data(),
                             p.len.data(), nullptr));
  h->scoreMode = -1; // node scores now hold the path recursion
  return p;
}

Graph pathGraph(const Graph& g, const LatticePaths& p, int b) {
  const size_t row = (size_t)b * p.stride;
  const int len = p.len[b];
  Graph out(nullptr, {g});
  if (len >= 0) {
    out.addNode(true, len == 0);
  }
  for (int i = 0; i < len; i++) {
    out.addNode(false, i == len - 1);
    out.addArc(i, i + 1, p.il[row + i], p.ol[row + i], p.w[row + i]);
  }
  // shortest.cpp:262-270: the reference keeps the path arcs end -> start and indexes them
  // with the output graph's (start -> end) arc ids; reproduced as is.
  std::vector<int> rev(p.arcs.begin() + row, p.arcs.begin() + row + std::max(len, 0));
  std::reverse(rev.begin(), rev.end());
  auto gradFunc = [rev = std::move(rev)](std::vector<Graph>& inputs, Graph& deltas) {
    std::vector<float> grad(inputs[0].numArcs(), 0.0f);
    for (size_t a = 0; a < deltas.numArcs(); ++a) {
      grad[rev[a]] += deltas.weight(a);
    }
    inputs[0].addGrad(std::move(grad));
  };
  out.setGradFunc(std::move(gradFunc));
  return out;
}

} // namespace detail

/* an entry of a batched lattice is decoded by a launch over the whole batch; its row is taken */
Graph viterbiPath(const Graph& g) {
  using namespace detail;
  std::shared_ptr<LatticeHandle> handle;
  int bi = 0;
  if (g.scoringLattice() && g.scoringLattice()->composed) {
    handle = g.scoringLattice();
    bi = g.latticeIndex();
  } else {
    auto c = threadContext();
    ViewStorage vs;
    makeView(g, vs);
    gtnb_lattice* lat = nullptr;
    {
      std::lock_guard<std::mutex> l(c->lock);
      check(c, gtnb_pack(c->ctx, 1, &vs.view, &lat));
    }
    handle = std::make_shared<LatticeHandle>();
    handle->owner = c;
    handle->lat = lat;
    handle->B = 1;
  }
  // (a lattice of its own: g's node count is the row length, no read-back of the sizes)
  return pathGraph(g, latticePaths(handle, handle->B > 1 ? 0 : (int)g.numNodes()), bi);
}

} // namespace gtn
