/*
 * gtn/graph.h -- gtn::Graph with the reference's public surface
 * (/root/reference/gtn/graph.h:56-465: every public member keeps its name,
 * signature and semantics) on top of the C ABI (include/gtn_b200.h).
 *
 * What is different underneath:
 *  - a Graph returned by compose()/intersect() with a gtn::linearGraph operand
 *    lives in HBM as one entry of a packed CSR lattice batch; its host
 *    topology is materialised only if somebody inspects nodes or arcs.
 *  - linearGraph(T, C) remembers that it is the emissions chain, and
 *    setWeights() also accepts a device pointer (no round trip through the
 *    host for tensors that are already on the GPU).
 */
#pragma once

#include <cassert>
#include <climits>
#include <cstdint>
#include <functional>
#include <memory>
#include <mutex>
#include <vector>

namespace gtn {

/** The index of the epsilon label (graph.h:21). */
constexpr int epsilon{-1};

namespace detail {
struct LatticeHandle; // a packed device batch (gtnb_lattice) + the context that owns it
struct DeviceBuffer; // device memory owned by a context
} // namespace detail

class Graph {
 private:
  struct Node {
    Node(bool start, bool accept) : start(start), accept(accept){};
    bool start{false};
    bool accept{false};
    std::vector<int> in;
    std::vector<int> out;
  };

  struct Arc {
    Arc(int srcNode, int dstNode, int ilabel, int olabel)
        : srcNode(srcNode), dstNode(dstNode), ilabel(ilabel), olabel(olabel){};
    int srcNode;
    int dstNode;
    int ilabel;
    int olabel;
  };

 public:
  using GradFunc = std::function<void(std::vector<Graph>& inputs, Graph& deltas)>;
  Graph(GradFunc gradFunc, std::vector<Graph> inputs);
  Graph(bool calcGrad = true);

  int addNode(bool start = false, bool accept = false);
  size_t addArc(size_t srcNode, size_t dstNode, int label);
  size_t addArc(size_t srcNode, size_t dstNode, int ilabel, int olabel, float weight = 0.0);

  size_t numArcs() const;
  size_t numNodes() const;
  size_t numStart() const {
    return host().start.size();
  }
  size_t numAccept() const {
    return host().accept.size();
  }

  float item() const;
  static Graph deepCopy(const Graph& src);
  void arcSort(bool olabel = false);
  void markArcSorted(bool olabel = false) {
    if (olabel) {
      sharedGraph_->olabelSorted = true;
    } else {
      sharedGraph_->ilabelSorted = true;
    }
  }
  bool ilabelSorted() const {
    return sharedGraph_->ilabelSorted;
  }
  bool olabelSorted() const {
    return sharedGraph_->olabelSorted;
  }

  float* weights();
  const float* weights() const;
  /** `weights` may be a host pointer (copied, graph.cpp:179-181) or a device pointer. */
  void setWeights(const float* weights);
  void labelsToArray(int* out, bool ilabel = true);
  std::vector<int> labelsToVector(bool ilabel = true);

  void addGrad(std::vector<float>&& other);
  void addGrad(const std::vector<float>& other);
  void addGrad(const Graph& other);
  bool calcGrad() const {
    return sharedGrad_->calcGrad;
  };
  bool isGradAvailable() const {
    return sharedGrad_->grad != nullptr;
  }
  Graph& grad();
  const Graph& grad() const;
  void setCalcGrad(bool calcGrad);
  void zeroGrad();
  std::uintptr_t id();
  GradFunc gradFunc() {
    return sharedGrad_->gradFunc;
  };
  void setGradFunc(GradFunc gradFunc) {
    if (calcGrad()) {
      sharedGrad_->gradFunc = gradFunc;
    }
  }
  std::vector<Graph>& inputs() const {
    return sharedGrad_->inputs;
  };
  void setInputs(std::vector<Graph> inputs);
  Graph withoutWeights() const {
    Graph other = *this;
    other.sharedWeights_ = nullptr;
    return other;
  }

  const std::vector<int>& start() const {
    return host().start;
  };
  const std::vector<int>& accept() const {
    return host().accept;
  };
  bool isStart(size_t i) const {
    return node(i).start;
  };
  bool isAccept(size_t i) const {
    return node(i).accept;
  };
  void makeAccept(size_t i) {
    auto& n = node(i);
    if (!n.accept) {
      sharedGraph_->accept.push_back(static_cast<int>(i));
      n.accept = true;
      topologyEdited();
    }
  };
  size_t numOut(size_t i) const {
    return node(i).out.size();
  }
  const std::vector<int>& out(size_t i) const {
    return node(i).out;
  }
  int out(size_t i, size_t j) const {
    return node(i).out[j];
  }
  size_t numIn(size_t i) const {
    return node(i).in.size();
  }
  const std::vector<int>& in(size_t i) const {
    return node(i).in;
  }
  size_t in(size_t i, size_t j) const {
    return node(i).in[j];
  }

  int srcNode(size_t i) const {
    return arc(i).srcNode;
  }
  int dstNode(size_t i) const {
    return arc(i).dstNode;
  }
  int label(size_t i) const {
    return arc(i).ilabel;
  }
  int ilabel(size_t i) const {
    return arc(i).ilabel;
  }
  int olabel(size_t i) const {
    return arc(i).olabel;
  }
  float weight(size_t i) const;
  void setWeight(size_t i, float weight);

  /* ---- additions (not part of the reference surface) ------------------ */

  /** True for a gtn::linearGraph whose topology has not been edited since. */
  bool isLinear() const {
    return sharedGraph_->linearFrames >= 0;
  }
  int linearFrames() const {
    return sharedGraph_->linearFrames;
  }
  int linearLabels() const {
    return sharedGraph_->linearLabels;
  }
  /** True while the graph exists only in HBM (no host topology yet). */
  bool isDeviceResident() const {
    return sharedGraph_->lattice != nullptr && !sharedGraph_->hostReady;
  }
  /** Device lattice this graph is entry `latticeIndex()` of (may be null). */
  std::shared_ptr<detail::LatticeHandle> lattice() const {
    return sharedGraph_->lattice;
  }
  /**
   * The lattice, but only while it still IS this graph: null once the topology was edited (the
   * edit drops it) or this handle's weights are no longer the lattice's (setWeights, setWeight, a
   * write through weights(), or a gradient graph that merely shares the topology).  The device
   * shortest-distance / path ops use this one and otherwise re-pack the host view.
   */
  std::shared_ptr<detail::LatticeHandle> scoringLattice() const {
    if (!sharedWeights_ || !sharedWeights_->latticeWeights) return nullptr;
    return sharedGraph_->lattice;
  }
  int latticeIndex() const {
    return sharedGraph_->latticeIndex;
  }
  /** Attach a device lattice entry (used by compose); host topology becomes lazy. */
  static Graph fromLattice(
      std::shared_ptr<detail::LatticeHandle> lattice,
      int index,
      GradFunc gradFunc,
      std::vector<Graph> inputs);
  /** Device copy of the weights (set by setWeights(device pointer) or cached by an earlier op). */
  std::shared_ptr<detail::DeviceBuffer> deviceWeights() const;
  /** Remember a device copy of the current host weights; dropped as soon as they may change. */
  void cacheDeviceWeights(std::shared_ptr<detail::DeviceBuffer> buf) const;
  /**
   * Install a gradient whose values still live on the device: `fetch` fills the host
   * vector the first time anybody reads it.  When a gradient is already present the
   * contribution is queued behind it and added when the gradient is read: fetching it
   * now could run a batch's deferred backward in the middle of backward().
   * acc (optional): adds the contribution straight into dst (no temporary); returns false if it cannot, then
   * fetch + add is used.
   */
  void addLazyGrad(
      size_t numArcs, std::function<void(std::vector<float>&)> fetch,
      std::function<bool(float* dst, size_t n)> acc = nullptr);
  /** True while these weights are exactly one contribution that is still on the device (see addLazyGrad). */
  bool hasLazyWeights() const {
    return sharedWeights_ && sharedWeights_->lazyFetch != nullptr && sharedWeights_->lazyAdds.empty();
  }
  /** True while any contribution to these weights has not been added up on the host yet. */
  bool hasPendingWeights() const {
    return sharedWeights_ && (sharedWeights_->lazyFetch != nullptr || !sharedWeights_->lazyAdds.empty());
  }
  /**
   * The sum of the contributions to these weights that were made on the host, resolving nothing that is still on
   * the device.  Returns false, leaving `out` alone, when there are none.
   */
  bool hostContributions(std::vector<float>& out) const;
  /** The slice of a batch-wide device buffer that holds these weights, if a batched list op gathered them. */
  std::shared_ptr<detail::DeviceBuffer> batchSlice(size_t* offset) const;
  void cacheBatchSlice(std::shared_ptr<detail::DeviceBuffer> buf, size_t offset) const;

 private:
  size_t addArc(size_t srcNode, size_t dstNode, int label, float) = delete;
  size_t addArc(size_t srcNode, size_t dstNode, int label, double) = delete;

  struct SharedGraph {
    std::vector<Arc> arcs;
    std::vector<Node> nodes;
    std::vector<int> start;
    std::vector<int> accept;
    bool ilabelSorted{false};
    bool olabelSorted{false};
    std::mutex grad_lock;
    // emissions chain marker (creations.cpp:20-33)
    int linearFrames{-1};
    int linearLabels{-1};
    // lazily materialised device lattice entry
    std::shared_ptr<detail::LatticeHandle> lattice;
    int latticeIndex{0};
    bool hostReady{true};
    std::mutex materialize_lock;
  };

  struct SharedWeights {
    std::vector<float> host;
    std::shared_ptr<detail::DeviceBuffer> device; // set by setWeights(device pointer)
    bool hostStale{false}; // device holds the truth, host not yet filled
    std::function<void(std::vector<float>&)> lazyFetch; // see addLazyGrad, fromLattice
    // further contributions that arrived while a gradient was already present: added to the host vector when
    // somebody reads it (the batched list ops install one per op and entry)
    struct LazyAdd {
      std::function<void(std::vector<float>&)> fetch; // empty for a host contribution
      std::function<bool(float*, size_t)> acc; // may be empty
      std::vector<float> host; // the values of a host contribution (addGrad)
    };
    std::vector<LazyAdd> lazyAdds;
    // a slice of a batch-wide device buffer that holds exactly these weights (gathered by a batched list
    // op, gtn/batched.cpp); dropped with `device` whenever the weights may change
    std::shared_ptr<detail::DeviceBuffer> batch;
    size_t batchOffset{0};
    bool latticeWeights{false}; // these ARE the (unmodified) arc weights of sharedGraph_->lattice
    std::mutex lock;
  };

  struct SharedGrad {
    GradFunc gradFunc{nullptr};
    std::vector<Graph> inputs;
    std::unique_ptr<Graph> grad{nullptr};
    bool calcGrad;
  };

  // after any topology edit: the device forms no longer describe this graph
  void topologyEdited() {
    sharedGraph_->linearFrames = sharedGraph_->linearLabels = -1;
    sharedGraph_->lattice.reset();
    if (sharedWeights_) sharedWeights_->latticeWeights = false;
  }
  // host topology, materialising it from the device lattice on first use
  const SharedGraph& host() const;
  SharedGraph& host();
  void materialize() const;
  std::vector<float>& hostWeights() const;

  const Node& node(size_t i) const {
    assert(i < numNodes());
    return host().nodes[i];
  }
  Node& node(size_t i) {
    return host().nodes[i];
  }
  const Arc& arc(size_t i) const {
    assert(i < numArcs());
    return host().arcs[i];
  }

  std::shared_ptr<SharedGraph> sharedGraph_{std::make_shared<SharedGraph>()};
  std::shared_ptr<SharedWeights> sharedWeights_{std::make_shared<SharedWeights>()};
  std::shared_ptr<SharedGrad> sharedGrad_{std::make_shared<SharedGrad>()};

  friend Graph linearGraph(int M, int N, bool calcGrad);
};

} // namespace gtn
