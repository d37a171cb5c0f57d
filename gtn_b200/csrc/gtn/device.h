/*
 * gtn/device.h -- glue between the gtn:: C++ surface and the C ABI
 * (include/gtn_b200.h).  Not part of the reference's surface.
 */
#pragma once

#include <memory>
#include <mutex>
#include <utility>
#include <string>
#include <vector>

#include "gtn/graph.h"
#include "gtn_b200.h"

namespace gtn {
namespace detail {

/* One C-ABI context (device + stream).  Every thread gets its own, lazily: the
 * reference's parallelMap worker threads therefore run "one utterance per stream". */
struct Context {
  gtnb_ctx* ctx{nullptr};
  std::mutex lock; // a lattice may be used from a thread other than its creator
  // pinned read-back block for the batched list ops (gtn/batched.cpp): the whole batch's emission gradient
  // comes back in ONE copy and the entries' lazy gradients are host slices of it while `pinnedOwner` says so
  // slot 0: a batched lattice's emission gradients, slot 1: a batched normaliser's
  float* pinned[2]{nullptr, nullptr};
  size_t pinnedCount[2]{0, 0};
  const void* pinnedOwner[2]{nullptr, nullptr};
  ~Context();
};

std::shared_ptr<Context> threadContext();

/** Map a C-ABI status to the exception type the reference throws. */
void check(const std::shared_ptr<Context>& c, int status);

struct DeviceBuffer {
  std::shared_ptr<Context> owner;
  float* ptr{nullptr};
  size_t count{0};
  DeviceBuffer(std::shared_ptr<Context> c, size_t n);
  ~DeviceBuffer();
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;
};

struct LatticeHandle {
  std::shared_ptr<Context> owner;
  gtnb_lattice* lat{nullptr};
  int B{0};
  bool composed{false};
  std::shared_ptr<DeviceBuffer> emissions; // kept alive for the lattice's lifetime
  std::vector<int> frames; // T per entry (composed lattices)
  int labels{0}; // C
  bool linearFirst{false};
  int scoreMode{-1}; // semiring of the node scores currently saved in the lattice (-1: none)
  std::shared_ptr<struct BatchState> batch; // set by the batched list ops (gtn/batched.cpp)
  std::pair<const std::vector<int32_t>&, const std::vector<int32_t>&> sizes(); // (nodes, arcs) per entry, cached
  ~LatticeHandle();

 private:
  std::mutex sizesLock;
  std::vector<int32_t> nn, na;
};

/* Deferred, batched backward of the B entries of one lattice built by a list op: every entry's gradFunc
 * only RECORDS its seed; the first read of any resulting gradient runs gtnb_backward + gtnb_compose_grad
 * once for the whole batch (gtn/batched.cpp). */
struct BatchState {
  std::mutex m;
  int mode{-1}; // semiring of the pending shortest-distance backward (-1: none recorded)
  std::vector<float> sdDelta; // seeds of the shortest-distance backward, per entry (0: not requested)
  std::vector<std::vector<float>> hostDeltas; // arc gradients handed in from the host, per entry (rare)
  bool flushed{false};
  std::shared_ptr<DeviceBuffer> dLinear, dGraph; // gradients w.r.t. the emissions [B][stride] / the graphs' arcs
  size_t stride{0};
  std::vector<size_t> graphOff; // entry b's slab in dGraph
  // the entries' own arc gradients from the recorded seeds, kept on the host once the lattice's arc gradients no
  // longer hold them (host deltas added on top, or a later single-entry backward); empty while they do
  std::vector<std::vector<float>> arcGrads;
};

/* A single-entry op is about to launch a backward on the batched lattice h: if the batch's own backward has
 * already run, keep the entries' arc gradients its lazy gradients still read (gtn/batched.cpp).  Forces nothing. */
void keepBatchArcGrads(const std::shared_ptr<LatticeHandle>& h);

/* The best paths of every entry of a lattice, one gtnb_viterbi_path: entry b's arcs start at b * stride.  maxNodes:
 * the node count of the largest entry, or 0 to read it from the lattice. */
struct LatticePaths {
  int stride{0};
  std::vector<int32_t> arcs, il, ol, len;
  std::vector<float> w;
};
LatticePaths latticePaths(const std::shared_ptr<LatticeHandle>& h, int maxNodes = 0);
/* viterbiPath's result for g from row b of p (shortest.cpp:250-270) */
Graph pathGraph(const Graph& g, const LatticePaths& p, int b);

/* Host arrays backing a gtnb_graph_view of a Graph (valid while alive). */
struct ViewStorage {
  std::vector<uint8_t> flags;
  std::vector<int32_t> src, dst, il, ol, inPtr, inArcs, outPtr, outArcs, start, accept;
  std::vector<float> w;
  gtnb_graph_view view;
};
void makeView(const Graph& g, ViewStorage& s);

/** True if `p` points to device memory; `*device` (optional) receives the GPU it lives on. */
bool isDevicePointer(const void* p, int* device = nullptr);

} // namespace detail
} // namespace gtn
