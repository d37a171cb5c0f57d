/*
 * gtn/functions.h -- the hot-path functions of the reference's gtn/functions.h:19-152,
 * same names, argument meaning and error behaviour.  compose / intersect with a
 * gtn::linearGraph operand, forwardScore, viterbiScore, viterbiPath and their
 * gradients run as sm_90a kernels through the C ABI; general (epsilon / non-linear)
 * composition and the rational operations (concat, closure, union_, remove:
 * gtn/rational.cpp) are host graph construction, as in the reference.
 */
#pragma once

#include <vector>

#include "gtn/graph.h"

namespace gtn {

/** Negate a scalar graph (functions.cpp:18-30). */
Graph negate(const Graph& g);
/** Add two scalar graphs (functions.cpp:32-46). */
Graph add(const Graph& g1, const Graph& g2);
/** Subtract two scalar graphs (functions.cpp:48-64). */
Graph subtract(const Graph& g1, const Graph& g2);

enum class Projection {
  NONE = 0,
  INPUT = 1,
  OUTPUT = 2,
};
/** Recorded copy of a graph, optionally projected (functions.cpp:66-91). */
Graph clone(const Graph& g, Projection projection = Projection::NONE);
Graph projectInput(const Graph& g);
Graph projectOutput(const Graph& g);

/** Concatenation: accept states of g_i are joined to the start states of g_{i+1} by epsilon arcs (functions.cpp:93-155). */
Graph concat(const Graph& g1, const Graph& g2);
Graph concat(const std::vector<Graph>& graphs);
/** Kleene closure (functions.cpp:157-190). */
Graph closure(const Graph& g);
/** Union (functions.cpp:192-223). */
Graph union_(const std::vector<Graph>& graphs);
/** Remove arcs labelled `label` (default: epsilon), bridging their end points (functions.cpp:253-318). */
Graph remove(const Graph& g, int label = epsilon);
Graph remove(const Graph& g, int ilabel, int olabel);

/** Compose two transducers (functions.cpp:225-237). */
Graph compose(const Graph& g1, const Graph& g2);
/** Intersect two acceptors (functions.cpp:239-251). */
Graph intersect(const Graph& g1, const Graph& g2);

/** Shortest distance in the log semiring (functions.cpp:320-322). */
Graph forwardScore(const Graph& g);
/** Shortest distance in the tropical semiring (functions.cpp:324-326). */
Graph viterbiScore(const Graph& g);
/** Best path as a chain graph (functions.cpp:328-330). */
Graph viterbiPath(const Graph& g);

/**
 * List forms (bindings/python/gtn/_functions.cpp:69-135): one packed launch for the whole list where the graphs
 * allow it -- every pair a (graph, gtn::linearGraph) composition, every score or path over the entries of such a
 * batch, every score over emission chains -- else parallelMap of the single-graph function.  See gtn/batched.cpp.
 */
std::vector<Graph> compose(const std::vector<Graph>& graphs1, const std::vector<Graph>& graphs2);
std::vector<Graph> intersect(const std::vector<Graph>& graphs1, const std::vector<Graph>& graphs2);
std::vector<Graph> forwardScore(const std::vector<Graph>& graphs);
std::vector<Graph> viterbiScore(const std::vector<Graph>& graphs);
/** The entries of one batched lattice, each once: one decoding launch for the list; else parallelMap. */
std::vector<Graph> viterbiPath(const std::vector<Graph>& graphs);

namespace detail {
/** Host graph construction for the general case (epsilons, arbitrary operands). */
Graph composeHost(const Graph& first, const Graph& second, bool intersectMode);
/** Does an arc of g carry epsilon on the side matched against a linear graph's labels? */
bool matchedSideHasEpsilon(const Graph& g, bool useIlabel);
/** detail::compose (compose.cpp:377-522) for B arbitrary operand pairs in one device call (k_gcompose.cu):
 * same node / arc numbering and gradInfo as the reference.  Size-1 lists broadcast.  Returns false (and
 * leaves `out` alone) when the device cannot take the batch (product state space too large). */
bool composeGraphsDevice(
    const std::vector<const Graph*>& first, const std::vector<const Graph*>& second, bool intersectMode,
    std::vector<Graph>& out);
/** GTNB_COMPOSE_DEVICE = auto (default) | always | never: whether compose / intersect of two arbitrary
 * graphs runs on the device.  auto: when there is a GPU and the product state space has at least
 * kComposeDeviceStates states (a list: kComposeDeviceListStates per pair, one batched call amortises the launches)
 * -- from there on the device search beat the host construction on an H100 (scripts/bench_gcompose.py). */
constexpr double kComposeDeviceStates = 65536.0;
constexpr double kComposeDeviceListStates = 32768.0;
int composeDevicePolicy(); // 0 auto, 1 always, 2 never
void setComposeDevicePolicy(int policy);
int deviceCount();
} // namespace detail

} // namespace gtn
