/*
 * tests/emu/graph_viterbi_emu.cpp -- TEST INFRASTRUCTURE: runs the SOURCE of gtn_b200/csrc/k_implicit.cu's tropical
 * forward instantiations and its traceback kernel (gtnb_graph_viterbi's device route) on the CPU through
 * tests/emu/simt_emu.h.  The kernels and layouts are picked as launch_implicit_forward / _trace pick them (unless the
 * caller overrides the lanes or the traceback's block); only the device tables are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_implicit.cu"

#include <vector>

using gtnb::GraphMeta;

extern "C" {

/*
 * viterbiPath / viterbiScore of intersect(g_b, emissions_b): the TROP forward, then implicit_trace_kernel.
 *   Tables as emu_graph_arc takes them (n_nodes, node_flags, in_ptr local to each graph, in_src / in_label / in_arc /
 *   in_w per in-entry, labels in [0, C)); emissions [B][T][C], input_lens[B].
 *   arc: the arc-label instantiations; lanes: -1 the kernel launch_implicit_forward would pick, 0 the one-CTA-per-
 *   utterance kernel (fast path or several nodes per thread, its own choice), else the wide kernel with that many
 *   lanes per node; frames: the traceback's staged block (0: as launched).
 *   Outputs: paths / arcs [B][T], scores [B], status [B] (bit 1 non-finite, bit 2 tie on the traced path).
 * Returns the lanes per node of the forward, negative on error.
 */
int emu_graph_viterbi(
    int B, int T, int C, const float* emissions, const int32_t* input_lens, const int32_t* n_nodes,
    const uint8_t* node_flags, const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label,
    const int32_t* in_arc, const float* in_w, int arc, int lanes, int frames, int32_t* paths, int32_t* arcs,
    float* scores_out, int32_t* status) {
  using namespace gtnb;
  std::vector<GraphMeta> meta(B);
  std::vector<uint8_t> flags;
  std::vector<int32_t> ptr, src, lab, ids;
  std::vector<float> w;
  long long nb = 0, pb = 0, ab = 0, scores_len = 0;
  int maxN = 0, maxA = 0, max_in = 0, max_out = 0;
  for (int b = 0; b < B; b++) {
    const int N = n_nodes[b], A = in_ptr[pb + N];
    GraphMeta& m = meta[b];
    std::memset(&m, 0, sizeof(m));
    m.sg_node_base = (long long)ptr.size();
    m.sg_arc_base = (long long)src.size();
    m.emis_off = (long long)b * T * C;
    m.node_base = scores_len;
    m.T = input_lens ? input_lens[b] : T;
    m.sg_N = N;
    m.sg_A = A;
    for (int n = 0; n <= N; n++) ptr.push_back(in_ptr[pb + n]);
    for (int n = 0; n < N; n++) flags.push_back(node_flags[nb + n]);
    flags.push_back(0);
    std::vector<int> outdeg(N, 0);
    for (int n = 0; n < N; n++) max_in = std::max(max_in, in_ptr[pb + n + 1] - in_ptr[pb + n]);
    for (int a = 0; a < A; a++) {
      src.push_back(in_src[ab + a]);
      lab.push_back(in_label[ab + a]);
      ids.push_back(in_arc[ab + a]);
      w.push_back(in_w[ab + a]);
      max_out = std::max(max_out, ++outdeg[in_src[ab + a]]);
    }
    scores_len += (long long)(m.T + 1) * ((N + 3) & ~3);
    maxN = std::max(maxN, N);
    maxA = std::max(maxA, A);
    ab += A;
    nb += N;
    pb += N + 1;
  }
  std::vector<float> scores((size_t)scores_len + 16, 0.0f), out((size_t)std::max(B, 1));
  for (int b = 0; b < B; b++) status[b] = 0;
  const int G = lanes >= 0 ? lanes : wide_lanes(max_in, max_out, maxN, C, false, arc != 0);
  const ImpLayout lf = make_imp_layout(maxN, maxA, false, G > 0, C, arc != 0);
  const auto forward = arc ? implicit_forward_kernel_for<true, true>(G) : implicit_forward_kernel_for<false, true>(G);
  emu::launch(B, kImpThreads, lf.total, [&] {
    forward(meta.data(), flags.data(), ptr.data(), src.data(), lab.data(), w.data(), emissions, scores.data(),
            out.data(), status, C, lf);
  });
  const TraceLayout lt = frames > 0 ? make_trace_layout(maxN, maxA, C, frames) : trace_layout(maxN, maxA, C);
  emu::launch(B, kImpThreads, lt.total, [&] {
    implicit_trace_kernel(meta.data(), flags.data(), ptr.data(), src.data(), lab.data(), w.data(), ids.data(),
                          emissions, scores.data(), status, paths, arcs, scores_out, T, C, lt);
  });
  if (emu::g_launch_failed.exchange(false)) return -emu::kEmuNoThreads;
  return G;
}

} // extern "C"
