/*
 * tests/emu/graph_emu.cpp -- TEST INFRASTRUCTURE: runs the SOURCE of gtn_b200/csrc/k_implicit.cu's arc-label
 * instantiations (gtnb_graph_loss on graphs whose nodes have in-arcs of different labels) on the CPU through
 * tests/emu/simt_emu.h.  Only the launch geometry and the device tables are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_implicit.cu"

#include <vector>

using gtnb::GraphMeta;

extern "C" {

/*
 * forwardScore(intersect(g_b, emissions_b)) and its backward with caller-chosen deltas, through the arc-label
 * kernels picked the way launch_implicit_forward / _backward pick them for a lattice with arc_labels set (several
 * nodes per thread, or the G-lanes-per-node wide kernels; force_narrow: always the former).
 *   n_nodes[B]; node_flags (bit 0 start, bit 1 accept); in_ptr (N_b + 1 entries per graph, offsets local to the
 *   graph); in_src / in_label / in_arc (Graph arc id) / in_w per in-entry (labels in [0, C));
 *   arc_base[B]: first slot of graph b in grad_graph (Graph arc numbering, zero on entry).
 *   emissions [B][T][C], input_lens[B]; out_scores[B]; grad [B][T][C] zero on entry; status[B].
 * Returns the lanes per node of the backward (0 = several nodes per thread), negative on error.
 */
int emu_graph_arc(
    int B, int T, int C, const float* emissions, const int32_t* input_lens, const int32_t* n_nodes,
    const uint8_t* node_flags, const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label,
    const int32_t* in_arc, const float* in_w, const int64_t* arc_base, const float* deltas, int force_narrow,
    float* out_scores, float* grad, float* grad_graph, int32_t* status) {
  using namespace gtnb;
  std::vector<GraphMeta> meta(B);
  std::vector<uint8_t> flags;
  std::vector<int32_t> ptr, src, lab, arc;
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
    m.grad_graph_off = arc_base[b];
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
      arc.push_back(in_arc[ab + a]);
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
  std::vector<float> scores((size_t)scores_len + 16, 0.0f);
  for (int b = 0; b < B; b++) status[b] = 0;
  const int Gf = force_narrow ? 0 : wide_lanes(max_in, max_out, maxN, C, false, true);
  const int Gb = force_narrow ? 0 : wide_lanes(max_in, max_out, maxN, C, true, true);
  const ImpLayout lf = make_imp_layout(maxN, maxA, false, Gf > 0, C, true);
  const ImpLayout lb = make_imp_layout(maxN, maxA, true, Gb > 0, C, true);
#define FWD_ARGS \
  meta.data(), flags.data(), ptr.data(), src.data(), lab.data(), w.data(), emissions, scores.data(), out_scores, status, C, lf
#define BWD_ARGS                                                                                                \
  meta.data(), flags.data(), ptr.data(), src.data(), lab.data(), w.data(), arc.data(), grad_graph, emissions, \
      scores.data(), out_scores, deltas, grad, (long long)T * C, C, lb
#define RUN_FWD(K) emu::launch(B, kImpThreads, lf.total, [&] { K(FWD_ARGS); })
#define RUN_BWD(K) emu::launch(B, kImpThreads, lb.total, [&] { K(BWD_ARGS); })
  switch (Gf) {
    case 0: RUN_FWD(implicit_forward_kernel<true>); break;
    case 1: RUN_FWD((implicit_forward_wide_kernel<1, true>)); break;
    case 2: RUN_FWD((implicit_forward_wide_kernel<2, true>)); break;
    case 4: RUN_FWD((implicit_forward_wide_kernel<4, true>)); break;
    case 8: RUN_FWD((implicit_forward_wide_kernel<8, true>)); break;
    case 16: RUN_FWD((implicit_forward_wide_kernel<16, true>)); break;
    default: RUN_FWD((implicit_forward_wide_kernel<32, true>)); break;
  }
  switch (Gb) {
    case 0: RUN_BWD((implicit_backward_kernel<true, true>)); break;
    case 1: RUN_BWD((implicit_backward_wide_kernel<1, true, true>)); break;
    case 2: RUN_BWD((implicit_backward_wide_kernel<2, true, true>)); break;
    case 4: RUN_BWD((implicit_backward_wide_kernel<4, true, true>)); break;
    case 8: RUN_BWD((implicit_backward_wide_kernel<8, true, true>)); break;
    case 16: RUN_BWD((implicit_backward_wide_kernel<16, true, true>)); break;
    default: RUN_BWD((implicit_backward_wide_kernel<32, true, true>)); break;
  }
#undef RUN_FWD
#undef RUN_BWD
#undef FWD_ARGS
#undef BWD_ARGS
  if (emu::g_launch_failed.exchange(false)) return -emu::kEmuNoThreads;
  return Gb;
}

} // extern "C"
