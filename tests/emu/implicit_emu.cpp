/*
 * tests/emu/implicit_emu.cpp -- TEST INFRASTRUCTURE: runs the SOURCE of gtn_b200/csrc/k_implicit.cu
 * (the criterion's implicit-lattice sweeps: the hot kernels of bench.py) on the CPU through
 * tests/emu/simt_emu.h.  emu_implicit_general picks its kernels and layouts as launch_implicit_forward / _backward
 * do; emu_implicit and emu_implicit_ctc run the narrow kernels directly.  The device tables are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_ctc.cu"
#include "../../gtn_b200/csrc/k_implicit.cu"

#include <vector>

using gtnb::GraphMeta;

namespace {

struct Tables {
  std::vector<GraphMeta> meta;
  std::vector<uint8_t> flags;
  std::vector<int32_t> in_ptr, in_src, in_label, in_arc;
  std::vector<float> in_w;
  long long scores_len = 0;
  int maxN = 0, maxA = 0;
};

/* graph b given as CSR by destination: ptr[N+1], src, label, w (labels already matched) */
void add_graph(Tables& t, int b, int T_frames, long long emis_off, int N, const uint8_t* fl, const int32_t* ptr,
               const int32_t* src, const int32_t* label, const float* w) {
  GraphMeta m;
  std::memset(&m, 0, sizeof(m));
  m.sg_node_base = (long long)t.in_ptr.size();
  m.sg_arc_base = (long long)t.in_src.size();
  m.emis_off = emis_off;
  m.node_base = t.scores_len;
  m.T = T_frames;
  m.sg_N = N;
  m.sg_A = ptr[N];
  for (int n = 0; n <= N; n++) t.in_ptr.push_back(ptr[n]);
  for (int n = 0; n < N; n++) t.flags.push_back(fl[n]);
  t.flags.push_back(0);
  for (int a = 0; a < ptr[N]; a++) {
    t.in_src.push_back(src[a]);
    t.in_label.push_back(label[a]);
    t.in_w.push_back(w[a]);
    t.in_arc.push_back(a);
  }
  const int pitch = (N + 3) & ~3;
  t.scores_len += (long long)(T_frames + 1) * pitch;
  t.maxN = std::max(t.maxN, N);
  t.maxA = std::max(t.maxA, (int)ptr[N]);
  t.meta.push_back(m);
  (void)b;
}

} // namespace

extern "C" {

/*
 * forwardScore(intersect(g_b, emissions_b)) and its backward (deltas = -1, as gtnb_ctc_loss seeds
 * it) for B graphs given as concatenated CSR-by-destination tables:
 *   n_nodes[B]; node_flags (bit 0 start, bit 1 accept), in_ptr (N_b + 1 entries per graph, arc
 *   offsets local to the graph), in_src / in_label / in_w per in-entry.
 *   emissions [B][T][C], input_lens[B]; out_scores[B]; grad [B][T][C] zero on entry; status[B].
 */
int emu_implicit(
    int B, int T, int C, const float* emissions, const int32_t* input_lens, const int32_t* n_nodes,
    const uint8_t* node_flags, const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label,
    const float* in_w, float* out_scores, float* grad, int32_t* status) {
  Tables t;
  long long nb = 0, pb = 0, ab = 0;
  for (int b = 0; b < B; b++) {
    const int N = n_nodes[b];
    add_graph(t, b, input_lens ? input_lens[b] : T, (long long)b * T * C, N, node_flags + nb, in_ptr + pb,
              in_src + ab, in_label + ab, in_w + ab);
    ab += in_ptr[pb + N];
    nb += N;
    pb += N + 1;
  }
  std::vector<float> scores((size_t)t.scores_len + 16, 0.0f);
  for (int b = 0; b < B; b++) status[b] = 0;
  const gtnb::ImpLayout lf = gtnb::make_imp_layout(t.maxN, t.maxA, false);
  emu::launch(B, gtnb::kImpThreads, lf.total, [&] {
    gtnb::implicit_forward_kernel(t.meta.data(), t.flags.data(), t.in_ptr.data(), t.in_src.data(),
                                  t.in_label.data(), t.in_w.data(), emissions, scores.data(), out_scores, status,
                                  C, lf);
  });
  std::vector<float> deltas(B, -1.0f);
  const gtnb::ImpLayout lb = gtnb::make_imp_layout(t.maxN, t.maxA, true);
  emu::launch(B, gtnb::kImpThreads, lb.total, [&] {
    gtnb::implicit_backward_kernel<false>(t.meta.data(), t.flags.data(), t.in_ptr.data(), t.in_src.data(),
                                          t.in_label.data(), t.in_w.data(), t.in_arc.data(), nullptr, emissions,
                                          scores.data(), out_scores, deltas.data(), grad, (long long)T * C, C,
                                          lb);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

/*
 * As emu_implicit, with the kernel family picked the way launch_implicit_forward / _backward do (one
 * node per thread, several nodes per thread, or the G-lanes-per-node "wide" kernels for in- / out-degrees
 * above three: dense ASG transitions), the graph-arc gradients included (grad_graph: A_b floats per graph,
 * concatenated, zero on entry; in_arc maps in-entries to Graph arc ids) and caller-chosen deltas.
 * Returns the lanes per node used (0 = the narrow kernels), negative on error.
 */
int emu_implicit_general(
    int B, int T, int C, const float* emissions, const int32_t* input_lens, const int32_t* n_nodes,
    const uint8_t* node_flags, const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label,
    const int32_t* in_arc, const float* in_w, const float* deltas, float* out_scores, float* grad, float* grad_graph,
    int32_t* status) {
  using namespace gtnb;
  Tables t;
  long long nb = 0, pb = 0, ab = 0;
  int max_in = 0, max_out = 0;
  for (int b = 0; b < B; b++) {
    const int N = n_nodes[b];
    add_graph(t, b, input_lens ? input_lens[b] : T, (long long)b * T * C, N, node_flags + nb, in_ptr + pb,
              in_src + ab, in_label + ab, in_w + ab);
    const int A = in_ptr[pb + N];
    std::vector<int> outdeg(N, 0);
    for (int n = 0; n < N; n++) max_in = std::max(max_in, in_ptr[pb + n + 1] - in_ptr[pb + n]);
    for (int a = 0; a < A; a++) max_out = std::max(max_out, ++outdeg[in_src[ab + a]]);
    for (int a = 0; a < A; a++) t.in_arc[t.meta[b].sg_arc_base + a] = in_arc[ab + a];
    t.meta[b].grad_graph_off = ab;
    ab += A;
    nb += N;
    pb += N + 1;
  }
  std::vector<float> scores((size_t)t.scores_len + 16, 0.0f);
  for (int b = 0; b < B; b++) status[b] = 0;
  const int Gf = wide_lanes(max_in, max_out, t.maxN, C, false), Gb = wide_lanes(max_in, max_out, t.maxN, C, true);
  const ImpLayout lf = make_imp_layout(t.maxN, t.maxA, false, Gf > 0, C);
  const ImpLayout lb = make_imp_layout(t.maxN, t.maxA, true, Gb > 0, C);
  emu::launch(B, kImpThreads, lf.total, [&] {
    implicit_forward_kernel_for<false, false>(Gf)(t.meta.data(), t.flags.data(), t.in_ptr.data(), t.in_src.data(),
                                                  t.in_label.data(), t.in_w.data(), emissions, scores.data(),
                                                  out_scores, status, C, lf);
  });
  emu::launch(B, kImpThreads, lb.total, [&] {
    implicit_backward_kernel_for<false>(Gb, true)(t.meta.data(), t.flags.data(), t.in_ptr.data(), t.in_src.data(),
                                                  t.in_label.data(), t.in_w.data(), t.in_arc.data(), grad_graph,
                                                  emissions, scores.data(), out_scores, deltas, grad,
                                                  (long long)T * C, C, lb);
  });
  if (emu::g_launch_failed.exchange(false)) return -emu::kEmuNoThreads;
  return Gb;
}

/*
 * The CTC criterion's device side as gtnb_ctc_loss runs it: k_ctc.cu's ctc_build_kernel writes the
 * target-graph tables, k_implicit.cu sweeps them.  targets concatenated, target_lens[B].
 * Also returns the tables of graph 0 (for a check against the reference's ctcGraph): n_arcs0,
 * ptr0[N0+1], src0 / label0 (capacity 3 N0).
 */
int emu_implicit_ctc(
    int B, int T, int C, const float* emissions, const int32_t* input_lens, const int32_t* targets,
    const int32_t* target_lens, int blank, float* out_scores, float* grad, int32_t* status, int32_t* ptr0,
    int32_t* src0, int32_t* label0) {
  std::vector<GraphMeta> meta(B);
  std::vector<int32_t> tgt_off(B);
  long long nodes = 0, arcs = 0, scores_len = 0, acc = 0, toff = 0;
  int maxN = 0;
  for (int b = 0; b < B; b++) {
    const int L = 2 * target_lens[b] + 1;
    GraphMeta& m = meta[b];
    std::memset(&m, 0, sizeof(m));
    m.sg_node_base = nodes;
    m.sg_arc_base = arcs;
    m.acc_base = acc;
    m.emis_off = (long long)b * T * C;
    m.node_base = scores_len;
    m.T = input_lens ? input_lens[b] : T;
    m.sg_N = L;
    tgt_off[b] = (int32_t)toff;
    toff += target_lens[b];
    nodes += L + 1;
    arcs += 3 * L;
    acc += 2;
    scores_len += (long long)(T + 1) * ((L + 3) & ~3);
    maxN = std::max(maxN, L);
  }
  std::vector<uint8_t> flags(nodes, 0);
  std::vector<int32_t> in_ptr(nodes, 0), in_src(arcs, 0), in_label(arcs, 0), in_arc(arcs, 0), il(arcs, 0),
      ol(arcs, 0), acc_nodes(acc, 0);
  std::vector<float> in_w(arcs, 0.0f);
  emu::launch(B, 256, 0, [&] {
    gtnb::ctc_build_kernel(meta.data(), targets, tgt_off.data(), target_lens, blank, C, flags.data(), in_ptr.data(),
                           in_src.data(), in_label.data(), in_arc.data(), in_w.data(), il.data(), ol.data(),
                           acc_nodes.data());
  });
  int maxA = 0;
  for (int b = 0; b < B; b++) {
    meta[b].sg_A = in_ptr[meta[b].sg_node_base + meta[b].sg_N];
    maxA = std::max(maxA, meta[b].sg_A);
  }
  if (ptr0) {
    const int N0 = meta[0].sg_N;
    for (int n = 0; n <= N0; n++) ptr0[n] = in_ptr[n];
    for (int a = 0; a < in_ptr[N0]; a++) {
      src0[a] = in_src[a];
      label0[a] = in_label[a];
    }
  }
  std::vector<float> scores((size_t)scores_len + 16, 0.0f);
  for (int b = 0; b < B; b++) status[b] = 0;
  const gtnb::ImpLayout lf = gtnb::make_imp_layout(maxN, maxA, false);
  emu::launch(B, gtnb::kImpThreads, lf.total, [&] {
    gtnb::implicit_forward_kernel(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(),
                                  in_w.data(), emissions, scores.data(), out_scores, status, C, lf);
  });
  std::vector<float> deltas(B, -1.0f);
  const gtnb::ImpLayout lb = gtnb::make_imp_layout(maxN, maxA, true);
  emu::launch(B, gtnb::kImpThreads, lb.total, [&] {
    gtnb::implicit_backward_kernel<false>(meta.data(), flags.data(), in_ptr.data(), in_src.data(), in_label.data(),
                                          in_w.data(), in_arc.data(), nullptr, emissions, scores.data(),
                                          out_scores, deltas.data(), grad, (long long)T * C, C, lb);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

} // extern "C"
