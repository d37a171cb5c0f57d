/*
 * tests/emu/compose_emu.cpp -- TEST INFRASTRUCTURE: the SOURCE of gtn_b200/csrc/k_compose.cu
 * (frame-synchronous device composition: alive sets, counts, scans, CSR emission, and compose's
 * gradFunc) and of k_shortest.cu's generic shortest-distance kernels on the CPU through
 * tests/emu/simt_emu.h.  The slab layout of gtnb_capi.cu's composed_alloc and the launch geometry
 * of launch_compose / launch_forward / launch_backward are restated here; the staged kernels' plan, fused layout and
 * instantiations are k_staged.cu's own.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_compose.cu"
#include "../../gtn_b200/csrc/k_shortest.cu"
#include "../../gtn_b200/csrc/k_order.cu"
#include "../../gtn_b200/csrc/k_staged.cu"

#include <vector>

using gtnb::GraphMeta;

namespace {
long long align_up(long long x, long long a) {
  return (x + a - 1) / a * a;
}


/* the packed batch as composed_alloc lays it out + the four compose launches */
struct Lat {
  int B = 0, W = 0, maxT = 0;
  long long tn = 0, ta = 0, tl = 0, tc = 0;
  std::vector<GraphMeta> meta;
  std::vector<uint8_t> sg_flags;
  std::vector<int32_t> sg_ptr, sg_src, sg_lab, sg_arc, acc_stage, lnp, lap;
  std::vector<float> sg_w;
  std::vector<uint32_t> alive, rp;
  std::vector<int2> arcs, gi;
};

int build_lattice(
    Lat& L, int B, int T, int C, const float* emissions, const int32_t* lens, const int32_t* n_nodes,
    const uint8_t* flags, const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label, const int32_t* in_arc,
    const float* in_w, const int32_t* n_acc, const int32_t* acc) {
  using namespace gtnb;
  auto& meta = L.meta;
  auto& sg_flags = L.sg_flags;
  auto &sg_ptr = L.sg_ptr, &sg_src = L.sg_src, &sg_lab = L.sg_lab, &sg_arc = L.sg_arc, &acc_stage = L.acc_stage;
  auto& sg_w = L.sg_w;
  meta.assign(B, GraphMeta{});
  long long tn = 0, ta = 0, tl = 0, tc = 0, gg = 0, nb = 0, pb = 0, ab = 0, accb = 0;
  int maxN = 0, maxT = 0;
  for (int b = 0; b < B; b++) {
    const int N = n_nodes[b], A = in_ptr[pb + N], Tb = lens ? lens[b] : T;
    GraphMeta& m = meta[b];
    std::memset(&m, 0, sizeof(m));
    m.sg_node_base = (long long)sg_ptr.size();
    m.sg_arc_base = (long long)sg_src.size();
    int all_valid = 1, uniform = 1;
    for (int n = 0; n <= N; n++) sg_ptr.push_back(in_ptr[pb + n]);
    for (int n = 0; n < N; n++) sg_flags.push_back(flags[nb + n]);
    sg_flags.push_back(0);
    while (sg_ptr.size() % kAlign) sg_ptr.push_back(0), sg_flags.push_back(0);
    for (int a = 0; a < A; a++) {
      sg_src.push_back(in_src[ab + a]);
      sg_lab.push_back(in_label[ab + a]);
      sg_arc.push_back(in_arc[ab + a]);
      sg_w.push_back(in_w[ab + a]);
      all_valid &= in_label[ab + a] >= 0;
    }
    for (int n = 0; n < N; n++)
      for (int a = in_ptr[pb + n]; a < in_ptr[pb + n + 1]; a++) uniform &= in_label[ab + a] == in_label[ab + in_ptr[pb + n]];
    while (sg_src.size() % kAlign || sg_src.empty())
      sg_src.push_back(0), sg_lab.push_back(0), sg_arc.push_back(0), sg_w.push_back(0.0f);
    m.node_base = tn;
    m.arc_base = ta;
    m.lvl_base = tl;
    m.acc_base = tc;
    m.emis_off = (long long)b * T * C;
    m.grad_graph_off = gg;
    gg += A;
    m.L = Tb + 1;
    m.n_accept = n_acc[b];
    m.LB = -1;
    m.T = Tb;
    m.sg_N = N;
    m.sg_A = A;
    m.sg_all_valid = all_valid;
    m.sg_uniform = uniform;
    const long long capN = align_up((long long)(Tb + 1) * N + 1, kAlign), capA = align_up(std::max<long long>((long long)Tb * A, 1), kAlign);
    m.cap_N = (int)capN;
    m.cap_A = (int)capA;
    m.cap_L = (int)align_up(Tb + 2, kAlign);
    tn += capN;
    ta += capA;
    tl += m.cap_L;
    const long long capAcc = align_up(std::max(n_acc[b], 1), kAlign);
    acc_stage.resize(tc + capAcc, 0);
    for (int i = 0; i < n_acc[b]; i++) acc_stage[tc + i] = acc[accb + i];
    tc += capAcc;
    maxN = std::max(maxN, N);
    maxT = std::max(maxT, Tb);
    nb += N;
    pb += N + 1;
    ab += A;
    accb += n_acc[b];
  }
  const int W = (maxN + 31) / 32;
  if (W > kMaxWords) return 1;
  L.alive.assign((size_t)B * (maxT + 1) * W + 16, 0);
  L.rp.assign((size_t)tn + 16, 0);
  L.lnp.assign((size_t)tl + 16, 0);
  L.lap.assign((size_t)tl + 16, 0);
  L.arcs.assign((size_t)ta + 16, int2{0, 0});
  L.gi.assign((size_t)ta + 16, int2{0, 0});
  auto &alive = L.alive, &rp = L.rp;
  auto &lnp = L.lnp, &lap = L.lap;
  auto &arcs = L.arcs, &gi = L.gi;

  emu::launch(B, 256, 0, [&] {
    compose_alive_kernel(meta.data(), sg_flags.data(), sg_ptr.data(), sg_src.data(), sg_lab.data(), alive.data(), W, maxT);
  });
  const int gx = (maxT + 1 + kWarpsPerBlock - 1) / kWarpsPerBlock;
  for (int by = 0; by < B; by++)
    for (int bx = 0; bx < gx; bx++)
      emu::launch(1, 32 * kWarpsPerBlock, 0, [&] {
        blockIdx.x = bx;
        blockIdx.y = by;
        compose_count_kernel(meta.data(), sg_ptr.data(), sg_src.data(), sg_lab.data(), alive.data(), W, maxT,
                             lnp.data(), lap.data());
      });
  emu::launch(B, 1024, 0, [&] {
    compose_scan_kernel(meta.data(), sg_flags.data(), alive.data(), W, maxT, lnp.data(), lap.data(), acc_stage.data());
  });
  for (int by = 0; by < B; by++)
    for (int bx = 0; bx < gx; bx++)
      emu::launch(1, 32 * kWarpsPerBlock, 0, [&] {
        blockIdx.x = bx;
        blockIdx.y = by;
        compose_emit_kernel(meta.data(), sg_flags.data(), sg_ptr.data(), sg_src.data(), sg_lab.data(), sg_arc.data(),
                            sg_w.data(), alive.data(), W, maxT, C, emissions, lnp.data(), lap.data(), rp.data(),
                            arcs.data(), gi.data());
      });

  L.B = B;
  L.W = W;
  L.maxT = maxT;
  L.tn = tn;
  L.ta = ta;
  L.tl = tl;
  L.tc = tc;
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

/* launch_relax_order on a lattice build_lattice made: lattice_relax_order_kernel, then lattice_sort_rows_kernel,
 * which moves arc_grad (nullable) with the arcs */
void relax_order(Lat& L, int B, const int32_t* n_nodes, const int32_t* in_ptr, const int32_t* out_pos,
                 const int32_t* start_rank, int max_out, float* arc_grad) {
  using namespace gtnb;
  // the two extra tables, in the slab layout build_lattice gave the others
  std::vector<int32_t> sg_out_pos(L.sg_src.size(), 0), sg_start_rank(L.sg_ptr.size(), -1);
  long long nb = 0, pb = 0, ab = 0;
  int maxN = 0;
  for (int b = 0; b < B; b++) {
    const int N = n_nodes[b], A = in_ptr[pb + N];
    for (int a = 0; a < A; a++) sg_out_pos[L.meta[b].sg_arc_base + a] = out_pos[ab + a];
    for (int n = 0; n < N; n++) sg_start_rank[L.meta[b].sg_node_base + n] = start_rank[nb + n];
    maxN = std::max(maxN, N);
    nb += N;
    pb += N + 1;
    ab += A;
  }
  std::vector<int32_t> relax((size_t)L.ta + 16, 0);
  // launch_relax_order's shared-memory size: positions / keys + the key bitmaps and their prefix popcounts
  emu::launch(B, kOrderThreads, sizeof(int) * (4 * std::max(maxN, 1) + 4 * ((std::max(maxN, 1) * (max_out + 1) + 31) / 32)), [&] {
    lattice_relax_order_kernel(L.meta.data(), L.sg_flags.data(), L.sg_ptr.data(), L.sg_src.data(), L.sg_lab.data(),
                               sg_out_pos.data(), sg_start_rank.data(), L.alive.data(), L.W, L.maxT, max_out + 1,
                               L.lnp.data(), L.rp.data(), relax.data(), L.acc_stage.data());
  });
  {
    int capN = 1;
    for (int b = 0; b < B; b++) capN = std::max(capN, L.meta[b].cap_N);
    const int ggx = std::min((capN + 255) / 256, 4096);
    for (int by = 0; by < B; by++)
      for (int bx = 0; bx < ggx; bx++)
        emu::launch(1, 256, 0, [&] {
          blockIdx.x = bx;
          blockIdx.y = by;
          gridDim.x = ggx;
          lattice_sort_rows_kernel(L.meta.data(), L.rp.data(), relax.data(), L.arcs.data(), L.gi.data(), arc_grad);
        });
  }
}

} // namespace

extern "C" {

/*
 * compose(g_b, linearGraph(T_b, C) with the given emissions) for B graphs given as concatenated
 * CSR-by-destination tables (n_nodes[B], in_ptr with N_b + 1 entries per graph, offsets local):
 * flags bit 0 start / bit 1 accept, in_src / in_label (-1: cannot match) / in_arc (Graph arc id) / in_w,
 * accept lists acc (n_acc[B]).  Outputs per graph b (capacities (T+1) N_b + 1 nodes, T A_b arcs,
 * concatenated at node_off[b] / arc_off[b] which the caller computes the same way):
 *   out_N[b], out_A[b], row_ptr, arc_src, arc_w, gi_graph, gi_emis, lvl_node_ptr (T_b + 2 per graph at
 *   lvl_off[b]), accept nodes of the lattice (acc_out, n_acc_out[b]).
 * arc_grad (nullable, indexed like the arcs): if given, compose's gradFunc is run into grad_graph
 * (A_b per graph, concatenated) and grad_emis [B][T][C] (both zero on entry).
 */
int emu_compose(
    int B, int T, int C, const float* emissions, const int32_t* lens, const int32_t* n_nodes, const uint8_t* flags,
    const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label, const int32_t* in_arc, const float* in_w,
    const int32_t* n_acc, const int32_t* acc, int32_t* out_N, int32_t* out_A, uint32_t* row_ptr, int32_t* arc_src,
    float* arc_w, int32_t* gi_graph, int32_t* gi_emis, int32_t* lvl_node_ptr, int32_t* acc_out, int32_t* n_acc_out,
    const float* arc_grad, float* grad_graph, float* grad_emis) {
  using namespace gtnb;
  Lat L;
  if (int rc = build_lattice(L, B, T, C, emissions, lens, n_nodes, flags, in_ptr, in_src, in_label, in_arc, in_w, n_acc, acc))
    return rc;
  auto& meta = L.meta;
  auto &rp = L.rp;
  auto &lnp = L.lnp, &acc_stage = L.acc_stage;
  auto &arcs = L.arcs, &gi = L.gi;
  const long long ta = L.ta;
  // hand the lattices back, graph by graph, in the caller's (unaligned) capacities
  long long no = 0, ao = 0, lo = 0, co = 0;
  for (int b = 0; b < B; b++) {
    const GraphMeta& m = meta[b];
    out_N[b] = m.N;
    out_A[b] = m.A;
    for (int n = 0; n <= m.N; n++) row_ptr[no + n] = rp[m.node_base + n];
    for (int a = 0; a < m.A; a++) {
      arc_src[ao + a] = arcs[m.arc_base + a].x;
      arc_w[ao + a] = __int_as_float(arcs[m.arc_base + a].y);
      gi_graph[ao + a] = gi[m.arc_base + a].x;
      gi_emis[ao + a] = gi[m.arc_base + a].y;
    }
    for (int l = 0; l <= m.T + 1; l++) lvl_node_ptr[lo + l] = lnp[m.lvl_base + l];
    n_acc_out[b] = m.n_accept;
    for (int i = 0; i < m.n_accept; i++) acc_out[co + i] = acc_stage[m.acc_base + i];
    no += (long long)(m.T + 1) * m.sg_N + 1;
    ao += std::max<long long>((long long)m.T * m.sg_A, 1);
    lo += m.T + 2;
    co += n_acc[b];
  }
  if (arc_grad) {
    std::vector<float> ag((size_t)ta + 16, 0.0f);
    long long src_off = 0;
    for (int b = 0; b < B; b++) {
      for (int a = 0; a < meta[b].A; a++) ag[meta[b].arc_base + a] = arc_grad[src_off + a];
      src_off += std::max<long long>((long long)meta[b].T * meta[b].sg_A, 1);
    }
    int capN = 1;
    for (int b = 0; b < B; b++) capN = std::max(capN, meta[b].cap_N);
    const int ggx = std::min((capN + 255) / 256, 4096);
    for (int by = 0; by < B; by++)
      for (int bx = 0; bx < ggx; bx++)
        emu::launch(1, 256, 0, [&] {
          blockIdx.x = bx;
          blockIdx.y = by;
          gridDim.x = ggx;
          compose_grad_kernel(meta.data(), rp.data(), ag.data(), gi.data(), grad_graph, grad_emis, (long long)T * C);
        });
  }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

/*
 * The materialised criterion path end to end, as gtnb_ctc_loss runs it with the "implicit" and
 * "staged" flags off: compose -> sd_forward_generic (log semiring) -> sd_backward_generic (deltas)
 * -> compose's gradFunc.  Graph tables as in emu_compose.  out_scores[B] = forwardScore of the
 * lattice; grad_emis [B][T][C] (zero on entry) receives deltas[b] * d score / d emissions; grad_graph
 * likewise per graph arc.  With viterbi != 0 additionally: viterbiScore into vit_scores[B] and the best
 * path's emission labels into vit_labels [B][T] (MODE_PATH forward + traceback + gather_prov).
 */
int emu_materialised(
    int B, int T, int C, const float* emissions, const int32_t* lens, const int32_t* n_nodes, const uint8_t* flags,
    const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label, const int32_t* in_arc, const float* in_w,
    const int32_t* n_acc, const int32_t* acc, const float* deltas, float* out_scores, float* grad_graph,
    float* grad_emis, int viterbi, float* vit_scores, int32_t* vit_labels) {
  using namespace gtnb;
  Lat L;
  if (int rc = build_lattice(L, B, T, C, emissions, lens, n_nodes, flags, in_ptr, in_src, in_label, in_arc, in_w, n_acc, acc))
    return rc;
  std::vector<float> scores((size_t)L.tn + 16, 0.0f), node_grad((size_t)L.tn + 16, 0.0f), arc_grad((size_t)L.ta + 16, 0.0f);
  std::vector<int32_t> back_ptr((size_t)L.tn + 16, -1), best(B, -1);
  emu::launch(B, kThreads, 0, [&] {
    sd_forward_generic<MODE_LOG>(L.meta.data(), L.lnp.data(), L.rp.data(), L.arcs.data(), nullptr, L.acc_stage.data(),
                                 scores.data(), back_ptr.data(), out_scores, best.data());
  });
  emu::launch(B, kThreads, 0, [&] {
    sd_backward_generic<false>(L.meta.data(), L.lnp.data(), nullptr, nullptr, L.rp.data(), L.arcs.data(),
                               L.acc_stage.data(), scores.data(), out_scores, best.data(), deltas, node_grad.data(),
                               arc_grad.data());
  });
  int capN = 1;
  for (int b = 0; b < B; b++) capN = std::max(capN, L.meta[b].cap_N);
  const int ggx = std::min((capN + 255) / 256, 4096);
  for (int by = 0; by < B; by++)
    for (int bx = 0; bx < ggx; bx++)
      emu::launch(1, 256, 0, [&] {
        blockIdx.x = bx;
        blockIdx.y = by;
        gridDim.x = ggx;
        compose_grad_kernel(L.meta.data(), L.rp.data(), arc_grad.data(), L.gi.data(), grad_graph, grad_emis,
                            (long long)T * C);
      });
  if (viterbi) {
    emu::launch(B, kThreads, 0, [&] {
      sd_forward_generic<MODE_PATH>(L.meta.data(), L.lnp.data(), L.rp.data(), L.arcs.data(), nullptr, L.acc_stage.data(),
                                    scores.data(), back_ptr.data(), vit_scores, best.data());
    });
    std::vector<int32_t> path((size_t)B * std::max(T, 1), -1), plen(B, 0), pg((size_t)B * std::max(T, 1), -1),
        pl((size_t)B * std::max(T, 1), -1);
    emu::launch((B + 63) / 64, 64, 0, [&] {
      traceback_kernel(L.meta.data(), L.arcs.data(), back_ptr.data(), best.data(), B, T, path.data(), plen.data());
    });
    if (T > 0)
      for (int by = 0; by < B; by++)
        for (int bx = 0; bx < (T + 127) / 128; bx++)
          emu::launch(1, 128, 0, [&] {
            blockIdx.x = bx;
            blockIdx.y = by;
            gather_prov_kernel(L.meta.data(), L.gi.data(), L.arcs.data(), T, path.data(), plen.data(), pg.data(),
                               pl.data(), nullptr);
          });
    for (int b = 0; b < B; b++)
      for (int t = 0; t < T; t++) {
        const int32_t j = t < plen[b] ? pl[(size_t)b * T + t] : -1; // arc of the emissions chain: frame * C + label
        vit_labels[(size_t)b * T + t] = j >= 0 ? j % C : -1;
      }
  }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

/*
 * viterbiPath through the materialised lattice put in the reference's tie-breaking order (k_order.cu, the
 * "exact_ties" option): compose -> lattice_relax_order_kernel -> lattice_sort_rows_kernel -> the MODE_PATH
 * sweep (staged != 0: sd_forward_staged of k_staged.cu, else sd_forward_generic) -> traceback -> label
 * provenance.  out_pos: per in-entry, the position of the arc in its source's out-arc list; start_rank: per
 * node, its index in g.start() or -1 (concatenated like flags).
 */
int emu_viterbi_exact(
    int B, int T, int C, const float* emissions, const int32_t* lens, const int32_t* n_nodes, const uint8_t* flags,
    const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label, const int32_t* in_arc, const float* in_w,
    const int32_t* out_pos, const int32_t* start_rank, int max_out, const int32_t* n_acc, const int32_t* acc,
    int staged, float* vit_scores, int32_t* vit_labels, int32_t* vit_graph_arcs) {
  using namespace gtnb;
  Lat L;
  if (int rc = build_lattice(L, B, T, C, emissions, lens, n_nodes, flags, in_ptr, in_src, in_label, in_arc, in_w, n_acc, acc))
    return rc;
  relax_order(L, B, n_nodes, in_ptr, out_pos, start_rank, max_out, nullptr);
  std::vector<float> scores((size_t)L.tn + 16, 0.0f);
  std::vector<int32_t> back_ptr((size_t)L.tn + 16, -1), best(B, -1);
  if (staged) {
    int max_L = 0, mN = 0, mA = 0;
    for (int b = 0; b < B; b++) {
      max_L = std::max(max_L, L.meta[b].L);
      mN = std::max(mN, L.meta[b].sg_N);
      mA = std::max(mA, L.meta[b].sg_A);
    }
    const Layout lf = make_layout(mN, mA, max_L, 1, 2, false);
    emu::launch(B, 32 * consumer_warps(1) + 32, lf.total, [&] {
      sd_forward_staged<MODE_PATH, 1>(L.meta.data(), L.lnp.data(), L.lap.data(), L.rp.data(), L.arcs.data(),
                                      L.acc_stage.data(), scores.data(), back_ptr.data(), vit_scores, best.data(), lf);
    });
  } else {
    emu::launch(B, kThreads, 0, [&] {
      sd_forward_generic<MODE_PATH>(L.meta.data(), L.lnp.data(), L.rp.data(), L.arcs.data(), nullptr,
                                    L.acc_stage.data(), scores.data(), back_ptr.data(), vit_scores, best.data());
    });
  }
  std::vector<int32_t> path((size_t)B * std::max(T, 1), -1), plen(B, 0), pg((size_t)B * std::max(T, 1), -1),
      pl((size_t)B * std::max(T, 1), -1);
  emu::launch((B + 63) / 64, 64, 0, [&] {
    traceback_kernel(L.meta.data(), L.arcs.data(), back_ptr.data(), best.data(), B, T, path.data(), plen.data());
  });
  if (T > 0)
    for (int by = 0; by < B; by++)
      for (int bx = 0; bx < (T + 127) / 128; bx++)
        emu::launch(1, 128, 0, [&] {
          blockIdx.x = bx;
          blockIdx.y = by;
          gather_prov_kernel(L.meta.data(), L.gi.data(), L.arcs.data(), T, path.data(), plen.data(), pg.data(),
                             pl.data(), nullptr);
        });
  for (int b = 0; b < B; b++)
    for (int t = 0; t < T; t++) {
      const bool on = t < plen[b];
      vit_labels[(size_t)b * T + t] = on ? pl[(size_t)b * T + t] % C : -1;
      vit_graph_arcs[(size_t)b * T + t] = on ? pg[(size_t)b * T + t] : -1;
    }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

/*
 * The exact-ties row sort on a lattice whose arc gradients a backward pass wrote before it (gtnb_backward may run
 * before the sort): compose -> arc_grad = grad_in -> lattice_relax_order_kernel -> lattice_sort_rows_kernel.
 * Tables as in emu_viterbi_exact.  grad_in, grad_out, gi_in and gi_out hold the arcs graph after graph, n_arcs[b]
 * (out) of them each: grad_in in compose order, grad_out the sorted arc_grad, gi_in / gi_out every arc's provenance
 * {graph arc, emissions arc} before / after the sort.
 */
int emu_sort_rows_with_grads(
    int B, int T, int C, const float* emissions, const int32_t* lens, const int32_t* n_nodes, const uint8_t* flags,
    const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label, const int32_t* in_arc, const float* in_w,
    const int32_t* out_pos, const int32_t* start_rank, int max_out, const int32_t* n_acc, const int32_t* acc,
    const float* grad_in, float* grad_out, int32_t* gi_in, int32_t* gi_out, int32_t* n_arcs) {
  using namespace gtnb;
  Lat L;
  if (int rc = build_lattice(L, B, T, C, emissions, lens, n_nodes, flags, in_ptr, in_src, in_label, in_arc, in_w, n_acc, acc))
    return rc;
  std::vector<float> arc_grad(L.arcs.size(), 0.0f);
  long long off = 0;
  for (int b = 0; b < B; b++) {
    n_arcs[b] = L.meta[b].A;
    for (int a = 0; a < L.meta[b].A; a++) {
      const long long k = off + a, d = L.meta[b].arc_base + a;
      arc_grad[d] = grad_in[k];
      gi_in[2 * k] = L.gi[d].x;
      gi_in[2 * k + 1] = L.gi[d].y;
    }
    off += L.meta[b].A;
  }
  relax_order(L, B, n_nodes, in_ptr, out_pos, start_rank, max_out, arc_grad.data());
  off = 0;
  for (int b = 0; b < B; b++) {
    for (int a = 0; a < L.meta[b].A; a++) {
      const long long k = off + a, d = L.meta[b].arc_base + a;
      grad_out[k] = arc_grad[d];
      gi_out[2 * k] = L.gi[d].x;
      gi_out[2 * k + 1] = L.gi[d].y;
    }
    off += L.meta[b].A;
  }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

/*
 * The materialised criterion path through the TMA-staged persistent kernels (k_staged.cu; G = 1, the
 * CTC-degree family): compose -> sd_forward_staged -> either sd_backward_staged + compose's gradFunc
 * (fused == 0) or sd_backward_fused (fused != 0).  cp.async.bulk / mbarrier are emulated (simt_emu.h).
 * Tables as in emu_compose; out_scores[B]; grad_emis [B][T][C] zero on entry; viterbi != 0 additionally
 * runs the MODE_PATH sweep + traceback (labels into vit_labels [B][T], scores into vit_scores).
 * Returns 0, or 3 when k_staged.cu's plan is not G = 1 (mean degree > 4), does not fit, or refuses the fused layout.
 */
int emu_materialised_staged(
    int B, int T, int C, const float* emissions, const int32_t* lens, const int32_t* n_nodes, const uint8_t* flags,
    const int32_t* in_ptr, const int32_t* in_src, const int32_t* in_label, const int32_t* in_arc, const float* in_w,
    const int32_t* n_acc, const int32_t* acc, const float* deltas, int fused, float* out_scores, float* grad_emis,
    int viterbi, float* vit_scores, int32_t* vit_labels) {
  using namespace gtnb;
  Lat L;
  if (int rc = build_lattice(L, B, T, C, emissions, lens, n_nodes, flags, in_ptr, in_src, in_label, in_arc, in_w, n_acc, acc))
    return rc;
  int maxN = 0, maxA = 0;
  for (int b = 0; b < B; b++) {
    maxN = std::max(maxN, L.meta[b].sg_N);
    maxA = std::max(maxA, L.meta[b].sg_A);
  }
  const StagedPlan p = plan(L.meta.data(), B, maxN, maxA);
  if (!p.ok || p.G != 1) return 3;
  const Layout &lf = p.fwd, &lb = p.bwd;
  Layout lay = lb; // sd_backward_fused's
  if (fused && !fused_layout(lay, maxN, maxA)) return 3;
  constexpr int kT = 32 * consumer_warps(1) + 32;
  std::vector<float> scores((size_t)L.tn + 16, 0.0f), arc_grad((size_t)L.ta + 16, 0.0f);
  std::vector<int32_t> back_ptr((size_t)L.tn + 16, -1), best(B, -1);
  emu::launch(B, kT, lf.total, [&] {
    sd_forward_staged_kernel_for(MODE_LOG, p.G)(L.meta.data(), L.lnp.data(), L.lap.data(), L.rp.data(),
                                                L.arcs.data(), L.acc_stage.data(), scores.data(), back_ptr.data(),
                                                out_scores, best.data(), lf);
  });
  if (fused) {
    emu::launch(B, kT, lay.total, [&] {
      sd_backward_fused(L.meta.data(), L.lnp.data(), L.lap.data(), L.rp.data(), L.arcs.data(), L.gi.data(),
                        L.acc_stage.data(), scores.data(), out_scores, deltas, L.sg_ptr.data(), L.sg_src.data(),
                        L.sg_lab.data(), grad_emis, (long long)T * C, C, lay);
    });
  } else {
    emu::launch(B, kT, lb.total, [&] {
      sd_backward_staged_kernel_for(false, p.G)(L.meta.data(), L.lnp.data(), L.lap.data(), L.rp.data(),
                                                L.arcs.data(), L.acc_stage.data(), scores.data(), out_scores,
                                                best.data(), deltas, arc_grad.data(), lb);
    });
    int capN = 1;
    for (int b = 0; b < B; b++) capN = std::max(capN, L.meta[b].cap_N);
    const int ggx = std::min((capN + 255) / 256, 4096);
    for (int by = 0; by < B; by++)
      for (int bx = 0; bx < ggx; bx++)
        emu::launch(1, 256, 0, [&] {
          blockIdx.x = bx;
          blockIdx.y = by;
          gridDim.x = ggx;
          compose_grad_kernel(L.meta.data(), L.rp.data(), arc_grad.data(), L.gi.data(), nullptr, grad_emis,
                              (long long)T * C);
        });
  }
  if (viterbi) {
    emu::launch(B, kT, lf.total, [&] {
      sd_forward_staged_kernel_for(MODE_PATH, p.G)(L.meta.data(), L.lnp.data(), L.lap.data(), L.rp.data(),
                                                   L.arcs.data(), L.acc_stage.data(), scores.data(), back_ptr.data(),
                                                   vit_scores, best.data(), lf);
    });
    std::vector<int32_t> path((size_t)B * std::max(T, 1), -1), plen(B, 0), pg((size_t)B * std::max(T, 1), -1),
        pl((size_t)B * std::max(T, 1), -1);
    emu::launch((B + 63) / 64, 64, 0, [&] {
      traceback_kernel(L.meta.data(), L.arcs.data(), back_ptr.data(), best.data(), B, T, path.data(), plen.data());
    });
    if (T > 0)
      for (int by = 0; by < B; by++)
        for (int bx = 0; bx < (T + 127) / 128; bx++)
          emu::launch(1, 128, 0, [&] {
            blockIdx.x = bx;
            blockIdx.y = by;
            gather_prov_kernel(L.meta.data(), L.gi.data(), L.arcs.data(), T, path.data(), plen.data(), pg.data(),
                               pl.data(), nullptr);
          });
    for (int b = 0; b < B; b++)
      for (int t = 0; t < T; t++) vit_labels[(size_t)b * T + t] = t < plen[b] ? pl[(size_t)b * T + t] % C : -1;
  }
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads; // the host refused the threads
  return 0;
}

} // extern "C"
