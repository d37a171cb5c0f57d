/*
 * tests/emu/decode_async_emu.cpp -- TEST INFRASTRUCTURE for gtnb_viterbi_transitions_async and
 * gtnb_viterbi_dense_async: the SOURCE of k_ctc.cu's decode_async_prepare_kernel and decode_async_finalize_kernel, alone
 * and around k_sparse.cu's tropical sweep and trace (one CTA per utterance) over G's tables from the shipped builder
 * (gtnb_product.h), run on the CPU through tests/emu/simt_emu.h.  Only the launch geometry and the packing of the
 * tables into SparseDev are restated here.
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_ctc.cu"
#include "../../gtn_b200/csrc/k_sparse.cu"
#include "../../gtn_b200/csrc/gtnb_product.h"

#include <vector>

extern "C" {

/* decode_async_prepare_kernel as launch_decode_async_prepare launches it; input_lens nullable */
int emu_decode_prepare(int B, int T, const int32_t* input_lens, int32_t* lens, int32_t* valid, int32_t* kstatus) {
  using namespace gtnb;
  emu::launch((B + 255) / 256, 256, 0, [&] { decode_async_prepare_kernel(B, T, input_lens, lens, valid, kstatus); });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

/* decode_async_finalize_kernel as launch_decode_async_finalize launches it; paths, arcs, status nullable */
int emu_decode_finalize(int B, int T, const int32_t* lens, const int32_t* kstatus, const int32_t* valid,
                        int32_t* paths, int32_t* arcs, float* scores, int32_t* status) {
  using namespace gtnb;
  emu::launch(B, 256, 0, [&] {
    decode_async_finalize_kernel(T, lens, kstatus, valid, paths, arcs, scores, status);
  });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

/*
 * The device route of gtnb_viterbi_transitions_async for an epsilon-free G inside the one-CTA envelope: prepare, the
 * tropical sweep and trace, finalize.  emissions [B][T][C]; input_lens nullable; G (S nodes, nG arcs), w [nG].  Out:
 * paths, arcs [B][T], scores [B], status [B].  Returns 0, 1 outside the envelope, 77 when the host refused the threads.
 */
int emu_decode_route(int B, int T, int C, const float* emissions, const int32_t* input_lens, int S, int nG,
                     const uint8_t* g_flags, const int32_t* g_src, const int32_t* g_dst, const int32_t* g_label,
                     const float* w, int32_t* paths, int32_t* arcs, float* scores, int32_t* status) {
  using namespace gtnb;
  gtnb_graph_view G{};
  G.num_nodes = S;
  G.num_arcs = nG;
  G.node_flags = g_flags;
  G.arc_src = g_src;
  G.arc_dst = g_dst;
  G.arc_ilabel = G.arc_olabel = g_label;
  SparseTables t;
  sparse_tables(G, C, &t);
  if (S < 1 || S > kSparseMaxStates || t.A > kSparseMaxArcs || C > kSparseMaxLabels) return 1;
  std::vector<int32_t> flags(t.flags.begin(), t.flags.end());
  const SparseDev dev{t.S, t.A, sparse_den_lanes(t.S, t.A), flags.data(), t.in_ptr.data(), t.in_src.data(),
                      t.in_lab.data(), t.in_arc.data(), t.out_ptr.data(), t.out_dst.data(), t.out_lab.data(),
                      t.out_arc.data()};
  std::vector<int32_t> lens(B + 1), valid(B + 1), kstatus(B + 1), head(B + 1);
  std::vector<uint16_t> bp((size_t)B * T * S + 1, 0);
  emu::launch((B + 255) / 256, 256, 0, [&] {
    decode_async_prepare_kernel(B, T, input_lens, lens.data(), valid.data(), kstatus.data());
  });
  emu::launch(B, kSparseThreads, sizeof(float) * sparse_vit_smem_floats(S, C), [&] {
    sparse_viterbi_forward_kernel(dev, T, C, lens.data(), emissions, (long long)T * C, w, bp.data(), head.data(),
                                  scores, kstatus.data());
  });
  emu::launch((B * 32 + 255) / 256, 256, 0, [&] {
    sparse_viterbi_trace_kernel(dev, B, T, lens.data(), bp.data(), head.data(), paths, arcs, kstatus.data());
  });
  emu::launch(B, 256, 0, [&] {
    decode_async_finalize_kernel(T, lens.data(), kstatus.data(), valid.data(), paths, arcs, scores, status);
  });
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

} // extern "C"
