/*
 * tests/emu/backoff_align_emu.cpp -- TEST INFRASTRUCTURE for gtnb_backoff_transitions_viterbi: the SOURCE of
 * k_sparse.cu's alignment kernels (sparse_eps_align_kernel, sparse_eps_align_trace_kernel) run on the CPU through
 * tests/emu/simt_emu.h, over per-utterance numerators packed as backoff_align_run packs them.  The packing of the
 * tables into SparseEpsDev is backoff_emu.cpp's HostEps.
 */
#include "backoff_emu.cpp"

extern "C" {

/*
 * The alignment's device route after the gather: graph b (S[b] nodes, nA[b] arcs, labels -1: epsilon arcs, arrays
 * concatenated in utterance order) for utterance b, its back-pointers at the sum of (T_b' + 1) * S_b' over the
 * utterances before it; w: the gathered weights of all arcs in that order; arc_of: the A arc of every product arc in
 * the batch's numbering, a_first [B] every utterance's first A arc.  Out: paths, arcs [B][T], scores [B], status [B]
 * (zeroed here).  Returns 0, 1 outside the envelope, 77 when the host refused the threads.
 */
int emu_backoff_align(int B, int T, int C, const float* emissions, const int32_t* lens, const int32_t* S,
                      const int32_t* nA, const uint8_t* flags, const int32_t* src, const int32_t* dst,
                      const int32_t* label, const float* w, const int32_t* arc_of, const int32_t* a_first,
                      int32_t* paths, int32_t* arcs, float* scores, int32_t* status) {
  using namespace gtnb;
  HostEps h;
  std::vector<SparseEpsDev> desc;
  long long rows = 0, node0 = 0, arc0 = 0;
  int max_S = 1;
  for (int b = 0; b < B; b++) {
    const gtnb_graph_view v = view_of(S[b], nA[b], flags + node0, src + arc0, dst + arc0, label + arc0, nullptr);
    const SparseTables t = eps_tables_of(v, C);
    if (!t.cycle.empty() || !sparse_eps_supported(t.S, t.A, t.E, t.L, t.max_in_all, C)) return 1;
    desc.push_back(h.add(t, (int32_t)arc0, rows, 0));
    rows += (long long)(lens[b] + 1) * S[b];
    max_S = std::max(max_S, t.S);
    node0 += S[b];
    arc0 += nA[b];
  }
  std::vector<uint16_t> bp((size_t)rows + 1, 0);
  std::vector<int32_t> head(B + 1, 0);
  for (int b = 0; b < B; b++) status[b] = 0;
  emu::launch(B, kSparseThreads, sizeof(float) * sparse_vit_smem_floats(max_S, C), [&] {
    sparse_eps_align_kernel(desc.data(), C, lens, emissions, (long long)T * C, w, bp.data(), head.data(), scores,
                            status);
  });
  emu::launch((B * 32 + 255) / 256, 256, 0, [&] {
    sparse_eps_align_trace_kernel(desc.data(), B, T, lens, bp.data(), head.data(), arc_of, a_first, paths, arcs,
                                  status);
  });
  if (emu::g_launch_failed.exchange(false)) return emu::kEmuNoThreads;
  return 0;
}

} // extern "C"
