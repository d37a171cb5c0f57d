/*
 * tests/emu/edit_emu.cpp -- TEST INFRASTRUCTURE for gtnb_edit_distance_async: the SOURCE of k_edit.cu's
 * edit_distance_kernel run on the CPU through tests/emu/simt_emu.h, at the launch geometry of launch_edit_distance or
 * at a forced strip height K and warp count, with the shipped word hash or a degenerate one that makes every word
 * pair collide (so the exact span compare decides every word id).
 */
#define GTNB_HOST_EMU 1
#include "../../gtn_b200/csrc/k_edit.cu"

#include <vector>

namespace {

/* every word hashes to 0: equality rests on the exact compare alone */
struct CollideHash {
  static uint64_t combine(uint64_t, int32_t) { return 0; }
};

template <int K, class H>
void run(const gtnb::EditPlan& p, int warps, int B, const int32_t* hyp, int N, const int32_t* hyp_lens,
         const int32_t* ref, int M, const int32_t* ref_lens, int word_sep, int32_t* distance, int32_t* ops,
         int32_t* units, int32_t* status, int32_t* hyp_align, int32_t* ref_align, uint32_t* moves) {
  emu::launch(B, 32 * warps, p.smem_bytes, [&] {
    gtnb::edit_distance_kernel<K, H>(hyp, N, hyp_lens, ref, M, ref_lens, word_sep, p.cols, distance, ops, units,
                                     status, hyp_align, ref_align, moves);
  });
}

template <class H>
int dispatch(int K, const gtnb::EditPlan& p, int warps, int B, const int32_t* hyp, int N, const int32_t* hyp_lens,
             const int32_t* ref, int M, const int32_t* ref_lens, int word_sep, int32_t* distance, int32_t* ops,
             int32_t* units, int32_t* status, int32_t* hyp_align, int32_t* ref_align, uint32_t* moves) {
#define GTNB_EDIT_EMU(K_)                                                                                    \
  case K_:                                                                                                   \
    run<K_, H>(p, warps, B, hyp, N, hyp_lens, ref, M, ref_lens, word_sep, distance, ops, units, status,     \
               hyp_align, ref_align, moves);                                                                 \
    return 0;
  switch (K) {
    GTNB_EDIT_EMU(1)
    GTNB_EDIT_EMU(2)
    GTNB_EDIT_EMU(4)
    GTNB_EDIT_EMU(8)
    GTNB_EDIT_EMU(16)
  }
#undef GTNB_EDIT_EMU
  return 1;
}

} // namespace

extern "C" {

/* the plan launch_edit_distance takes for these bounds: K, warps, cols */
void emu_edit_plan(int N, int M, int word_sep, int* out) {
  const gtnb::EditPlan p = gtnb::edit_plan(N, M, word_sep);
  out[0] = p.K;
  out[1] = p.warps;
  out[2] = p.cols;
}

/*
 * One launch.  K = 0: the plan's K and warps, else those forced (1 when they cannot hold the rows bound or K is not a
 * bucket).  collide: the degenerate hash.  with_alignment: the move scratch is given (hyp_align / ref_align each
 * nullable).  Returns 0, 1 for a bad forced geometry, 77 when the host refused the threads.
 */
int emu_edit(int B, const int32_t* hyp, int N, const int32_t* hyp_lens, const int32_t* ref, int M,
             const int32_t* ref_lens, int word_sep, int K, int warps, int collide, int with_alignment,
             int32_t* distance, int32_t* ops, int32_t* units, int32_t* status, int32_t* hyp_align,
             int32_t* ref_align) {
  gtnb::EditPlan p = gtnb::edit_plan(N, M, word_sep);
  if (K == 0) {
    K = p.K;
    warps = p.warps;
  }
  const int un = word_sep >= 0 ? (N + 1) / 2 : N, um = word_sep >= 0 ? (M + 1) / 2 : M;
  if (warps < 1 || warps > gtnb::kEditMaxWarps || 32 * K * warps < (un < um ? un : um)) return 1;
  std::vector<uint32_t> moves(with_alignment ? (size_t)B * warps * (p.cols + 31) * 32 : 0, 0xdeadbeefu);
  const int rc = collide ? dispatch<CollideHash>(K, p, warps, B, hyp, N, hyp_lens, ref, M, ref_lens, word_sep,
                                                 distance, ops, units, status, hyp_align, ref_align,
                                                 with_alignment ? moves.data() : nullptr)
                         : dispatch<gtnb::EditHash>(K, p, warps, B, hyp, N, hyp_lens, ref, M, ref_lens, word_sep,
                                                    distance, ops, units, status, hyp_align, ref_align,
                                                    with_alignment ? moves.data() : nullptr);
  if (rc) return rc;
  return emu::g_launch_failed.exchange(false) ? emu::kEmuNoThreads : 0;
}

} // extern "C"
