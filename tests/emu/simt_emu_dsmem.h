/*
 * tests/emu/simt_emu_dsmem.h -- TEST INFRASTRUCTURE: distributed shared memory for the SIMT emulator of simt_emu.h
 * (mapa + st.shared::cluster: a store into the shared memory of a peer CTA of the cluster).  The emulator's clusters
 * do not know their CTAs, so a launch that uses remote stores goes through launch_clusters_dsmem: every thread files
 * its CTA under (cluster, rank) before it runs the kernel, and a remote store looks the peer up there.  The kernel's
 * first barrier.cluster, which it needs on the device too before it touches a peer, orders the filing of every CTA
 * before any lookup.
 */
#pragma once

#include "simt_emu.h"

namespace emu {

constexpr unsigned kMaxClusterSize = 16;
struct PeerTable {
  std::mutex lock;
  std::map<Cluster*, std::array<Cta*, kMaxClusterSize>> ctas; // (a map's values stay where they are)
};
inline PeerTable g_peers;
inline thread_local std::array<Cta*, kMaxClusterSize>* g_my_peers = nullptr;

/* launch_clusters for a kernel that stores into its peers' shared memory */
template <class F>
void launch_clusters_dsmem(unsigned grid, unsigned csize, unsigned block, size_t smem_bytes, F&& body) {
  launch_clusters(grid, csize, block, smem_bytes, [&] {
    {
      std::lock_guard<std::mutex> l(g_peers.lock);
      g_my_peers = &g_peers.ctas[g_cluster];
      (*g_my_peers)[g_cluster_rank] = g_cta;
    }
    body();
  });
}

/* the shared-window address addr of this CTA in the CTA of cluster rank `rank` */
template <class T>
T* cluster_shared_ptr(uint32_t addr, unsigned rank) {
  return reinterpret_cast<T*>(reinterpret_cast<unsigned char*>((*g_my_peers)[rank]->dynamic_smem()) +
                              (addr - kWindowBias));
}

} // namespace emu
