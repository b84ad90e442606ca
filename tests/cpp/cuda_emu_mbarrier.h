// TEST INFRASTRUCTURE (CPU tier): mbarrier and st.async into a peer block's shared memory, as the push exchange of the pose LM
// uses them (csrc/ba.cu includes this header when it is compiled by the host compiler, after tests/cpp/cuda_emu.h, whose
// cluster emulation runs the blocks of a cluster at the same time).
//
// The barrier's 64-bit word of shared memory packs what the hardware keeps: bit 63 the phase, bits 48..62 the expected
// arrivals, bits 32..47 the pending arrivals, bits 0..31 the signed transaction count (bytes may land before the barrier is
// armed for the phase, so it can go negative).  A phase completes when both counts reach zero.
#pragma once
#include <stdint.h>
#include <thread>

static inline void emu_mbar_init(unsigned long long *bar, unsigned count) {
  __atomic_store_n(bar, ((unsigned long long)count << 48) | ((unsigned long long)count << 32), __ATOMIC_SEQ_CST);
}

// adds `tx` to the transaction count (negative: bytes that landed) and takes `arrivals` off the pending arrivals
static inline void emu_mbar_update(unsigned long long *bar, int tx, unsigned arrivals) {
  unsigned long long old = __atomic_load_n(bar, __ATOMIC_SEQ_CST), next;
  do {
    const unsigned long long phase = old >> 63, expected = (old >> 48) & 0x7FFF;
    const unsigned long long pending = ((old >> 32) & 0xFFFF) - arrivals;
    const int32_t cnt = (int32_t)(uint32_t)old + tx;
    if (pending == 0 && cnt == 0) next = ((phase ^ 1) << 63) | (expected << 48) | (expected << 32);
    else next = (phase << 63) | (expected << 48) | ((pending & 0xFFFF) << 32) | (uint32_t)cnt;
  } while (!__atomic_compare_exchange_n(bar, &old, next, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST));
}

// mbarrier.arrive.expect_tx: one arrival, `bytes` more to receive in the current phase
static inline void emu_mbar_arrive_expect_tx(unsigned long long *bar, unsigned bytes) { emu_mbar_update(bar, (int)bytes, 1); }

// mbarrier.try_wait.parity: true once the phase of that parity has completed
static inline bool emu_mbar_try_wait_parity(unsigned long long *bar, unsigned parity) {
  if ((unsigned)(__atomic_load_n(bar, __ATOMIC_SEQ_CST) >> 63) != parity) return true;
  std::this_thread::yield();
  return false;
}

// st.async.shared::cluster.mbarrier::complete_tx::bytes: v to block `rank`'s copy of *dst, counted on that block's copy of *bar
template <class T> static inline void emu_st_async(T *dst, T v, unsigned long long *bar, unsigned rank) {
  const cooperative_groups::cluster_group cl;
  *cl.map_shared_rank(dst, rank) = v;                              // published by the sequentially consistent update below
  emu_mbar_update(cl.map_shared_rank(bar, rank), -(int)sizeof(T), 0);
}
