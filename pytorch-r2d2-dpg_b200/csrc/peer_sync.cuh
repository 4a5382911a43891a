#pragma once
// Flag primitives of the peer-memory exchanges (peer.cu: gradients, global_replay.cu: global replay sampling): release
// stores of an iteration-numbered flag into a peer's buffer, acquire loads on the waiting side, every wait bounded.
#include "common.cuh"

namespace r2d2 {

constexpr unsigned long long kSpinLimitNs = 4000000000ull;

__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// epochs only grow; a peer is at most one ahead.  An expired wait sets *status = 1 and returns.
__device__ __forceinline__ void spin_until(const unsigned* flag, unsigned value, unsigned* status) {
  const unsigned long long t0 = global_ns();
  if (*reinterpret_cast<volatile unsigned*>(status)) return;   // a wait already expired: the run is lost, do not stall it further
  while ((int)(ld_acquire_sys(flag) - value) < 0) {
    if (global_ns() - t0 > kSpinLimitNs) {
      *status = 1u;
      return;
    }
    __nanosleep(100);
  }
}

}  // namespace r2d2
