// Shared device/host helpers for libr2d2_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "r2d2_b200.h"  // C ABI: error codes, config structs

namespace r2d2 {

// ---- error plumbing (C ABI: every entry returns int, message via r2d2_last_error) -------------
void set_last_error(const std::string& msg);
const char* last_error();


#define R2D2_CUDA_TRY(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::r2d2::set_last_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" +      \
                             __FILE__ + ":" + std::to_string(__LINE__));                      \
      return R2D2_ERR_CUDA;                                                           \
    }                                                                                         \
  } while (0)

#define R2D2_TRY(expr)                                                                        \
  do {                                                                                        \
    int _rc = (expr);                                                                         \
    if (_rc != R2D2_OK) return _rc;                                                   \
  } while (0)

#define R2D2_REQUIRE(cond, msg)                                                               \
  do {                                                                                        \
    if (!(cond)) {                                                                            \
      ::r2d2::set_last_error(std::string("argument check failed: ") + #cond + " (" + msg + ")"); \
      return R2D2_ERR_ARG;                                                            \
    }                                                                                         \
  } while (0)

// kernel-launch accounting (bench.py reports gpu_launches from it)
void count_launch(int n = 1);
long long launch_count();

// once-per-device guard for cudaFuncSetAttribute calls (function attributes are per device; a process may drive several)
struct PerDeviceOnce {
  unsigned long long done = 0;   // bit d set: already done on device d (d < 64); benign race: the call is idempotent
  bool need() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
    if (done & (1ull << dev)) return false;
    done |= (1ull << dev);
    return true;
  }
};

// streaming multiprocessors of the current device (cached per device): sizes grids of the grid-stride kernels and
// split-K factors
int num_sms();
// opt-in shared memory per block of the current device in bytes (cached per device; 227 KB on an H100)
int max_smem_optin();

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// ---- bf16 hi/lo split: x ~= hi + lo with ~16 significant bits; products hi*hi + hi*lo + lo*hi.
// Done with integer ops on the fp32 bit pattern (round-half-up on the magnitude, then keep the upper 16 bits): the
// F2F.BF16.F32 conversion instruction runs on a 16/clk/SM pipe and makes operand staging conversion-bound
// (2 conversions per element); IADD/LOP/PRMT/FADD issue at full rate.
__device__ __forceinline__ uint32_t bf16_hi_bits(float x) { return (__float_as_uint(x) + 0x8000u) & 0xFFFF0000u; }

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  const uint32_t h = bf16_hi_bits(x);
  const uint32_t l = bf16_hi_bits(x - __uint_as_float(h));
  hi = __ushort_as_bfloat16((unsigned short)(h >> 16));
  lo = __ushort_as_bfloat16((unsigned short)(l >> 16));
}

__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
  // a -> low 16 bits (lower k index), b -> high 16 bits
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// two consecutive elements -> one packed word per plane (x0 in the low half)
__device__ __forceinline__ void split_pack2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const uint32_t h0 = bf16_hi_bits(x0), h1 = bf16_hi_bits(x1);
  hi = __byte_perm(h0, h1, 0x7632);
  const uint32_t l0 = __float_as_uint(x0 - __uint_as_float(h0)) + 0x8000u;
  const uint32_t l1 = __float_as_uint(x1 - __uint_as_float(h1)) + 0x8000u;
  lo = __byte_perm(l0, l1, 0x7632);
}

// mma.sync m16n8k16 bf16 x bf16 -> f32 (legacy tensor path; SASS: HMMA.16816.F32.BF16)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_ptr) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_ptr);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_ptr) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(smem_ptr);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// one full 32-byte sector per lane (p 32-byte aligned), as two 16-byte accesses
__device__ __forceinline__ void st_global_v8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void ld_global_v8(const float* p, float (&v)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }
// accurate tanh (tanhf) is used everywhere results are compared at 1e-3 relative against fp32 torch.

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace r2d2
