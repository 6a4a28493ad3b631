// dj_device.cuh -- device-side primitives shared by the sm_90a kernels:
// hashes, Philox / Feistel generator pieces, block scan, launch bookkeeping.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dj_b200.h"

namespace dj {

// ---------------------------------------------------------------- error / launch bookkeeping
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define DJ_CUDA_TRY(expr)                                                              \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      dj::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return DJ_ERR_CUDA;                                                              \
    }                                                                                  \
  } while (0)

#define DJ_LAUNCH_CHECK()                 \
  do {                                    \
    dj::count_launch();                   \
    DJ_CUDA_TRY(cudaPeekAtLastError());   \
  } while (0)

#define DJ_REQUIRE(cond, ...)      \
  do {                             \
    if (!(cond)) {                 \
      dj::set_error(__VA_ARGS__);  \
      return DJ_ERR_ARG;           \
    }                              \
  } while (0)

int sm_count();           // SMs persistent kernels size their grids for (physical - reserve)
int sm_count_physical();
void set_sm_reserve(int n);

// Brackets one kernel launch with CUDA events when profiling is enabled (dj_profile_enable).
struct ProfScope {
  int cat;
  cudaStream_t stream;
  int slot;
  ProfScope(int category, cudaStream_t st);
  ~ProfScope();
};

// ---------------------------------------------------------------- hashing
__host__ __device__ __forceinline__ uint32_t rotl32(uint32_t x, int r)
{
  return (x << r) | (x >> (32 - r));
}

__host__ __device__ __forceinline__ uint32_t fmix32(uint32_t h)
{
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}

// MurmurHash3_x86_32 over the 8 little-endian bytes of an int64 key (cudf HASH_MURMUR3 for
// an int64 column; call sites src/distributed_join.cpp:211-225).
__host__ __device__ __forceinline__ uint32_t murmur3_i64(int64_t key, uint32_t seed)
{
  uint32_t h  = seed;
  uint32_t k0 = (uint32_t)(uint64_t)key, k1 = (uint32_t)((uint64_t)key >> 32);
  k0 *= 0xcc9e2d51u; k0 = rotl32(k0, 15); k0 *= 0x1b873593u;
  h ^= k0; h = rotl32(h, 13); h = h * 5u + 0xe6546b64u;
  k1 *= 0xcc9e2d51u; k1 = rotl32(k1, 15); k1 *= 0x1b873593u;
  h ^= k1; h = rotl32(h, 13); h = h * 5u + 0xe6546b64u;
  h ^= 8u;
  return fmix32(h);
}

// cuDF 0.19 row_hasher, single key column: hash_combine(0, element hash).
__host__ __device__ __forceinline__ uint32_t row_hash_i64(int64_t key, uint32_t seed, int hash_id)
{
  uint32_t h = hash_id == DJ_HASH_MURMUR3 ? murmur3_i64(key, seed) : (uint32_t)(uint64_t)key;
  return h + 0x9e3779b9u;
}

// Hash used for the join's private radix sub-partitioning; the radix levels consume its TOP bits.
// It must be independent of the rank-partition hash (rows on one rank share row_hash % nparts) but
// is otherwise free: two 64-bit multiplies with an xor-shift between them (about half the
// instructions of murmur3: the scatter kernels spend their time issuing instructions, not waiting on HBM).
__host__ __device__ __forceinline__ uint32_t local_hash_i64(int64_t key)
{
  uint64_t x = (uint64_t)key * 0x9E3779B97F4A7C15ull;
  x ^= x >> 29;
  x *= 0xD6E8FEB86659FD93ull;
  return (uint32_t)(x >> 32);
}

// Slot hash inside one shared-memory bucket: must be independent of local_hash's radix bits.
__host__ __device__ __forceinline__ uint32_t slot_hash_i64(int64_t key)
{
  uint32_t lo = (uint32_t)(uint64_t)key, hi = (uint32_t)((uint64_t)key >> 32);
  uint32_t x  = lo ^ (hi * 0x85ebca6bu + 0x632be5abu);
  x *= 0x9E3779B1u;
  x ^= x >> 15;
  x *= 0x2c1b3c6du;
  return x;
}

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x)
{
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}

// ---------------------------------------------------------------- generator pieces
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                                       uint32_t c3, uint32_t k0, uint32_t k1,
                                                       uint32_t out[4])
{
#pragma unroll
  for (int r = 0; r < 10; r++) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__host__ __device__ __forceinline__ double u01(uint32_t hi, uint32_t lo)
{
  return (double)((((uint64_t)hi << 32) | lo) >> 11) * (1.0 / 9007199254740992.0);
}

__host__ __device__ __forceinline__ uint64_t feistel_perm(uint64_t x, uint64_t L, int half,
                                                          uint64_t seed, uint32_t src_rank)
{
  const uint32_t mask = (uint32_t)(((uint64_t)1 << half) - 1);
  do {
    uint32_t l = (uint32_t)(x >> half) & mask, r = (uint32_t)x & mask;
#pragma unroll
    for (uint32_t rnd = 0; rnd < 6; rnd++) {
      uint32_t f = fmix32(r * 0x9E3779B1u + (uint32_t)seed + 0x7F4A7C15u * (rnd + 1) +
                          0x85EBCA77u * src_rank + (uint32_t)(seed >> 32));
      uint32_t t = l ^ (f & mask);
      l          = r;
      r          = t;
    }
    x = ((uint64_t)l << half) | r;
  } while (x >= L);
  return x;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------- block-wide exclusive scan
// Exclusive prefix sum of one int per thread across a THREADS-wide CTA.  `warp_sums` is
// 33 ints of shared memory; warp_sums[32] receives the block total.  Contains two
// __syncthreads (callers must sync again before reusing warp_sums).
template <int THREADS>
__device__ __forceinline__ int block_exclusive_scan(int v, int* warp_sums)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = lane < THREADS / 32 ? warp_sums[lane] : 0;
    int wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, wi, d);
      if (lane >= d) wi += t;
    }
    if (lane < THREADS / 32) warp_sums[lane] = wi - w;  // exclusive warp offsets
    if (lane == 31) warp_sums[32] = wi;
  }
  __syncthreads();
  return warp_sums[warp] + incl - v;
}

// ---------------------------------------------------------------- PTX helpers (mbarrier + TMA)
__device__ __forceinline__ uint32_t smem_u32(const void* p)
{
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity)
{
  asm volatile(
    "{\n"
    ".reg .pred p;\n"
    "WAIT_LOOP:\n"
    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
    "@p bra WAIT_DONE;\n"
    "bra WAIT_LOOP;\n"
    "WAIT_DONE:\n"
    "}\n" ::"r"(smem_u32(bar)),
    "r"(parity)
    : "memory");
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         unsigned long long* bar)
{
  asm volatile(
    "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
      smem_u32(smem_dst)),
    "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
    : "memory");
}

// position of row p inside the 16-byte aligned window staged for it (partition.cu: stage_column)
__device__ __forceinline__ int skip_of(const int64_t* p)
{
  return (int)((reinterpret_cast<uintptr_t>(p) & 15) >> 3);
}


__device__ __forceinline__ unsigned lanemask_lt()
{
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}
#endif

}  // namespace dj
