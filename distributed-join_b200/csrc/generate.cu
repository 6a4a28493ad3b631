// generate.cu -- known-selectivity build/probe generator, partition-id and checksum helpers.
//
// Restates generate_input_tables (generate_dataset/generate_dataset.cuh:47-135,163-260) and
// the rank offsets of generate_tables_distributed (src/generate_table.cuh:192-202) with a
// counter-based RNG so any row of any source rank can be produced independently, on the GPU
// here and bit-identically on the CPU in oracle/dj_oracle.c:
//   unique build keys : build[i] = perm(i), perm a Feistel permutation of [0, rand_max]
//                       (the reference's lottery draws a random distinct subset, :64-84);
//   duplicates allowed: build[i] = floor(u * rand_max)                          (:85-86);
//   probe row         : hit iff u < selectivity -> key of a uniformly random build ROW
//                       (:114-122), else a key guaranteed absent from build     (:126-128).
#include "dj_device.cuh"
#include "dj_internal.h"

namespace dj {

namespace {

struct GenDev {
  int64_t nb, np, rand_max;
  double selectivity;
  uint64_t seed;
  int unique;
  int half;  // Feistel half width for L = rand_max + 1
};

__host__ __device__ inline int feistel_half(uint64_t L)
{
  int bits = 2;
  while (((uint64_t)1 << bits) < L) bits += 2;
  return bits / 2;
}

__device__ __forceinline__ void gen_draw(const GenDev& g, int stream, int attempt, int src,
                                         int64_t row, double& x0, double& x1)
{
  uint32_t o[4];
  philox4x32_10((uint32_t)row, (uint32_t)((uint64_t)row >> 32),
                (uint32_t)stream | ((uint32_t)attempt << 8), (uint32_t)src, (uint32_t)g.seed,
                (uint32_t)(g.seed >> 32), o);
  x0 = u01(o[0], o[1]);
  x1 = u01(o[2], o[3]);
}

__device__ __forceinline__ int64_t clampi(int64_t v, int64_t hi) { return v > hi ? hi : v; }

__device__ __forceinline__ int64_t build_local(const GenDev& g, int src, int64_t row)
{
  const int64_t L = g.rand_max + 1;
  if (g.unique) return (int64_t)feistel_perm((uint64_t)row, (uint64_t)L, g.half, g.seed, (uint32_t)src);
  double x0, x1;
  gen_draw(g, 0, 0, src, row, x0, x1);
  return clampi((int64_t)(x0 * (double)g.rand_max), g.rand_max);
}

__device__ __forceinline__ int64_t probe_local(const GenDev& g, int src, int64_t row,
                                               const uint32_t* bitmap)
{
  const int64_t L = g.rand_max + 1;
  double x0, x1;
  gen_draw(g, 1, 0, src, row, x0, x1);
  const bool no_miss_keys = g.unique && (L - g.nb <= 0);
  if (x0 < g.selectivity || no_miss_keys) {
    const int64_t j = clampi((int64_t)(x1 * (double)g.nb), g.nb - 1);
    return build_local(g, src, j);
  }
  if (g.unique) {
    const int64_t m = clampi((int64_t)(x1 * (double)(L - g.nb)), L - g.nb - 1);
    return (int64_t)feistel_perm((uint64_t)(g.nb + m), (uint64_t)L, g.half, g.seed, (uint32_t)src);
  }
  int64_t c = clampi((int64_t)(x1 * (double)L), L - 1);
  for (int attempt = 1; attempt < 64 && ((bitmap[c >> 5] >> (c & 31)) & 1u); attempt++) {
    gen_draw(g, 1, attempt, src, row, x0, x1);
    c = clampi((int64_t)(x1 * (double)L), L - 1);
  }
  for (int64_t step = 0; step < L && ((bitmap[c >> 5] >> (c & 31)) & 1u); step++) c = (c + 1) % L;
  return c;
}

__global__ void bitmap_kernel(GenDev g, int src, uint32_t* bitmap)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < g.nb;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = build_local(g, src, i);
    atomicOr(&bitmap[k >> 5], 1u << (k & 31));
  }
}

__global__ void generate_kernel(GenDev g, int which, int src, int64_t row_begin, int64_t count,
                                const uint32_t* bitmap, int64_t* keys, int64_t* payload)
{
  const int64_t n_rank = which ? g.np : g.nb;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < count;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = row_begin + t;
    const int64_t k   = which ? probe_local(g, src, row, bitmap) : build_local(g, src, row);
    keys[t]           = k + g.rand_max * (int64_t)src;
    payload[t]        = row + n_rank * (int64_t)src;
  }
}

__global__ void partition_ids_kernel(const int64_t* keys, int64_t n, uint32_t seed, int hash_id,
                                     int nparts, int32_t* out)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int32_t)(row_hash_i64(keys[i], seed, hash_id) % (uint32_t)nparts);
}

__global__ void checksum_kernel(const int64_t* c0, const int64_t* c1, const int64_t* c2,
                                const int64_t* c3, int64_t n, unsigned long long* out2)
{
  unsigned long long s1 = 0, s2 = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t a = (uint64_t)c0[i], b = (uint64_t)c1[i], c = (uint64_t)c2[i], d = (uint64_t)c3[i];
    uint64_t x = mix64(a + 0x9e3779b97f4a7c15ULL);
    x          = mix64(x ^ b);
    x          = mix64(x + c);
    x          = mix64(x ^ d);
    uint64_t y = mix64(d * 0xd6e8feb86659fd93ULL + 1);
    y          = mix64(y + c);
    y          = mix64(y ^ b);
    y          = mix64(y + a);
    s1 += x;
    s2 += y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out2[0], s1);
    atomicAdd(&out2[1], s2);
  }
}

GenDev to_dev(const dj_gen_params* p)
{
  GenDev g;
  g.nb          = p->nb;
  g.np          = p->np;
  g.rand_max    = p->rand_max;
  g.selectivity = p->selectivity;
  g.seed        = p->seed;
  g.unique      = p->unique_build_keys;
  g.half        = feistel_half((uint64_t)p->rand_max + 1);
  return g;
}

int grid_for(int64_t n, int threads)
{
  int64_t blocks = (n + threads - 1) / threads;
  int64_t cap    = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

}  // namespace

const void* generate_module_kernel() { return (const void*)checksum_kernel; }

}  // namespace dj

using namespace dj;

extern "C" int dj_generate_build_bitmap(const dj_gen_params* p, int src_rank, uint32_t* d_bitmap,
                                        void* stream)
{
  DJ_REQUIRE(p && d_bitmap, "generate_build_bitmap: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t words = (size_t)((p->rand_max + 1 + 31) / 32);
  DJ_CUDA_TRY(cudaMemsetAsync(d_bitmap, 0, words * 4, st));
  if (p->nb > 0) {
    bitmap_kernel<<<grid_for(p->nb, 256), 256, 0, st>>>(to_dev(p), src_rank, d_bitmap);
    DJ_LAUNCH_CHECK();
  }
  return DJ_OK;
}

extern "C" int dj_generate_rows_i64(const dj_gen_params* p, int which, int src_rank,
                                    int64_t row_begin, int64_t count, const uint32_t* d_bitmap,
                                    int64_t* d_keys, int64_t* d_payload, void* stream)
{
  DJ_REQUIRE(p && d_keys && d_payload, "generate_rows: null argument");
  DJ_REQUIRE(which == 0 || which == 1, "generate_rows: which must be 0 (build) or 1 (probe)");
  DJ_REQUIRE(p->rand_max >= 1 && p->nb >= 1, "generate_rows: rand_max and nb must be >= 1");
  DJ_REQUIRE(!p->unique_build_keys || p->nb <= p->rand_max + 1,
             "generate_rows: unique build keys need nb <= rand_max + 1");
  DJ_REQUIRE(which == 0 || p->unique_build_keys || d_bitmap,
             "generate_rows: probe rows with duplicate build keys need the build bitmap");
  if (count <= 0) return DJ_OK;
  generate_kernel<<<grid_for(count, 256), 256, 0, (cudaStream_t)stream>>>(
    to_dev(p), which, src_rank, row_begin, count, d_bitmap, d_keys, d_payload);
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

extern "C" int dj_partition_ids_i64(const int64_t* d_keys, int64_t nrows, uint32_t seed,
                                    int hash_id, int nparts, int32_t* d_out_ids, void* stream)
{
  DJ_REQUIRE(nparts >= 1, "partition_ids: nparts must be >= 1");
  if (nrows <= 0) return DJ_OK;
  partition_ids_kernel<<<grid_for(nrows, 256), 256, 0, (cudaStream_t)stream>>>(
    d_keys, nrows, seed, hash_id, nparts, d_out_ids);
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}

extern "C" int dj_multiset_checksum4(const int64_t* d_c0, const int64_t* d_c1, const int64_t* d_c2,
                                     const int64_t* d_c3, int64_t nrows, uint64_t* d_out2,
                                     void* stream)
{
  if (nrows <= 0) return DJ_OK;
  checksum_kernel<<<grid_for(nrows, 256), 256, 0, (cudaStream_t)stream>>>(
    d_c0, d_c1, d_c2, d_c3, nrows, (unsigned long long*)d_out2);
  DJ_LAUNCH_CHECK();
  return DJ_OK;
}
