// shuffle_on.cpp -- BASELINE config 4: shuffle_on() of a 4-column int64 table, the timing
// harness of the reference's benchmark/gpubdb_shuffle_on.cpp on a synthetic table (the parquet
// reader is out of scope): uniform int64 surrogate keys in column 0, row-derived payloads.
// Prints the reference's "Throughput (GB/s)" figure: table bytes of all ranks / elapsed.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../host/bootstrap.hpp"
#include "../host/compression.hpp"
#include "../host/error.hpp"
#include "../host/generate_table.hpp"
#include "../host/setup.hpp"
#include "../host/shuffle_on.hpp"
#include "../../include/dj_b200.h"

// 128-bit order-independent checksum of a 4 x int64 table (library helper, not the oracle)
static void table_checksum(cudf::table_view t, uint64_t out[2])
{
  uint64_t* d = nullptr;
  CUDA_RT_CALL(cudaMalloc(&d, 16));
  CUDA_RT_CALL(cudaMemset(d, 0, 16));
  if (dj_multiset_checksum4(t.column(0).head<int64_t>(), t.column(1).head<int64_t>(), t.column(2).head<int64_t>(),
                            t.column(3).head<int64_t>(), t.num_rows(), d, nullptr) != DJ_OK)
    throw std::runtime_error(dj_last_error());
  CUDA_RT_CALL(cudaMemcpy(out, d, 16, cudaMemcpyDeviceToHost));
  CUDA_RT_CALL(cudaFree(d));
}

int main(int argc, char* argv[])
{
  dj_bootstrap::init(&argc, &argv);
  set_cuda_device();
  int64_t rows_per_rank = 400'000'000;
  int iterations        = 3;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "--nrows") && i + 1 < argc) rows_per_rank = atoll(argv[i + 1]);
    if (!strcmp(argv[i], "--iterations") && i + 1 < argc) iterations = atoi(argv[i + 1]);
  }
  Communicator* communicator{nullptr};
  registered_memory_resource* registered_mr{nullptr};
  rmm::mr::pool_memory_resource<rmm::mr::device_memory_resource>* pool_mr{nullptr};
  setup_memory_pool_and_communicator(communicator, registered_mr, pool_mr, "NCCL", "none", 0);
  const int rank = communicator->mpi_rank, size = communicator->mpi_size;

  // four int64 columns: random keys (the generator's duplicate-allowed build stream) + 3 payloads.
  // Keys come from [0, 2^34]: that stream keeps a bitmap of rand_max + 1 bits (2 GB here), which has
  // to fit on an 80 GB GPU next to the table and its shuffled copy.
  std::unique_ptr<cudf::table> kp, unused;
  std::tie(kp, unused) = generate_build_probe_tables<int64_t, int64_t>((cudf::size_type)rows_per_rank, 1, 0.0,
                                                                       (int64_t)1 << 34, false, rank);
  std::vector<std::unique_ptr<cudf::column>> cols;
  {
    auto v = kp->view();
    for (int c = 0; c < 4; c++) {
      cols.push_back(cudf::make_numeric_column(cudf::data_type(cudf::type_id::INT64), (cudf::size_type)rows_per_rank));
      CUDA_RT_CALL(cudaMemcpy(cols.back()->mutable_view().head<char>(), v.column(c == 0 ? 0 : 1).head<char>(),
                              (size_t)rows_per_rank * 8, cudaMemcpyDeviceToDevice));
    }
  }
  kp.reset();
  unused.reset();
  cudf::table input(std::move(cols));
  warmup_all_to_all(communicator);

  uint64_t ck_before[2];
  table_checksum(input.view(), ck_before);
  double best = 1e30;
  int64_t rows_after = 0, misplaced = 0;
  uint64_t ck_after[2] = {0, 0};
  for (int it = 0; it < iterations; it++) {
    CUDA_RT_CALL(cudaDeviceSynchronize());
    dj_bootstrap::barrier();
    const double t0 = dj_bootstrap::wtime();
    auto shuffled   = shuffle_on(input.view(), {0}, communicator, generate_none_compression_options(input.view()),
                                 cudf::hash_id::HASH_MURMUR3, cudf::DEFAULT_HASH_SEED);
    dj_bootstrap::barrier();
    const double t = dj_bootstrap::wtime() - t0;
    rows_after     = dj_bootstrap::allreduce_sum(shuffled->num_rows());
    if (t < best) best = t;
    if (it == iterations - 1) {
      // property checks outside the timed region (test/test_shuffle_on.cpp:78-83 generalised):
      // every row is on the rank its key hashes to, and the global row multiset is unchanged
      table_checksum(shuffled->view(), ck_after);
      const int64_t n = shuffled->num_rows();
      if (n > 0) {
        int32_t* ids = nullptr;
        CUDA_RT_CALL(cudaMalloc(&ids, (size_t)n * 4));
        if (dj_partition_ids_i64(shuffled->view().column(0).head<int64_t>(), n, cudf::DEFAULT_HASH_SEED, DJ_HASH_MURMUR3,
                                 size, ids, nullptr) != DJ_OK)
          throw std::runtime_error(dj_last_error());
        std::vector<int32_t> h((size_t)n);
        CUDA_RT_CALL(cudaMemcpy(h.data(), ids, (size_t)n * 4, cudaMemcpyDeviceToHost));
        for (int32_t v : h) misplaced += v != rank;
        CUDA_RT_CALL(cudaFree(ids));
      }
    }
  }
  // checksums are sums mod 2^64 over rows: the per-rank values add up to the global one
  const int64_t sum_before0 = dj_bootstrap::allreduce_sum((int64_t)ck_before[0]);
  const int64_t sum_before1 = dj_bootstrap::allreduce_sum((int64_t)ck_before[1]);
  const int64_t sum_after0  = dj_bootstrap::allreduce_sum((int64_t)ck_after[0]);
  const int64_t sum_after1  = dj_bootstrap::allreduce_sum((int64_t)ck_after[1]);
  misplaced                 = dj_bootstrap::allreduce_sum(misplaced);
  const bool verified = rows_after == rows_per_rank * size && misplaced == 0 && sum_before0 == sum_after0 &&
                        sum_before1 == sum_after1;
  if (rank == 0) {
    const double bytes = (double)rows_per_rank * size * 4 * 8;
    std::cout << "Elasped time (s): " << best << std::endl;
    std::cout << "Throughput (GB/s): " << bytes / best / 1e9 << std::endl;
    std::cout << "{\"benchmark\": \"shuffle_on\", \"n_gpus\": " << size << ", \"rows_per_rank\": " << rows_per_rank
              << ", \"rows_after\": " << rows_after << ", \"seconds\": " << best
              << ", \"throughput_GBps\": " << bytes / best / 1e9 << ", \"misplaced_rows\": " << misplaced
              << ", \"multiset_checksum_preserved\": " << (sum_before0 == sum_after0 && sum_before1 == sum_after1)
              << ", \"verified\": " << verified << "}" << std::endl;
    std::cout << (verified ? "shuffle_on check: OK (rows preserved, co-located, checksum preserved)"
                           : "shuffle_on check: MISMATCH") << std::endl;
  }
  if (!verified) {
    dj_bootstrap::finalize();
    return 1;
  }
  destroy_memory_pool_and_communicator(communicator, registered_mr, pool_mr, "NCCL", "none");
  dj_bootstrap::finalize();
  return 0;
}
