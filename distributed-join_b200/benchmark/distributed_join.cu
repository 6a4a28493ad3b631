// distributed_join.cu -- the reference's synthetic join benchmark (benchmark/distributed_join.cu)
// built against libdj_b200.  Same flags, same parameter report, same "Elasped time (s)"
// line; MPI calls are replaced by dj_bootstrap (ranks come from RANK/WORLD_SIZE), row counts are
// 64-bit, and a JSON line with rows/s is printed next to the reference's output.
//
//   torchrun --no-python --nproc-per-node 8 bin/distributed_join --communicator NCCL
//            --build-table-nrows 100000000 --probe-table-nrows 100000000 --nvlink-domain-size 8
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <memory>
#include <stdexcept>
#include <string>
#include <tuple>

#include <cuda_profiler_api.h>

#include "../host/bootstrap.hpp"
#include "../host/communicator.hpp"
#include "../host/compression.hpp"
#include "../host/distributed_join.hpp"
#include "../host/error.hpp"
#include "../host/generate_table.hpp"
#include "../host/setup.hpp"

static std::string key_type     = "int64_t";
static std::string payload_type = "int64_t";
static int64_t BUILD_TABLE_NROWS_EACH_RANK = 100'000'000;
static int64_t PROBE_TABLE_NROWS_EACH_RANK = 100'000'000;
static double SELECTIVITY                  = 0.3;
static bool IS_BUILD_TABLE_KEY_UNIQUE      = true;
static int OVER_DECOMPOSITION_FACTOR       = 1;
static std::string COMMUNICATOR_NAME       = "NCCL";  // the reference defaults to UCX
static std::string REGISTRATION_METHOD     = "none";
static int64_t COMMUNICATOR_BUFFER_SIZE    = 1'600'000'000LL;
static bool COMPRESSION                    = false;
static int NVLINK_DOMAIN_SIZE              = 1;
static bool REPORT_TIMING                  = false;
static int ITERATIONS                      = 1;  // the reference times one cold run

static void parse_command_line_arguments(int argc, char* argv[])
{
  auto value = [&](int i) -> const char* {
    if (i + 1 >= argc) throw std::runtime_error(std::string("missing value after ") + argv[i]);
    return argv[i + 1];
  };
  for (int i = 1; i < argc; i++) {
    const std::string a = argv[i];
    if (a == "--key-type") key_type = value(i);
    if (a == "--payload-type") payload_type = value(i);
    if (a == "--build-table-nrows") BUILD_TABLE_NROWS_EACH_RANK = std::atoll(value(i));
    if (a == "--probe-table-nrows") PROBE_TABLE_NROWS_EACH_RANK = std::atoll(value(i));
    if (a == "--selectivity") SELECTIVITY = std::atof(value(i));
    if (a == "--duplicate-build-keys") IS_BUILD_TABLE_KEY_UNIQUE = false;
    if (a == "--over-decomposition-factor") OVER_DECOMPOSITION_FACTOR = std::atoi(value(i));
    if (a == "--communicator") COMMUNICATOR_NAME = value(i);
    if (a == "--compression") COMPRESSION = true;
    if (a == "--registration-method") REGISTRATION_METHOD = value(i);
    if (a == "--nvlink-domain-size") NVLINK_DOMAIN_SIZE = std::atoi(value(i));
    if (a == "--report-timing") REPORT_TIMING = true;
    if (a == "--iterations") ITERATIONS = std::atoi(value(i));
  }
}

static void report_configuration()
{
  if (dj_bootstrap::rank() != 0) return;
  const int mpi_size = dj_bootstrap::size();
  std::cout << "========== Parameters ==========" << std::endl << std::boolalpha;
  std::cout << "Key type: " << key_type << std::endl;
  std::cout << "Payload type: " << payload_type << std::endl;
  std::cout << "Number of rows in the build table: " << BUILD_TABLE_NROWS_EACH_RANK * mpi_size / 1e6 << " million"
            << std::endl;
  std::cout << "Number of rows in the probe table: " << PROBE_TABLE_NROWS_EACH_RANK * mpi_size / 1e6 << " million"
            << std::endl;
  std::cout << "Selectivity: " << SELECTIVITY << std::endl;
  std::cout << "Keys in build table are unique: " << IS_BUILD_TABLE_KEY_UNIQUE << std::endl;
  std::cout << "Over-decomposition factor: " << OVER_DECOMPOSITION_FACTOR << std::endl;
  std::cout << "Communicator: " << COMMUNICATOR_NAME << std::endl;
  std::cout << "Compression: " << COMPRESSION << std::endl;
  std::cout << "NVLink domain size: " << NVLINK_DOMAIN_SIZE << std::endl;
  std::cout << "================================" << std::endl;
}

int main(int argc, char* argv[])
{
  dj_bootstrap::init(&argc, &argv);
  set_cuda_device();
  parse_command_line_arguments(argc, argv);
  report_configuration();
  if (std::max(BUILD_TABLE_NROWS_EACH_RANK, PROBE_TABLE_NROWS_EACH_RANK) > INT32_MAX)
    throw std::runtime_error("per-rank tables are limited to cudf::size_type rows at this API level");

  const int64_t RAND_MAX_VAL = std::max(BUILD_TABLE_NROWS_EACH_RANK, PROBE_TABLE_NROWS_EACH_RANK) * 2;
  const int mpi_rank = dj_bootstrap::rank(), mpi_size = dj_bootstrap::size();

  Communicator* communicator{nullptr};
  registered_memory_resource* registered_mr{nullptr};
  rmm::mr::pool_memory_resource<rmm::mr::device_memory_resource>* pool_mr{nullptr};
  setup_memory_pool_and_communicator(communicator, registered_mr, pool_mr, COMMUNICATOR_NAME, REGISTRATION_METHOD,
                                     COMMUNICATOR_BUFFER_SIZE);

  void* preallocated_pinned_buffer;
  CUDA_RT_CALL(cudaMallocHost(&preallocated_pinned_buffer, mpi_size * sizeof(size_t)));
  if (COMPRESSION) warmup_nvcomp();

  std::unique_ptr<cudf::table> left, right;
  auto generate = [&](auto key_tag, auto payload_tag) {
    using KEY_T     = decltype(key_tag);
    using PAYLOAD_T = decltype(payload_tag);
    std::tie(left, right) = generate_tables_distributed<KEY_T, PAYLOAD_T>(
      (cudf::size_type)BUILD_TABLE_NROWS_EACH_RANK, (cudf::size_type)PROBE_TABLE_NROWS_EACH_RANK, SELECTIVITY,
      (KEY_T)RAND_MAX_VAL, IS_BUILD_TABLE_KEY_UNIQUE, communicator);
  };
  // same type matrix as the reference driver (benchmark/distributed_join.cu:225-253); 4-byte columns
  // are widened to the kernels' 8-byte rows inside the library shim
  if (key_type == "int64_t" && payload_type == "int64_t") generate(int64_t{}, int64_t{});
  else if (key_type == "int64_t" && payload_type == "int32_t") generate(int64_t{}, int32_t{});
  else if (key_type == "int32_t" && payload_type == "int64_t") generate(int32_t{}, int64_t{});
  else if (key_type == "int32_t" && payload_type == "int32_t") generate(int32_t{}, int32_t{});
  else throw std::runtime_error("Unknown key / payload type");
  if (key_type == "int32_t" && RAND_MAX_VAL * (int64_t)mpi_size > INT32_MAX)
    throw std::runtime_error("int32_t keys: rand_max * ranks exceeds the key range");

  auto left_compression_options  = generate_compression_options_distributed(left->view(), COMPRESSION);
  auto right_compression_options = generate_compression_options_distributed(right->view(), COMPRESSION);

  double best = 1e30;
  int64_t rows_out = 0;
  for (int it = 0; it < ITERATIONS; it++) {
    CUDA_RT_CALL(cudaDeviceSynchronize());
    dj_bootstrap::barrier();
    cudaProfilerStart();
    const double start = dj_bootstrap::wtime();
    std::unique_ptr<cudf::table> join_result = distributed_inner_join(
      left->view(), right->view(), {0}, {0}, communicator, left_compression_options, right_compression_options,
      OVER_DECOMPOSITION_FACTOR, REPORT_TIMING, preallocated_pinned_buffer, NVLINK_DOMAIN_SIZE);
    dj_bootstrap::barrier();
    const double stop = dj_bootstrap::wtime();
    cudaProfilerStop();
    rows_out = dj_bootstrap::allreduce_sum(join_result->num_rows());
    if (mpi_rank == 0) std::cout << "Elasped time (s) " << stop - start << std::endl;
    best = std::min(best, stop - start);
    join_result.reset();
  }
  if (mpi_rank == 0) {
    const double rows_in = (double)(BUILD_TABLE_NROWS_EACH_RANK + PROBE_TABLE_NROWS_EACH_RANK) * mpi_size;
    std::cout << "{\"benchmark\": \"distributed_join\", \"n_gpus\": " << mpi_size << ", \"seconds\": " << best
              << ", \"input_rows_per_s\": " << rows_in / best << ", \"output_rows\": " << rows_out
              << ", \"output_rows_per_s\": " << rows_out / best << "}" << std::endl;
  }

  left.reset();
  right.reset();
  CUDA_RT_CALL(cudaFreeHost(preallocated_pinned_buffer));
  CUDA_RT_CALL(cudaDeviceSynchronize());
  destroy_memory_pool_and_communicator(communicator, registered_mr, pool_mr, COMMUNICATOR_NAME, REGISTRATION_METHOD);
  dj_bootstrap::finalize();
  return 0;
}
