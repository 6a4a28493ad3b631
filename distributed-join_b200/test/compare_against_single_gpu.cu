// compare_against_single_gpu.cu -- the reference's strongest integration test
// (test/compare_against_single_gpu.cu:96-205,237-268) against libdj_b200: rank 0 generates
// build / probe tables with the known-selectivity generator and joins them on ONE GPU; the tables
// are dealt to all ranks with distribute_table, joined with distributed_inner_join, gathered with
// collect_tables, and both results must be the same row multiset (sorted, compared element-wise).
// Same case matrix as the reference without the compression cases (nvcomp is out of scope).
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstdio>
#include <iostream>
#include <memory>
#include <string>
#include <vector>

#include "../host/bootstrap.hpp"
#include "../host/compression.hpp"
#include "../host/distribute_table.hpp"
#include "../host/distributed_join.hpp"
#include "../host/error.hpp"
#include "../host/generate_table.hpp"
#include "../host/setup.hpp"

using cudf::type_id;

static const char* type_name(type_id t)
{
  switch (t) {
    case type_id::INT32: return "int32_t";
    case type_id::INT64: return "int64_t";
    case type_id::TIMESTAMP_DAYS: return "timestamp_D";
    case type_id::TIMESTAMP_MILLISECONDS: return "timestamp_ms";
    case type_id::TIMESTAMP_NANOSECONDS: return "timestamp_ns";
    case type_id::DURATION_DAYS: return "duration_D";
    case type_id::DURATION_SECONDS: return "duration_s";
    case type_id::DURATION_MICROSECONDS: return "duration_us";
    default: return "?";
  }
}

// host copy of a 4-column table as sorted rows (the role of cudf::sort + verify_correctness,
// test/compare_against_single_gpu.cu:44-54,171-196); every column is read at its own width
static std::vector<std::array<int64_t, 4>> sorted_rows(cudf::table_view t)
{
  const int64_t n = t.num_rows();
  std::vector<std::array<int64_t, 4>> rows((size_t)n);
  for (int c = 0; c < 4; c++) {
    const size_t es = cudf::size_of(t.column(c).type());
    std::vector<char> h((size_t)n * es);
    CUDA_RT_CALL(cudaMemcpy(h.data(), t.column(c).head<char>(), h.size(), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; i++)
      rows[(size_t)i][c] = es == 4 ? (int64_t) reinterpret_cast<const int32_t*>(h.data())[i]
                                   : reinterpret_cast<const int64_t*>(h.data())[i];
  }
  std::sort(rows.begin(), rows.end());
  return rows;
}

static bool run_test(type_id key_t, type_id payload_t, cudf::size_type build_table_size,
                     cudf::size_type probe_table_size, double selectivity, bool is_build_table_key_unique,
                     int over_decomposition_factor, int nvlink_domain_size, Communicator* communicator)
{
  const int mpi_rank = communicator->mpi_rank;
  std::unique_ptr<cudf::table> build, probe, reference;
  cudf::table_view build_view, probe_view;
  if (mpi_rank == 0) {
    const int64_t rand_max_val = (int64_t)build_table_size * 2;
    std::tie(build, probe)     = generate_build_probe_tables<int64_t, int64_t>(
      build_table_size, probe_table_size, selectivity, rand_max_val, is_build_table_key_unique);
    // handed out in the requested column types (values fit: rand_max is a size_type)
    const std::vector<cudf::data_type> types{cudf::data_type(key_t), cudf::data_type(payload_t)};
    build      = cudf::narrow_like(build->view(), types);
    probe      = cudf::narrow_like(probe->view(), types);
    build_view = build->view();
    probe_view = probe->view();
    reference  = cudf::inner_join(build->view(), probe->view(), {0}, {0});
  }
  std::unique_ptr<cudf::table> local_build = distribute_table(build_view, communicator);
  std::unique_ptr<cudf::table> local_probe = distribute_table(probe_view, communicator);

  std::unique_ptr<cudf::table> join_result_all_ranks = distributed_inner_join(
    local_build->view(), local_probe->view(), {0}, {0}, communicator,
    generate_none_compression_options(local_build->view()), generate_none_compression_options(local_probe->view()),
    over_decomposition_factor, false, nullptr, nvlink_domain_size);

  std::unique_ptr<cudf::table> join_result = collect_tables(join_result_all_ranks->view(), communicator);

  int64_t ok = 1;
  if (mpi_rank == 0) {
    ok = join_result->num_columns() == 4 && reference->num_columns() == 4 &&
         join_result->num_rows() == reference->num_rows();
    for (int c = 0; ok && c < 4; c++) ok = join_result->view().column(c).type() == reference->view().column(c).type();
    if (ok) ok = sorted_rows(join_result->view()) == sorted_rows(reference->view());
    std::cerr << std::boolalpha << "Test case (" << type_name(key_t) << "," << type_name(payload_t) << ","
              << build_table_size << "," << probe_table_size << "," << selectivity << "," << is_build_table_key_unique
              << "," << over_decomposition_factor << ",false," << nvlink_domain_size << ") "
              << (ok ? "passes successfully" : "FAILED") << " (" << reference->num_rows() << " rows).\n";
  }
  return dj_bootstrap::allreduce_sum(ok) == communicator->mpi_size;
}

int main(int argc, char* argv[])
{
  dj_bootstrap::init(&argc, &argv);
  set_cuda_device();
  Communicator* communicator{nullptr};
  registered_memory_resource* registered_mr{nullptr};
  rmm::mr::pool_memory_resource<rmm::mr::device_memory_resource>* pool_mr{nullptr};
  setup_memory_pool_and_communicator(communicator, registered_mr, pool_mr, "NCCL", "none", 0);
  const type_id I32 = type_id::INT32, I64 = type_id::INT64;
  bool ok = true;
  // test/compare_against_single_gpu.cu:237-268, compression == false rows
  ok &= run_test(I32, I32, 1'000'000, 5'000'000, 0.3, true, 10, 1, communicator);
  ok &= run_test(I64, I64, 1'000'000, 5'000'000, 0.3, true, 10, 1, communicator);
  ok &= run_test(I32, I32, 1'000'000, 5'000'000, 1.0, true, 10, 1, communicator);
  ok &= run_test(I64, I64, 1'000'000, 5'000'000, 1.0, true, 10, 1, communicator);
  ok &= run_test(I32, I32, 1'000'000, 1'000'000, 0.3, true, 10, 1, communicator);
  ok &= run_test(I64, I64, 1'000'000, 1'000'000, 0.3, true, 10, 1, communicator);
  ok &= run_test(I32, I32, 1'000'000, 5'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I64, I64, 1'000'000, 5'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I64, type_id::TIMESTAMP_DAYS, 1'000'000, 1'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I64, type_id::TIMESTAMP_MILLISECONDS, 1'000'000, 1'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I64, type_id::TIMESTAMP_NANOSECONDS, 1'000'000, 1'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I64, type_id::DURATION_DAYS, 1'000'000, 1'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I64, type_id::DURATION_SECONDS, 1'000'000, 1'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I64, type_id::DURATION_MICROSECONDS, 1'000'000, 1'000'000, 0.3, true, 1, 1, communicator);
  ok &= run_test(I32, I32, 1'000'000, 1'000'000, 0.3, true, 1, 2, communicator);
  ok &= run_test(I32, I32, 1'000'000, 1'000'000, 0.3, true, 10, 2, communicator);
  // beyond the reference's list: the whole NVLink domain (the fused path) and duplicate build keys
  ok &= run_test(I64, I64, 1'000'000, 5'000'000, 0.3, true, 10, communicator->mpi_size, communicator);
  ok &= run_test(I64, I64, 1'000'000, 5'000'000, 0.9, false, 4, communicator->mpi_size, communicator);
  ok &= run_test(I32, I64, 2'000'000, 2'000'000, 0.3, true, 1, communicator->mpi_size, communicator);
  destroy_memory_pool_and_communicator(communicator, registered_mr, pool_mr, "NCCL", "none");
  dj_bootstrap::finalize();
  if (!ok) return 1;
  if (dj_bootstrap::rank() == 0) std::cerr << "Test case \"compare_against_single_gpu\" passes successfully." << std::endl;
  return 0;
}
