// compare_against_analytical.cu -- the reference's analytical integration test
// (test/compare_against_analytical.cu) against libdj_b200: left keys 0,3,6,..., right keys
// 0,5,10,..., payload = row id; after distributed_inner_join the global row count must be
// size/5 and every row must satisfy  key%15==0, left payload == key/3, right payload == key/5.
// Each rank holds a contiguous slice (what distribute_table would hand it).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <memory>
#include <vector>

#include "../host/bootstrap.hpp"
#include "../host/compression.hpp"
#include "../host/distributed_join.hpp"
#include "../host/error.hpp"
#include "../host/setup.hpp"

template <typename T>
__global__ void fill_multiples(T* key, T* payload, int64_t first_row, int64_t n, int64_t multiple)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    key[i]     = (T)((first_row + i) * multiple);
    payload[i] = (T)(first_row + i);
  }
}

template <typename T>
__global__ void count_violations(const T* c0, const T* c1, const T* c2, const T* c3,
                                 int64_t n, unsigned long long* bad)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const bool ok = c0[i] % 15 == 0 && c1[i] == c0[i] / 3 && c2[i] % 15 == 0 && c3[i] == c2[i] / 5 && c0[i] == c2[i];
    if (!ok) atomicAdd(bad, 1ull);
  }
}

template <typename T>
static std::unique_ptr<cudf::table> slice_of_multiples(int64_t size, int64_t multiple, int rank, int world)
{
  const int64_t lo = size * rank / world, hi = size * (rank + 1) / world;
  std::vector<std::unique_ptr<cudf::column>> cols;
  for (int c = 0; c < 2; c++)
    cols.push_back(cudf::make_numeric_column(cudf::data_type(cudf::type_to_id<T>()), (cudf::size_type)(hi - lo)));
  fill_multiples<T><<<256, 256>>>(cols[0]->mutable_view().template head<T>(), cols[1]->mutable_view().template head<T>(), lo,
                                  hi - lo, multiple);
  CUDA_RT_CALL(cudaDeviceSynchronize());
  return std::make_unique<cudf::table>(std::move(cols));
}

template <typename T>
static bool run_test(int64_t size, int odf, int nvl, Communicator* communicator)
{
  const int rank = communicator->mpi_rank, world = communicator->mpi_size;
  auto left  = slice_of_multiples<T>(size, 3, rank, world);
  auto right = slice_of_multiples<T>(size, 5, rank, world);
  auto result = distributed_inner_join(left->view(), right->view(), {0}, {0}, communicator,
                                       generate_none_compression_options(left->view()),
                                       generate_none_compression_options(right->view()), odf, false, nullptr, nvl);
  unsigned long long* d_bad;
  CUDA_RT_CALL(cudaMalloc(&d_bad, 8));
  CUDA_RT_CALL(cudaMemset(d_bad, 0, 8));
  if (result->num_rows() > 0) {
    if (result->num_columns() != 4) return false;
    auto v = result->view();
    if (!(v.column(0).type() == cudf::data_type(cudf::type_to_id<T>()))) return false;  // types survive the join
    count_violations<T><<<256, 256>>>(v.column(0).template head<T>(), v.column(1).template head<T>(), v.column(2).template head<T>(),
                                      v.column(3).template head<T>(), v.num_rows(), d_bad);
  }
  unsigned long long bad = 0;
  CUDA_RT_CALL(cudaMemcpy(&bad, d_bad, 8, cudaMemcpyDeviceToHost));
  CUDA_RT_CALL(cudaFree(d_bad));
  const int64_t total_rows = dj_bootstrap::allreduce_sum(result->num_rows());
  const int64_t total_bad  = dj_bootstrap::allreduce_sum((int64_t)bad);
  const bool ok            = total_rows == size / 5 && total_bad == 0;
  if (rank == 0)
    std::cerr << (sizeof(T) == 4 ? "int32 " : "int64 ") << "size " << size << " odf " << odf << " nvl " << nvl << ": rows " << total_rows << " (expected "
              << size / 5 << "), violations " << total_bad << (ok ? " -> passes successfully" : " -> FAILED")
              << std::endl;
  return ok;
}

int main(int argc, char* argv[])
{
  dj_bootstrap::init(&argc, &argv);
  set_cuda_device();
  Communicator* communicator{nullptr};
  registered_memory_resource* registered_mr{nullptr};
  rmm::mr::pool_memory_resource<rmm::mr::device_memory_resource>* pool_mr{nullptr};
  setup_memory_pool_and_communicator(communicator, registered_mr, pool_mr, "NCCL", "none", 0);
  const int world = communicator->mpi_size;
  bool ok = true;
  // the reference's case list (test/compare_against_analytical.cu:194-201) without compression;
  // nvl = world exercises the fused NVLink path, nvl 1 / 2 the staged general path
  // the reference generates int32 tables here (test/compare_against_analytical.cu:64-81)
  ok &= run_test<int32_t>(30'000, 1, 1, communicator);
  ok &= run_test<int32_t>(300'000, 4, world, communicator);
  ok &= run_test<int64_t>(30'000, 1, 1, communicator);
  ok &= run_test<int64_t>(300'000, 1, 1, communicator);
  ok &= run_test<int64_t>(300'000, 4, 1, communicator);
  ok &= run_test<int64_t>(3'000'000, 1, world, communicator);
  ok &= run_test<int64_t>(3'000'000, 4, world, communicator);
  ok &= run_test<int64_t>(3'000'000, 4, 2, communicator);
  destroy_memory_pool_and_communicator(communicator, registered_mr, pool_mr, "NCCL", "none");
  dj_bootstrap::finalize();
  if (!ok) return 1;
  if (dj_bootstrap::rank() == 0) std::cerr << "Test case \"compare_against_analytical\" passes successfully." << std::endl;
  return 0;
}
