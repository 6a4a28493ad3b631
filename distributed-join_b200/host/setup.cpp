#include "setup.hpp"

#include <cstdlib>
#include <iostream>
#include <stdexcept>

#include "bootstrap.hpp"
#include "error.hpp"

void set_cuda_device()
{
  // one rank per GPU; LOCAL_RANK (torchrun) wins over rank % device_count (src/setup.cpp:35-49)
  int device_count = 0;
  CUDA_RT_CALL(cudaGetDeviceCount(&device_count));
  const char* local = std::getenv("LOCAL_RANK");
  const int rank    = dj_bootstrap::rank();
  const int device  = (local ? std::atoi(local) : rank) % device_count;
  CUDA_RT_CALL(cudaSetDevice(device));
  std::cout << "Rank " << rank << " select " << device << "/" << device_count << " GPU" << std::endl;
}

void setup_memory_pool_and_communicator(
  Communicator*& communicator, registered_memory_resource*& registered_mr,
  rmm::mr::pool_memory_resource<rmm::mr::device_memory_resource>*& pool_mr, std::string communicator_name,
  std::string, int64_t)
{
  registered_mr = nullptr;
  if (communicator_name != "NCCL")
    throw std::runtime_error("Unknown communicator name (this build provides \"NCCL\" only; UCX is out of scope)");
  size_t free_memory = 0, total_memory = 0;
  CUDA_RT_CALL(cudaMemGetInfo(&free_memory, &total_memory));
  const size_t pool_size = free_memory / 284 * 256;  // same sizing rule as src/setup.cpp:64
  communicator           = new NCCLCommunicator;
  communicator->initialize();
  pool_mr = new rmm::mr::pool_memory_resource<rmm::mr::device_memory_resource>(
    rmm::mr::get_current_device_resource(), pool_size, pool_size);
  rmm::mr::set_current_device_resource(pool_mr);
}

void destroy_memory_pool_and_communicator(
  Communicator* communicator, registered_memory_resource*,
  rmm::mr::pool_memory_resource<rmm::mr::device_memory_resource>* pool_mr, std::string, std::string)
{
  communicator->finalize();
  delete communicator;
  rmm::mr::set_current_device_resource(pool_mr ? pool_mr->get_upstream() : nullptr);
  delete pool_mr;
}
