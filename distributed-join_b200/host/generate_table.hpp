// generate_table.hpp -- the benchmark's input generators with the reference's signatures
// (src/generate_table.cuh:75-124,155-272) on top of libdj_b200's counter-based generator.
// Every row is a closed-form function of (source rank, row), so the distributed wrapper builds
// what each rank would have RECEIVED from the reference's equal-chunk all-to-all (:209-269)
// without communicating.  INT64 keys and payloads.
#pragma once

#include <memory>
#include <stdexcept>
#include <type_traits>
#include <utility>

#include "communicator.hpp"
#include "cudf_shim.hpp"
#include "error.hpp"

namespace dj_detail {
inline std::unique_ptr<cudf::table> make_two_column_table(int64_t rows)
{
  std::vector<std::unique_ptr<cudf::column>> cols;
  cols.push_back(cudf::make_numeric_column(cudf::data_type(cudf::type_id::INT64), (cudf::size_type)rows));
  cols.push_back(cudf::make_numeric_column(cudf::data_type(cudf::type_id::INT64), (cudf::size_type)rows));
  return std::make_unique<cudf::table>(std::move(cols));
}
}  // namespace dj_detail

// Local (single rank) build and probe tables: key column + payload column (= row id).
template <typename KEY_T, typename PAYLOAD_T>
std::pair<std::unique_ptr<cudf::table>, std::unique_ptr<cudf::table>> generate_build_probe_tables(
  cudf::size_type build_table_nrows, cudf::size_type probe_table_nrows, double selectivity, KEY_T rand_max,
  bool uniq_build_tbl_keys, int src_rank = 0, int64_t row_begin_build = 0, int64_t row_begin_probe = 0,
  int64_t nb_total = -1, int64_t np_total = -1)
{
  static_assert(std::is_same<KEY_T, int64_t>::value && std::is_same<PAYLOAD_T, int64_t>::value,
                "this build generates int64 keys and payloads");
  dj_gen_params g{};
  g.nb                = nb_total < 0 ? build_table_nrows : nb_total;
  g.np                = np_total < 0 ? probe_table_nrows : np_total;
  g.rand_max          = rand_max;
  g.selectivity       = selectivity;
  g.seed              = 1234;  // generate_dataset/generate_dataset.cuh:44
  g.unique_build_keys = uniq_build_tbl_keys ? 1 : 0;
  auto build = dj_detail::make_two_column_table(build_table_nrows);
  auto probe = dj_detail::make_two_column_table(probe_table_nrows);
  rmm::device_buffer bitmap;
  if (!uniq_build_tbl_keys) {
    bitmap = rmm::device_buffer((size_t)((rand_max + 1 + 31) / 32) * 4);
    DJ_CALL(dj_generate_build_bitmap(&g, src_rank, (uint32_t*)bitmap.data(), nullptr));
  }
  auto bv = build->mutable_view();
  auto pv = probe->mutable_view();
  DJ_CALL(dj_generate_rows_i64(&g, 0, src_rank, row_begin_build, build_table_nrows, nullptr,
                               bv.column(0).head<int64_t>(), bv.column(1).head<int64_t>(), nullptr));
  DJ_CALL(dj_generate_rows_i64(&g, 1, src_rank, row_begin_probe, probe_table_nrows, (const uint32_t*)bitmap.data(),
                               pv.column(0).head<int64_t>(), pv.column(1).head<int64_t>(), nullptr));
  CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
  return {std::move(build), std::move(probe)};
}

// Distributed tables: keys of source rank r live in [r*rand_max, (r+1)*rand_max], payloads are
// global row ids, and every rank ends up with rows [n/N*rank, n/N*(rank+1)) of every source.
template <typename KEY_T, typename PAYLOAD_T>
std::pair<std::unique_ptr<cudf::table>, std::unique_ptr<cudf::table>> generate_tables_distributed(
  cudf::size_type build_table_nrows_per_rank, cudf::size_type probe_table_nrows_per_rank, double selectivity,
  KEY_T rand_max_per_rank, bool uniq_build_tbl_keys, Communicator* communicator)
{
  static_assert((std::is_same<KEY_T, int64_t>::value || std::is_same<KEY_T, int32_t>::value) &&
                  (std::is_same<PAYLOAD_T, int64_t>::value || std::is_same<PAYLOAD_T, int32_t>::value),
                "keys and payloads are int32_t or int64_t");
  const int world = communicator->mpi_size, rank = communicator->mpi_rank;
  const int64_t bchunk = build_table_nrows_per_rank / world, pchunk = probe_table_nrows_per_rank / world;
  dj_gen_params g{};
  g.nb                = build_table_nrows_per_rank;
  g.np                = probe_table_nrows_per_rank;
  g.rand_max          = rand_max_per_rank;
  g.selectivity       = selectivity;
  g.seed              = 1234;
  g.unique_build_keys = uniq_build_tbl_keys ? 1 : 0;
  auto build = dj_detail::make_two_column_table(bchunk * world);
  auto probe = dj_detail::make_two_column_table(pchunk * world);
  auto bv    = build->mutable_view();
  auto pv    = probe->mutable_view();
  rmm::device_buffer bitmap;
  if (!uniq_build_tbl_keys) bitmap = rmm::device_buffer((size_t)((rand_max_per_rank + 1 + 31) / 32) * 4);
  for (int src = 0; src < world; src++) {
    if (!uniq_build_tbl_keys) DJ_CALL(dj_generate_build_bitmap(&g, src, (uint32_t*)bitmap.data(), nullptr));
    DJ_CALL(dj_generate_rows_i64(&g, 0, src, bchunk * rank, bchunk, nullptr,
                                 bv.column(0).head<int64_t>() + src * bchunk,
                                 bv.column(1).head<int64_t>() + src * bchunk, nullptr));
    DJ_CALL(dj_generate_rows_i64(&g, 1, src, pchunk * rank, pchunk, (const uint32_t*)bitmap.data(),
                                 pv.column(0).head<int64_t>() + src * pchunk,
                                 pv.column(1).head<int64_t>() + src * pchunk, nullptr));
  }
  CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
  if (!std::is_same<KEY_T, int64_t>::value || !std::is_same<PAYLOAD_T, int64_t>::value) {
    // generated as int64, handed out in the requested widths (values fit: rand_max is a size_type)
    std::vector<cudf::data_type> types{cudf::data_type(cudf::type_to_id<KEY_T>()),
                                       cudf::data_type(cudf::type_to_id<PAYLOAD_T>())};
    build = cudf::narrow_like(build->view(), types);
    probe = cudf::narrow_like(probe->view(), types);
    CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
  }
  return {std::move(build), std::move(probe)};
}
