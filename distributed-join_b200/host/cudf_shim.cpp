#include "cudf_shim.hpp"

#include <algorithm>
#include <string>

namespace cudf {

namespace {
void require_fixed_width(table_view const& t, const char* what)
{
  for (auto const& c : t)
    if (!is_fixed_width(c.type()))
      throw std::runtime_error(std::string(what) + ": this build handles fixed-width columns only");
}

__global__ void widen_kernel(const int32_t* in, int64_t* out, int64_t n)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = in[i];
}
__global__ void narrow_kernel(const int64_t* in, int32_t* out, int64_t n)
{
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int32_t)in[i];
}
int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, 132 * 16)); }
}  // namespace

bool all_i64(table_view const& t)
{
  for (auto const& c : t)
    if (size_of(c.type()) != 8) return false;
  return true;
}

std::unique_ptr<table> widen_to_i64(table_view const& t)
{
  require_fixed_width(t, "widen");
  std::vector<std::unique_ptr<column>> cols;
  const int64_t n = t.num_rows();
  for (auto const& c : t) {
    cols.push_back(make_fixed_width_column(data_type(type_id::INT64), (size_type)n));
    if (n == 0) continue;
    if (size_of(c.type()) == 8)
      CUDA_RT_CALL(cudaMemcpyAsync(cols.back()->mutable_view().head(), c.head(), (size_t)n * 8,
                                   cudaMemcpyDeviceToDevice, nullptr));
    else
      widen_kernel<<<grid_for(n), 256>>>(c.head<int32_t>(), cols.back()->mutable_view().head<int64_t>(), n);
  }
  CUDA_RT_CALL(cudaGetLastError());
  return std::make_unique<table>(std::move(cols));
}

std::unique_ptr<table> narrow_like(table_view const& t, std::vector<data_type> const& types)
{
  if ((size_t)t.num_columns() != types.size()) throw std::runtime_error("narrow_like: column count mismatch");
  std::vector<std::unique_ptr<column>> cols;
  const int64_t n = t.num_rows();
  for (size_type c = 0; c < t.num_columns(); c++) {
    cols.push_back(make_fixed_width_column(types[c], (size_type)n));
    if (n == 0) continue;
    if (size_of(types[c]) == 8)
      CUDA_RT_CALL(cudaMemcpyAsync(cols.back()->mutable_view().head(), t.column(c).head(), (size_t)n * 8,
                                   cudaMemcpyDeviceToDevice, nullptr));
    else
      narrow_kernel<<<grid_for(n), 256>>>(t.column(c).head<int64_t>(), cols.back()->mutable_view().head<int32_t>(), n);
  }
  CUDA_RT_CALL(cudaGetLastError());
  return std::make_unique<table>(std::move(cols));
}

std::pair<std::unique_ptr<table>, std::vector<size_type>> hash_partition(
  table_view const& input, std::vector<size_type> const& columns_to_hash, int num_partitions, hash_id hash_function,
  uint32_t seed)
{
  if (columns_to_hash.size() != 1) throw std::runtime_error("hash_partition: exactly one key column is supported");
  if (input.num_columns() < 2 || input.num_columns() > 4)
    throw std::runtime_error("hash_partition: 2..4 columns (key + 1..3 payload columns) are supported");
  require_fixed_width(input, "hash_partition");
  if (!all_i64(input)) {
    std::vector<data_type> types;
    for (auto const& c : input) types.push_back(c.type());
    auto wide   = widen_to_i64(input);
    auto result = hash_partition(wide->view(), columns_to_hash, num_partitions, hash_function, seed);
    return {narrow_like(result.first->view(), types), std::move(result.second)};
  }
  const size_type n   = input.num_rows();
  const size_type key = columns_to_hash[0];

  std::vector<std::unique_ptr<column>> out_cols;
  for (size_type c = 0; c < input.num_columns(); c++)
    out_cols.push_back(make_fixed_width_column(data_type(type_id::INT64), n));
  std::vector<const int64_t*> in_pay;
  std::vector<int64_t*> out_pay;
  for (size_type c = 0; c < input.num_columns(); c++) {
    if (c == key) continue;
    in_pay.push_back(input.column(c).head<int64_t>());
    out_pay.push_back(out_cols[c]->mutable_view().head<int64_t>());
  }
  rmm::device_buffer d_offsets(((size_t)num_partitions + 1) * 8);
  const size_t ws_bytes = dj_hash_partition_workspace_bytes(n, num_partitions);
  rmm::device_buffer ws(ws_bytes);
  DJ_CALL(dj_hash_partition_i64(input.column(key).head<int64_t>(), in_pay.data(), (int)in_pay.size(), n,
                                num_partitions, seed, (int)hash_function,
                                out_cols[key]->mutable_view().head<int64_t>(), out_pay.data(),
                                (int64_t*)d_offsets.data(), ws.data(), ws_bytes, nullptr));
  std::vector<int64_t> off64((size_t)num_partitions + 1);
  CUDA_RT_CALL(cudaMemcpyAsync(off64.data(), d_offsets.data(), off64.size() * 8, cudaMemcpyDeviceToHost, nullptr));
  CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
  // cuDF returns the num_partitions start offsets; callers append num_rows themselves
  std::vector<size_type> offsets(off64.begin(), off64.end() - 1);
  return {std::make_unique<table>(std::move(out_cols)), std::move(offsets)};
}

std::unique_ptr<table> inner_join(table_view const& left, table_view const& right,
                                  std::vector<size_type> const& left_on, std::vector<size_type> const& right_on)
{
  if (left_on.size() != 1 || right_on.size() != 1 || left.num_columns() != 2 || right.num_columns() != 2)
    throw std::runtime_error("inner_join: one key column and one payload column per side are supported");
  require_fixed_width(left, "inner_join");
  require_fixed_width(right, "inner_join");
  if (!all_i64(left) || !all_i64(right)) {
    std::vector<data_type> types;
    for (auto const& c : left) types.push_back(c.type());
    for (auto const& c : right) types.push_back(c.type());
    auto wl = widen_to_i64(left), wr = widen_to_i64(right);
    auto joined = inner_join(wl->view(), wr->view(), left_on, right_on);
    return narrow_like(joined->view(), types);
  }
  const size_type lk = left_on[0], rk = right_on[0];
  const int64_t nl = left.num_rows(), nr = right.num_rows();
  // build on the smaller side; the output stays left columns ++ right columns
  const bool build_left = nl <= nr;
  table_view const& B = build_left ? left : right;
  table_view const& P = build_left ? right : left;
  const size_type bk = build_left ? lk : rk, pk = build_left ? rk : lk;
  const size_t ws_bytes = dj_inner_join_workspace_bytes(B.num_rows(), P.num_rows());
  rmm::device_buffer ws(ws_bytes), d_count(8);
  int64_t capacity = std::max<int64_t>(std::max(nl, nr), 1);
  for (;;) {
    std::vector<std::unique_ptr<column>> cols;
    for (int c = 0; c < 4; c++) cols.push_back(make_fixed_width_column(data_type(type_id::INT64), (size_type)capacity));
    // output column order of the join kernel is (build key, build payload, probe key, probe payload)
    int64_t* o[4];
    for (int c = 0; c < 4; c++) o[c] = cols[c]->mutable_view().head<int64_t>();
    int64_t* bo_k = build_left ? o[lk] : o[2 + rk];
    int64_t* bo_p = build_left ? o[1 - lk] : o[2 + 1 - rk];
    int64_t* po_k = build_left ? o[2 + rk] : o[lk];
    int64_t* po_p = build_left ? o[2 + 1 - rk] : o[1 - lk];
    DJ_CALL(dj_inner_join_i64(B.column(bk).head<int64_t>(), B.column(1 - bk).head<int64_t>(), B.num_rows(),
                              P.column(pk).head<int64_t>(), P.column(1 - pk).head<int64_t>(), P.num_rows(), bo_k,
                              bo_p, po_k, po_p, capacity, (int64_t*)d_count.data(), ws.data(), ws_bytes, nullptr));
    int64_t n_out = 0;
    CUDA_RT_CALL(cudaMemcpyAsync(&n_out, d_count.data(), 8, cudaMemcpyDeviceToHost, nullptr));
    CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
    if (n_out <= capacity) {
      for (auto& c : cols) c->set_size((size_type)n_out);
      return std::make_unique<table>(std::move(cols));
    }
    if (n_out > INT32_MAX) throw std::runtime_error("inner_join: result exceeds cudf::size_type rows");
    capacity = n_out;  // exact retry
  }
}

std::unique_ptr<table> concatenate(std::vector<table_view> const& views)
{
  if (views.empty()) return std::make_unique<table>();
  size_type ncols = 0;
  int64_t rows    = 0;
  for (auto const& v : views) {
    if (v.num_columns() > ncols) ncols = v.num_columns();
    rows += v.num_rows();
  }
  if (rows > INT32_MAX) throw std::runtime_error("concatenate: result exceeds cudf::size_type rows");
  std::vector<std::unique_ptr<column>> cols;
  for (size_type c = 0; c < ncols; c++) {
    data_type t(type_id::INT64);
    for (auto const& v : views)
      if (v.num_columns() == ncols) t = v.column(c).type();
    cols.push_back(make_fixed_width_column(t, (size_type)rows));
    int64_t at      = 0;
    const size_t es = size_of(t);
    for (auto const& v : views) {
      if (v.num_columns() != ncols || v.num_rows() == 0) continue;  // empty batch results have no columns
      CUDA_RT_CALL(cudaMemcpyAsync(cols.back()->mutable_view().head<char>() + at * es, v.column(c).head<char>(),
                                   (size_t)v.num_rows() * es, cudaMemcpyDeviceToDevice, nullptr));
      at += v.num_rows();
    }
  }
  CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
  return std::make_unique<table>(std::move(cols));
}

}  // namespace cudf
