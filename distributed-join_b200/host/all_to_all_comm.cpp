#include "all_to_all_comm.hpp"

#include <chrono>
#include <iostream>
#include <numeric>
#include <stdexcept>

#include "error.hpp"

using std::vector;

void communicate_sizes(vector<int64_t> const& send_offset, vector<int64_t>& recv_offset,
                       CommunicationGroup comm_group, Communicator* communicator)
{
  // Every rank publishes its per-destination counts for the group it is in; one all-gather
  // replaces the reference's N MPI_Isend/Irecv pairs (src/all_to_all_comm.cpp:54-100).  Rows of
  // other groups ride along unused (at most mpi_size * group_size int64).
  const int g = comm_group.size();
  vector<int64_t> mine(g), all((size_t)communicator->mpi_size * g);
  for (int i = 0; i < g; i++) mine[i] = send_offset[i + 1] - send_offset[i];
  communicator->allgather_i64(mine.data(), g, all.data());
  const int me = comm_group.get_local_idx();
  recv_offset.assign(g + 1, 0);
  for (int i = 0; i < g; i++)
    recv_offset[i + 1] = recv_offset[i] + all[(size_t)comm_group.get_global_rank(i) * g + me];
}

void communicate_sizes(vector<cudf::size_type> const& send_offset, vector<int64_t>& recv_offset,
                       CommunicationGroup comm_group, Communicator* communicator)
{
  communicate_sizes(vector<int64_t>(send_offset.begin(), send_offset.end()), recv_offset, comm_group,
                    communicator);
}

void warmup_all_to_all(Communicator* communicator)
{
  // one small exchange with every peer so that NCCL sets its channels up outside timed regions
  const int n = communicator->mpi_size, me = communicator->mpi_rank;
  const int64_t elems = 1 << 16;
  rmm::device_buffer send((size_t)elems * n * 8), recv((size_t)elems * n * 8);
  communicator->start();
  for (int r = 0; r < n; r++) {
    if (r == me) continue;
    communicator->send((char*)send.data() + (size_t)r * elems * 8, elems, 8, r);
    communicator->recv((char*)recv.data() + (size_t)r * elems * 8, elems, 8, r);
  }
  communicator->stop();
}

void append_to_all_to_all_comm_buffers(cudf::table_view input, cudf::mutable_table_view output,
                                       vector<cudf::size_type> const& send_offsets,
                                       vector<int64_t> const& recv_offsets,
                                       vector<AllToAllCommBuffer>& buffers,
                                       vector<ColumnCompressionOptions> compression_options)
{
  if (input.num_columns() != output.num_columns())
    throw std::runtime_error("all-to-all: input and output tables have different column counts");
  const vector<int64_t> send64(send_offsets.begin(), send_offsets.end());
  for (cudf::size_type c = 0; c < input.num_columns(); c++) {
    const cudf::data_type dtype = input.column(c).type();
    if (!cudf::is_fixed_width(dtype))
      throw std::runtime_error("all-to-all: only fixed-width columns are supported by this build");
    if ((size_t)c < compression_options.size() &&
        compression_options[c].compression_method != CompressionMethod::none)
      throw std::runtime_error("all-to-all: compression is not supported by this build");
    buffers.emplace_back(input.column(c).head(), output.column(c).head(), send64, recv_offsets, dtype);
  }
}

static void exchange_one_buffer(AllToAllCommBuffer& b, CommunicationGroup const& group,
                                Communicator* communicator, bool include_current_rank)
{
  const int g = group.size(), me = group.get_local_idx();
  const int es = (int)cudf::size_of(b.dtype);
  for (int i = 0; i < g; i++) {
    if (i == me) {
      if (include_current_rank) {
        // the reference sends to itself through the communicator; a stream-ordered copy on the
        // same rank is the NVLink-free equivalent
        const int64_t n = b.send_offsets[i + 1] - b.send_offsets[i];
        if (n > 0)
          CUDA_RT_CALL(cudaMemcpyAsync((char*)b.recv_buffer + b.recv_offsets[i] * es,
                                       (const char*)b.send_buffer + b.send_offsets[i] * es, (size_t)n * es,
                                       cudaMemcpyDeviceToDevice, nullptr));
      }
      continue;
    }
    const int peer = group.get_global_rank(i);
    communicator->send((const char*)b.send_buffer + b.send_offsets[i] * es,
                       b.send_offsets[i + 1] - b.send_offsets[i], es, peer);
    communicator->recv((char*)b.recv_buffer + b.recv_offsets[i] * es,
                       b.recv_offsets[i + 1] - b.recv_offsets[i], es, peer);
  }
}

void all_to_all_comm(vector<AllToAllCommBuffer>& buffers, CommunicationGroup comm_group,
                     Communicator* communicator, bool include_current_rank, bool, void*)
{
  for (auto& b : buffers) {
    assert((int)b.send_offsets.size() == comm_group.size() + 1);
    if (!communicator->group_by_batch()) communicator->start();
    exchange_one_buffer(b, comm_group, communicator, include_current_rank);
    if (!communicator->group_by_batch()) communicator->stop();
  }
  if (include_current_rank) CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
}

void postprocess_all_to_all_comm(vector<AllToAllCommBuffer>&, CommunicationGroup, Communicator*, bool, bool) {}

AllToAllCommunicator::AllToAllCommunicator(cudf::table_view input_table, vector<cudf::size_type> offsets,
                                           CommunicationGroup comm_group, Communicator* communicator,
                                           vector<ColumnCompressionOptions> compression_options,
                                           bool explicit_copy_to_current_rank)
  : input_table(input_table), comm_group(comm_group), communicator(communicator),
    explicit_copy_to_current_rank(explicit_copy_to_current_rank), send_offsets(std::move(offsets)),
    compression_options(std::move(compression_options))
{
  if ((int)send_offsets.size() != comm_group.size() + 1)
    throw std::runtime_error("AllToAllCommunicator: offsets must have group size + 1 entries");
  communicate_sizes(send_offsets, recv_offsets, comm_group, communicator);
}

AllToAllCommunicator::AllToAllCommunicator(cudf::table_view input_table, vector<cudf::size_type> offsets,
                                           Communicator* communicator,
                                           vector<ColumnCompressionOptions> compression_options,
                                           bool explicit_copy_to_current_rank)
  : AllToAllCommunicator(input_table, std::move(offsets), CommunicationGroup(communicator->mpi_size, 1),
                         communicator, std::move(compression_options), explicit_copy_to_current_rank)
{
}

std::unique_ptr<cudf::table> AllToAllCommunicator::allocate_communicated_table()
{
  vector<std::unique_ptr<cudf::column>> cols;
  const int64_t rows = recv_offsets.back();
  if (rows > INT32_MAX) throw std::runtime_error("received table exceeds cudf::size_type rows");
  for (cudf::size_type c = 0; c < input_table.num_columns(); c++)
    cols.push_back(cudf::make_fixed_width_column(input_table.column(c).type(), (cudf::size_type)rows));
  auto out = std::make_unique<cudf::table>(std::move(cols));
  if (explicit_copy_to_current_rank) {
    // own partition lands now, so it cannot queue behind a join kernel later
    // (same reasoning as src/all_to_all_comm.cpp:711-714)
    const int me = comm_group.get_local_idx();
    auto mv      = out->mutable_view();
    for (cudf::size_type c = 0; c < input_table.num_columns(); c++) {
      const size_t es = cudf::size_of(input_table.column(c).type());
      const int64_t n = recv_offsets[me + 1] - recv_offsets[me];
      if (n > 0)
        CUDA_RT_CALL(cudaMemcpyAsync(mv.column(c).head<char>() + recv_offsets[me] * es,
                                     input_table.column(c).head<char>() + (int64_t)send_offsets[me] * es,
                                     (size_t)n * es, cudaMemcpyDeviceToDevice, nullptr));
    }
  }
  CUDA_RT_CALL(cudaStreamSynchronize(nullptr));
  return out;
}

void AllToAllCommunicator::launch_communication(cudf::mutable_table_view communicated_table, bool report_timing,
                                                void* preallocated_pinned_buffer)
{
  vector<AllToAllCommBuffer> buffers;
  append_to_all_to_all_comm_buffers(input_table, communicated_table, send_offsets, recv_offsets, buffers,
                                    compression_options);
  if (auto* nc = dynamic_cast<NCCLCommunicator*>(communicator)) {
    // NCCL backend: the whole table -- every column, every peer -- is ONE library call
    // (dj_all_to_all: a single ncclGroup of sends/receives straight between the final buffers)
    const int g = comm_group.size(), me = comm_group.get_local_idx();
    vector<int> ranks(g), elem_sizes;
    for (int i = 0; i < g; i++) ranks[i] = comm_group.get_global_rank(i);
    vector<const void*> send_cols;
    vector<void*> recv_cols;
    for (auto& b : buffers) {
      send_cols.push_back(b.send_buffer);
      recv_cols.push_back(b.recv_buffer);
      elem_sizes.push_back((int)cudf::size_of(b.dtype));
    }
    const vector<int64_t> send64(send_offsets.begin(), send_offsets.end());
    DJ_CALL(dj_all_to_all(nc->comm, g, ranks.data(), me, send_cols.data(), recv_cols.data(), send64.data(),
                          recv_offsets.data(), elem_sizes.data(), (int)buffers.size(),
                          explicit_copy_to_current_rank ? 0 : 1, nc->comm_stream));
    CUDA_RT_CALL(cudaStreamSynchronize(nc->comm_stream));
    return;
  }
  if (communicator->group_by_batch()) communicator->start();
  all_to_all_comm(buffers, comm_group, communicator, !explicit_copy_to_current_rank, report_timing,
                  preallocated_pinned_buffer);
  if (communicator->group_by_batch()) communicator->stop();
  postprocess_all_to_all_comm(buffers, comm_group, communicator, !explicit_copy_to_current_rank, report_timing);
}
