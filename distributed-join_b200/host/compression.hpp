// compression.hpp -- signature-compatible placeholder for the reference's nvcomp options
// (src/compression.hpp:45-58, src/compression.cpp:75-95).  Compression is out of scope: nvcomp
// is not a dependency, the benchmark default is off (benchmark/distributed_join.cu:107) and at
// H100 NVLink rates (450 GB/s per direction) it costs more than it saves.  Only `none` exists.
#pragma once

#include <stdexcept>
#include <vector>

#include "cudf_shim.hpp"

enum class CompressionMethod { none };

struct ColumnCompressionOptions {
  CompressionMethod compression_method = CompressionMethod::none;
};

inline std::vector<ColumnCompressionOptions> generate_none_compression_options(cudf::table_view input_table)
{
  return std::vector<ColumnCompressionOptions>((std::size_t)input_table.num_columns());
}

inline std::vector<ColumnCompressionOptions> generate_compression_options_distributed(
  cudf::table_view input_table, bool compression)
{
  if (compression)
    throw std::runtime_error("compression is not supported by this build (over NVLink it costs more than it saves)");
  return generate_none_compression_options(input_table);
}

inline void warmup_nvcomp() {}
