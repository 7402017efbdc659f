// Pre-computed batch-size timings: the counterpart of CudaChunkBenchmarks
// (dorado/basecall/benchmarks/CudaChunkBenchmarks.cpp:14-77 and the per-GPU tables next to it).  determine_batch_dims
// (CudaCaller.cpp:506-557) looks the (GPU name, model name) pair up before it falls back to timing every batch size at
// start-up.  Tables are produced on the GPU by tools/gen_chunk_benchmarks.py (forward + decode of one batch at the full
// chunk size, ms per chunk, only the batch sizes that improve on every smaller one, as the reference's generator keeps
// them); chunk_benchmarks_b200.inc holds what has been measured for this engine.
#include "engine.h"

#include <cstring>
#include <string>

namespace b200 {

namespace {

struct Timing {
    int batch_size;
    float ms_per_chunk;
};
struct Table {
    const char* gpu;
    const char* model;
    const Timing* rows;
    int count;
};

#include "chunk_benchmarks_b200.inc"

// GPUs that share a table (CudaChunkBenchmarks.cpp:39-46 keeps the same kind of alias list)
const char* canonical_gpu(const std::string& name) {
    if (name == "NVIDIA H100 80GB HBM3" || name == "NVIDIA H100 SXM5 80GB" || name == "NVIDIA H100") return "NVIDIA H100 80GB HBM3";
    return nullptr;
}

}  // namespace

int lookup_chunk_benchmarks(const char* gpu_name, const char* model_name, int32_t* batch_sizes, float* ms_per_chunk, int capacity) {
    if (!gpu_name || !model_name) throw std::invalid_argument("chunk benchmarks: null name");
    const char* gpu = canonical_gpu(gpu_name);
    if (!gpu) return 0;
    for (int k = 0; k < kNumTables; ++k) {
        const Table& t = kTables[k];
        if (std::strcmp(t.gpu, gpu) == 0 && std::strcmp(t.model, model_name) == 0) {
            for (int i = 0; i < t.count && i < capacity; ++i) {
                if (batch_sizes) batch_sizes[i] = t.rows[i].batch_size;
                if (ms_per_chunk) ms_per_chunk[i] = t.rows[i].ms_per_chunk;
            }
            return t.count;
        }
    }
    return 0;
}

std::string device_name(int device) {
    cudaDeviceProp prop{};
    B200_CUDA(cudaGetDeviceProperties(&prop, device));
    return prop.name;
}

}  // namespace b200
