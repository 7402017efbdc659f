// TEST INFRASTRUCTURE ONLY.
//
// Host program that EXECUTES the reference-side binding include/B200ModBaseModel.h: compiled against the reference's own
// headers (ModBaseModelConfig, torch_utils) and libtorch, as the header would be inside dorado, it loads the model the way
// load_modbase_model does -- config::load_modbase_model_config, then the *.tensor files through utils::load_tensors --
// wraps the module in the reference's ModuleWrapper and runs forward(sigs_N1T, seqs_NTC) once.
// Built where the reference tree exists by oracle/modbase_ref.mk into oracle/_ref/modbase_host; run on the GPU box by
// tests/test_modbase_gpu.py, which compares its output with the ctypes path on the same chunks.
//
// usage: modbase_host <model dir> <batch> <num chunks> <signal.f16> <kmers.i8> <out.f16>
//   model dir: config.toml and the *.tensor files; signal [n][chunk_size] fp16; kmers [n][T_seq][kmer_len * 4] int8
#include "B200ModBaseModel.h"

#include "config/ModBaseModelConfig.h"
#include "torch_utils/module_utils.h"

#include <torch/torch.h>

#include <cstdio>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

namespace {

std::vector<char> read_file(const std::string& path, size_t bytes) {
    std::ifstream f(path, std::ios::binary);
    std::vector<char> v(bytes);
    f.read(v.data(), static_cast<std::streamsize>(bytes));
    if (!f) throw std::runtime_error("cannot read " + std::to_string(bytes) + " bytes from " + path);
    return v;
}

}  // namespace

int main(int argc, char** argv) {
    if (argc != 7) {
        std::fprintf(stderr, "usage: %s <model dir> <batch> <num chunks> <signal.f16> <kmers.i8> <out.f16>\n", argv[0]);
        return 2;
    }
    try {
        at::InferenceMode guard;
        const auto config = dorado::config::load_modbase_model_config(argv[1]);
        const int batch = std::stoi(argv[2]), n = std::stoi(argv[3]);
        const auto [T_seq, C_seq] = config.chunked_sequence_input_TC();
        const int64_t T = config.context.chunk_size;
        auto sig_bytes = read_file(argv[4], size_t(n) * T * 2);
        auto seq_bytes = read_file(argv[5], size_t(n) * T_seq * C_seq);
        const at::Tensor sigs = at::from_blob(sig_bytes.data(), {n, 1, T}, at::kHalf);
        const at::Tensor seqs = at::from_blob(seq_bytes.data(), {n, T_seq, C_seq}, at::kChar);

        auto model = dorado::modbase::model::B200ModBaseModel(config, batch, 0);
        dorado::utils::ModuleWrapper module{torch::nn::ModuleHolder<torch::nn::AnyModule>{torch::nn::AnyModule(model)}};
        const at::Tensor out = module.forward(sigs, seqs).to(at::kCPU).contiguous();
        if (out.scalar_type() != at::kHalf || out.size(0) != n) throw std::runtime_error("unexpected output tensor");
        std::ofstream f(argv[6], std::ios::binary);
        f.write(static_cast<const char*>(out.data_ptr()), static_cast<std::streamsize>(out.numel() * 2));
        std::cout << "modbase_host: " << n << " chunks -> [" << out.size(0) << ", " << out.size(1) << "] fp16\n";
        return f ? 0 : 1;
    } catch (const std::exception& e) {
        std::cerr << "modbase_host: " << e.what() << "\n";
        return 1;
    }
}
