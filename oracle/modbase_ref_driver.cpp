// TEST INFRASTRUCTURE ONLY -- never linked into or called by the product path.
//
// C-ABI shim around the *unmodified* reference modified-base model code, compiled in place from the reference tree by
// oracle/modbase_ref.mk into oracle/_ref/libmodbase_ref.so (next to libdorado_ref.so, which provides the conv, LSTM and
// upsample modules it is built on):
//   * config     dorado/config/ModBaseModelConfig.cpp  (load_modbase_model_config and its checks)
//   * forward    dorado/modbase/nn/ModBaseModel.cpp    (load_modbase_model -> ModBaseConvLSTMV3Model on the CPU, fp32)
// Everything here is glue written for this repo; no reference source is copied.
#include "config/ModBaseModelConfig.h"
#include "modbase/nn/ModBaseModel.h"

#include <ATen/ATen.h>
#include <torch/serialize.h>
#include <torch/torch.h>

#include <algorithm>
#include <cctype>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace {

thread_local std::string g_err;

template <typename F>
int guarded(F&& fn) {
    try {
        at::InferenceMode guard;
        fn();
        return 0;
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
}

struct RefModBase {
    std::unique_ptr<dorado::config::ModBaseModelConfig> config;
    dorado::utils::ModuleWrapper module;
};

void put_conv(std::vector<int>& v, const dorado::config::ConvParams& c) {
    v.insert(v.end(), {c.insize, c.size, c.winlen, c.stride, int(c.activation)});
}

}  // namespace

// ModBaseModelConfig.cpp validates each modification code with this function of hts_utils/bam_utils.cpp, which needs
// htslib and is not built here.  The rule is the SAM specification's for the MM tag: a code is one letter or a ChEBI id
// (decimal digits).
namespace dorado::utils {
bool validate_bam_tag_code(const std::string& code) {
    if (code.size() == 1 && std::isalpha(static_cast<unsigned char>(code[0]))) return true;
    return !code.empty() && std::all_of(code.begin(), code.end(), [](char ch) { return std::isdigit(static_cast<unsigned char>(ch)) != 0; });
}
}  // namespace dorado::utils

extern "C" {

const char* ref_modbase_last_error() { return g_err.c_str(); }

// One weight file as the reference's load_tensors reads it (torch::load of a tensor vector), fp32.
int ref_modbase_save_tensor(const char* path, const float* data, int ndim, const int64_t* dims) {
    return guarded([&] {
        std::vector<int64_t> shape(dims, dims + ndim);
        at::Tensor t = at::from_blob(const_cast<float*>(data), shape, at::kFloat).clone();
        torch::save(std::vector<at::Tensor>{t}, std::string(path));
    });
}

// load_modbase_model_config(dir), flattened into `out` (capacity `cap`, *n = count):
//   model_type, size, kmer_len, num_out, stride, sequence_stride,
//   3 signal convs, 2 sequence convs, the merge conv (insize, size, winlen, stride, activation each),
//   number of LSTMs, (size, reverse) per LSTM, linear (in, out), upsample (size, scale_factor; -1 -1 if none),
//   samples_before, samples_after, chunk_size, bases_before, bases_after, context kmer_len, reverse, base_start_justify,
//   refine do_rough_rescale, center_idx, number of mods, motif_offset, motif base,
//   chunked_sequence_input_TC (T, C), chunked_signal_input_TC (T, C), chunked_output_TC (T, C)
int ref_modbase_config(const char* dir, int* out, int cap, int* n) {
    return guarded([&] {
        const auto c = dorado::config::load_modbase_model_config(dir);
        const auto& g = c.general;
        std::vector<int> v{int(g.model_type), g.size, g.kmer_len, g.num_out, g.stride, g.sequence_stride};
        const auto& m = g.modules.value();
        if (m.signal_convs.size() != 3 || m.sequence_convs.size() != 2) throw std::runtime_error("unexpected conv count");
        for (const auto& cv : m.signal_convs) put_conv(v, cv);
        for (const auto& cv : m.sequence_convs) put_conv(v, cv);
        put_conv(v, m.merge_conv);
        v.push_back(int(m.lstms.size()));
        for (const auto& l : m.lstms) v.insert(v.end(), {l.size, int(l.reverse)});
        v.insert(v.end(), {m.linear.in_size, m.linear.out_size});
        if (m.upsample.has_value()) v.insert(v.end(), {m.upsample->size, m.upsample->scale_factor});
        else v.insert(v.end(), {-1, -1});
        const auto& x = c.context;
        v.insert(v.end(), {int(x.samples_before), int(x.samples_after), int(x.chunk_size), x.bases_before, x.bases_after,
                           x.kmer_len, int(x.reverse), int(x.base_start_justify)});
        v.insert(v.end(), {int(c.refine.do_rough_rescale), int(c.refine.center_idx), int(c.mods.count),
                           int(c.mods.motif_offset), int(c.mods.base)});
        const auto [sT, sC] = c.chunked_sequence_input_TC();
        const auto [gT, gC] = c.chunked_signal_input_TC();
        const auto [oT, oC] = c.chunked_output_TC();
        v.insert(v.end(), {int(sT), int(sC), int(gT), int(gC), int(oT), int(oC)});
        if ((int)v.size() > cap) throw std::runtime_error("ref_modbase_config: output too small");
        std::memcpy(out, v.data(), v.size() * sizeof(int));
        *n = (int)v.size();
    });
}

// dir: config.toml and the *.tensor files load_modbase_conv_lstm_weights names.  The model on the CPU in fp32.
void* ref_modbase_create(const char* dir) {
    RefModBase* m = nullptr;
    const int rc = guarded([&] {
        auto owned = std::make_unique<RefModBase>();
        owned->config = std::make_unique<dorado::config::ModBaseModelConfig>(dorado::config::load_modbase_model_config(dir));
        const auto opts = at::TensorOptions().dtype(at::kFloat).device(at::kCPU);
        owned->module = dorado::modbase::load_modbase_model(*owned->config, opts, 1);
        m = owned.release();
    });
    return rc == 0 ? m : nullptr;
}

void ref_modbase_destroy(void* h) { delete static_cast<RefModBase*>(h); }

// sig [N][T] fp32, seq [N][T_seq][C_seq] int8 -> the forward's output [N][*out_elems] fp32 (out may be null to ask the size)
int ref_modbase_forward(void* h, const float* sig, int N, int T, const int8_t* seq, int T_seq, int C_seq, float* out,
                        int* out_elems) {
    auto* m = static_cast<RefModBase*>(h);
    return guarded([&] {
        at::Tensor s = at::from_blob(const_cast<float*>(sig), {N, 1, T}, at::kFloat).clone();
        at::Tensor q = at::from_blob(const_cast<int8_t*>(seq), {N, T_seq, C_seq}, at::kChar).clone();
        at::Tensor y = m->module.forward(s, q).contiguous();
        *out_elems = int(y.size(1));
        if (out) std::memcpy(out, y.data_ptr<float>(), size_t(y.numel()) * 4);
    });
}

}  // extern "C"
