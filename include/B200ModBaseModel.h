// B200ModBaseModel.h -- the reference-side binding of the modified-base engine: a torch module with the forward of
// ModBaseConvLSTMV3CUDAModel (dorado/modbase/nn/ModBaseModel.cpp:435-601) on top of the C ABI in b200call.h.
// Header-only; a dorado maintainer adds it under dorado/modbase/nn/ and constructs it in load_modbase_model's
// CONV_LSTM_V3 branch instead of the Koi model (ModBaseModel.cpp:630-637, see INTEGRATION.md).  libtorch is touched only
// at this edge (at::Tensor in and out, torch::load of the *.tensor weight files), never inside libb200call.so.
//
// Contract kept:
//   forward(sigs_N1T, seqs_NTC): signal [N, 1, chunk_size] (any float dtype, any device), k-mer one-hot
//   [N, T_seq, kmer_len * 4] int8  ->  fp16 [N, T_out * num_out] on the signal's device: the softmax over the classes
//   at every output step, flattened, as ModBaseCaller reads it (ModBaseCaller.cpp:125, 193).  N <= batch_size.
//   The weights are read from config.model_path in the order of load_modbase_conv_lstm_weights (ModBaseModel.cpp:49-75).
//   One module is one batch in flight (a runner of the engine); modules of one process share nothing but the GPU, and
//   errors throw std::runtime_error.
#pragma once

#include "b200call.h"

#include "config/ModBaseModelConfig.h"
#include "torch_utils/tensor_utils.h"

#include <ATen/ATen.h>
#include <torch/nn.h>

#include <stdexcept>
#include <string>
#include <vector>

namespace dorado::modbase::model {

struct B200ModBaseModelImpl : torch::nn::Module {
    B200ModBaseModelImpl(const config::ModBaseModelConfig& config, int batch_size, int device_index) : m_config(config) {
        if (config.general.model_type != config::ModelType::CONV_LSTM_V3 || !config.general.modules.has_value()) {
            throw std::runtime_error("B200ModBaseModel runs conv_lstm_v3 models only");
        }
        const auto& m = *config.general.modules;
        if (m.signal_convs.size() != 3 || m.sequence_convs.size() != 2 || m.lstms.size() != 2) {
            throw std::runtime_error("ModBaseConvLSTMV3Model expects 3 signal convolutions, 2 sequence convolutions and 2 lstms");
        }
        auto conv = [](const config::ConvParams& c) {
            return b200_conv_desc{c.insize, c.size, c.winlen, c.stride, static_cast<int32_t>(c.activation)};
        };
        b200_modbase_desc d{};
        for (int i = 0; i < 3; ++i) d.sig_convs[i] = conv(m.signal_convs[i]);
        for (int i = 0; i < 2; ++i) d.seq_convs[i] = conv(m.sequence_convs[i]);
        d.merge_conv = conv(m.merge_conv);
        d.lstm_size = m.lstms[0].size;
        d.num_out = config.general.num_out;
        d.upsample_scale = m.upsample.has_value() ? m.upsample->scale_factor : 0;
        d.kmer_len = config.general.kmer_len;
        d.chunk_size = static_cast<int32_t>(config.context.chunk_size);

        const auto names = tensor_names(config);
        const auto tensors = utils::load_tensors(config.model_path, names);
        if (tensors.size() != names.size()) throw std::runtime_error("B200ModBaseModel: unexpected number of weight tensors");
        std::vector<at::Tensor> keep;
        std::vector<b200_tensor> bt(tensors.size());
        for (size_t i = 0; i < tensors.size(); ++i) {
            keep.push_back(tensors[i].to(at::kCPU, at::kFloat).contiguous());
            bt[i].name = names[i].c_str();
            bt[i].data = keep.back().data_ptr<float>();
            bt[i].ndim = static_cast<int32_t>(keep.back().dim());
            for (int64_t k = 0; k < keep.back().dim() && k < 4; ++k) bt[i].dims[k] = keep.back().size(k);
        }
        check(b200_modbase_engine_create(&d, bt.data(), static_cast<int32_t>(bt.size()), device_index, &m_engine));
        const int rc = b200_modbase_runner_create(m_engine, batch_size, &m_runner);
        if (rc != B200_OK) {
            const std::string msg = b200_last_error();
            b200_modbase_engine_destroy(m_engine);
            throw std::runtime_error("b200call: " + msg);
        }
    }
    ~B200ModBaseModelImpl() override {
        b200_modbase_runner_destroy(m_runner);
        b200_modbase_engine_destroy(m_engine);
    }
    B200ModBaseModelImpl(const B200ModBaseModelImpl&) = delete;
    B200ModBaseModelImpl& operator=(const B200ModBaseModelImpl&) = delete;

    at::Tensor forward(const at::Tensor& sigs_N1T, const at::Tensor& seqs_NTC) {
        const int64_t N = sigs_N1T.size(0);
        if (sigs_N1T.dim() != 3 || sigs_N1T.size(1) != 1 || seqs_NTC.dim() != 3 || seqs_NTC.size(0) != N) {
            throw std::runtime_error("B200ModBaseModel::forward: expected signal [N, 1, T] and sequence [N, T_seq, C]");
        }
        if (N < 1 || N > b200_modbase_runner_batch_size(m_runner)) {
            throw std::runtime_error("B200ModBaseModel::forward: " + std::to_string(N) + " chunks for a batch of " +
                                     std::to_string(b200_modbase_runner_batch_size(m_runner)));
        }
        const at::Tensor sig = sigs_N1T.to(at::kCPU, at::kHalf).contiguous();
        const at::Tensor seq = seqs_NTC.to(at::kCPU, at::kChar).contiguous();
        const int64_t sig_len = sig.size(2), kmer_elems = seq.size(1) * seq.size(2);
        for (int64_t i = 0; i < N; ++i) {
            check(b200_modbase_runner_accept_chunk(
                    m_runner, static_cast<int32_t>(i), reinterpret_cast<const uint16_t*>(sig.data_ptr<at::Half>()) + i * sig_len,
                    sig_len, seq.data_ptr<int8_t>() + i * kmer_elems, kmer_elems));
        }
        const uint16_t* probs = nullptr;
        check(b200_modbase_runner_call_chunks(m_runner, static_cast<int32_t>(N), &probs));
        const int64_t row = int64_t(b200_modbase_runner_out_len(m_runner)) * b200_modbase_runner_num_out(m_runner);
        at::Tensor out = at::from_blob(const_cast<uint16_t*>(probs), {N, row}, at::kHalf).clone();
        return out.to(sigs_N1T.device());
    }

    // load_modbase_conv_lstm_weights (ModBaseModel.cpp:49-75): the *.tensor file list, which is also the engine's naming
    static std::vector<std::string> tensor_names(const config::ModBaseModelConfig& config) {
        std::vector<std::string> n;
        for (const char* c : {"sig_conv1", "sig_conv2", "sig_conv3", "seq_conv1", "seq_conv2", "merge_conv1"}) {
            n.push_back(std::string(c) + ".weight.tensor");
            n.push_back(std::string(c) + ".bias.tensor");
        }
        for (const char* l : {"lstm1.", "lstm2."}) {
            for (const char* s : {"weight_ih_l0.tensor", "weight_hh_l0.tensor", "bias_ih_l0.tensor", "bias_hh_l0.tensor"}) {
                n.push_back(std::string(l) + s);
            }
        }
        n.push_back("fc.weight.tensor");
        n.push_back("fc.bias.tensor");
        if (config.general.modules.has_value() && config.general.modules->upsample.has_value()) {
            n.push_back("linear_up.linear.weight.tensor");
            n.push_back("linear_up.linear.bias.tensor");
        }
        return n;
    }

    const config::ModBaseModelConfig& config() const { return m_config; }

private:
    static void check(int status) {
        if (status != B200_OK) throw std::runtime_error(std::string("b200call: ") + b200_last_error());
    }

    const config::ModBaseModelConfig m_config;
    b200_modbase_engine* m_engine = nullptr;
    b200_modbase_runner* m_runner = nullptr;
};

TORCH_MODULE(B200ModBaseModel);

}  // namespace dorado::modbase::model
