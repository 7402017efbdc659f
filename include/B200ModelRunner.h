// B200ModelRunner.h -- the reference-side binding: dorado::basecall::ModelRunnerBase implemented on top of the
// C ABI in b200call.h.  Header-only; this is the file a dorado maintainer adds under dorado/basecall/ (see
// INTEGRATION.md).  It is the successor of CudaModelRunner (dorado/basecall/CudaModelRunner.cpp:13-77) and
// CudaCaller (dorado/basecall/CudaCaller.cpp:149-720); libtorch is touched only at this edge (at::Tensor in
// accept_chunk, torch::load for the *.tensor weight files), never inside libb200call.so.
//
// Contract kept (SURVEY.md section 8b):
//   accept_chunk(idx, [C_in, chunk_size] half/float tensor)  -> copy into batch slot idx
//   call_chunks(n) -> exactly n DecodedChunk{sequence, qstring, moves}; moves.size() == chunk_size / stride;
//                     blocking; runners sharing a caller run concurrently on their own streams (one thread per runner);
//                     errors -> std::runtime_error
//   config(), chunk_size(), batch_size(), batch_timeouts_ms(), is_low_latency(), terminate(), restart(),
//   get_name() (unique), sample_stats() with the reference's keys "batches_called", "model_decode_ms".
#pragma once

#include "b200call.h"

#include "basecall/ModelRunnerBase.h"
#include "basecall/crf_utils.h"
#include "config/BasecallModelConfig.h"
#include "utils/dev_utils.h"

#include <ATen/ATen.h>

#include <atomic>
#include <cstdlib>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

namespace dorado::basecall {

// One model replica on one device; shared by the runners of that device (the reference's CudaCaller).
class B200Caller {
public:
    // low_latency: params.pipeline_type == PipelineType::simplex_low_latency (CudaCaller.cpp:149-152)
    // num_runners: how many runners create_basecall_runners is going to build on this caller (api/runner_creation.cpp:91-123)
    B200Caller(const config::BasecallModelConfig& model_config, int device_index, bool low_latency = false, int num_runners = 2)
            : m_config(model_config), m_device(device_index) {
        b200_model_desc d{};
        d.model_type = model_config.is_tx_model() ? B200_MODEL_TX : B200_MODEL_LSTM;
        d.num_convs = static_cast<int32_t>(model_config.convs.size());
        for (size_t i = 0; i < model_config.convs.size() && i < 8; ++i) {
            const auto& c = model_config.convs[i];
            d.convs[i] = {c.insize, c.size, c.winlen, c.stride, static_cast<int32_t>(c.activation)};
        }
        d.state_len = model_config.state_len;
        d.outsize = model_config.outsize;
        d.stride = model_config.stride;
        d.clamp = model_config.clamp ? 1 : 0;
        d.qscale = model_config.qscale;
        d.qbias = model_config.qbias;
        d.lstm_size = model_config.lstm_size;
        d.lstm_layers = model_config.lstm_layers;
        d.lstm_inner_dim = model_config.lstm_inner_dim.value_or(0);
        d.linear_bias = model_config.bias ? 1 : 0;
        d.out_features = model_config.is_tx_model() ? 0 : model_config.out_features.value_or(0);
        d.crf_scale = model_config.scale;
        if (model_config.is_tx_model()) {
            const auto& tx = model_config.tx->tx;
            d.d_model = tx.d_model;
            d.nhead = tx.nhead;
            d.dim_feedforward = tx.dim_feedforward;
            d.depth = tx.depth;
            d.attn_window_upper = tx.attn_window.first;
            d.attn_window_lower = tx.attn_window.second;
            d.deepnorm_alpha = tx.deepnorm_alpha;
            d.theta = tx.theta;
            d.max_seq_len = tx.max_seq_len;
            d.upsample_scale = model_config.tx->upsample.scale_factor;
            d.tx_crf_scale = model_config.tx->crf.scale;
            // The reference's dev option (TxModules.cpp:477-479): koi_use_f8=1 runs fc1 / fc2 on E4M3 operands with
            // remove_bits = 4 on the fp16 weights it keeps (b200call.h, tx_precision).  Together with an explicit koi_use_i8=1
            // (TxModules.cpp:936), the reference's default on an H100, the QKV projection also runs on int8 operands.  Off
            // unless asked for here: the fp16 path is the one held to the oracle.  koi_use_i8 without koi_use_f8 (int8 fc1)
            // and other remove_bits values have no counterpart, and leave the model in fp16.
            if (utils::get_dev_opt<bool>("koi_use_f8", false)) {
                d.tx_precision = utils::get_dev_opt<bool>("koi_use_i8", false) ? B200_TX_I8_QKV_FP8_FFN : B200_TX_FP8_FFN;
            }
        }
        // The reference's own override (ConvStack.cpp:77-87): DORADO_LSTM_MODE=CUTLASS_TNC_I8 selects the int8 LSTM layers
        // (b200call.h, lstm_precision).  The reference runs hac that way by default; here fp16 is the default and the mode is
        // taken only when asked for, on the shapes the engine has it for (others fail engine creation).
        if (!model_config.is_tx_model()) {
            const char* lstm_mode = std::getenv("DORADO_LSTM_MODE");
            if (lstm_mode != nullptr && std::string(lstm_mode) == "CUTLASS_TNC_I8") {
                d.lstm_precision = B200_LSTM_INT8;
            }
        }
        // Weights: the reference's own loader (crf_utils.cpp:26-150) gives the tensors in file-list order; the
        // engine wants them as named host fp32 arrays.
        const auto names = tensor_names(model_config);
        auto tensors = load_crf_model_weights(model_config);
        if (tensors.size() != names.size()) {
            throw std::runtime_error("B200Caller: unexpected number of weight tensors");
        }
        std::vector<at::Tensor> keep;
        std::vector<b200_tensor> bt(tensors.size());
        for (size_t i = 0; i < tensors.size(); ++i) {
            keep.push_back(tensors[i].to(at::kCPU, at::kFloat).contiguous());
            bt[i].name = names[i].c_str();
            bt[i].data = keep.back().data_ptr<float>();
            bt[i].ndim = static_cast<int32_t>(keep.back().dim());
            for (int64_t k = 0; k < keep.back().dim() && k < 4; ++k) {
                bt[i].dims[k] = keep.back().size(k);
            }
        }
        check(b200_engine_create(&d, bt.data(), static_cast<int32_t>(bt.size()), device_index, &m_engine));
        check(b200_engine_set_low_latency(m_engine, low_latency ? 1 : 0));
        check(b200_engine_set_num_runners(m_engine, num_runners));
    }
    ~B200Caller() { b200_engine_destroy(m_engine); }
    B200Caller(const B200Caller&) = delete;
    B200Caller& operator=(const B200Caller&) = delete;

    b200_engine* engine() const { return m_engine; }
    const config::BasecallModelConfig& config() const { return m_config; }
    int device() const { return m_device; }

    static void check(int status) {
        if (status != B200_OK) {
            throw std::runtime_error(std::string("b200call: ") + b200_last_error());
        }
    }

    // The reference's *.tensor file list (crf_utils.cpp:34-47, 104-150), which is also the naming the engine uses.
    static std::vector<std::string> tensor_names(const config::BasecallModelConfig& cfg) {
        std::vector<std::string> n;
        if (cfg.is_tx_model()) {
            for (size_t i = 0; i < cfg.convs.size(); ++i) {
                n.push_back("conv." + std::to_string(i) + ".conv.weight.tensor");
                n.push_back("conv." + std::to_string(i) + ".conv.bias.tensor");
            }
            for (int l = 0; l < cfg.tx->tx.depth; ++l) {
                const std::string p = "transformer_encoder." + std::to_string(l) + ".";
                for (const char* s : {"self_attn.Wqkv.weight.tensor", "self_attn.out_proj.weight.tensor",
                                      "self_attn.out_proj.bias.tensor", "ff.fc1.weight.tensor", "ff.fc2.weight.tensor",
                                      "norm1.weight.tensor", "norm2.weight.tensor"}) {
                    n.push_back(p + s);
                }
            }
            n.push_back("upsample.linear.weight.tensor");
            n.push_back("upsample.linear.bias.tensor");
            n.push_back("crf.linear.weight.tensor");
            return n;
        }
        for (size_t i = 0; i < cfg.convs.size(); ++i) {
            n.push_back(std::to_string(i) + ".conv.weight.tensor");
            n.push_back(std::to_string(i) + ".conv.bias.tensor");
        }
        for (int l = 0; l < cfg.lstm_layers; ++l) {
            const std::string p = std::to_string(cfg.convs.size() + l + 1) + ".rnn.";
            if (cfg.is_flstm_model()) {  // crf_utils.cpp:36-41
                for (const char* s : {"dn_weight_ih.tensor", "dn_weight_hh.tensor", "up_weight_ih.tensor", "up_weight_hh.tensor",
                                      "up_bias_ih.tensor", "up_bias_hh.tensor"}) {
                    n.push_back(p + s);
                }
                continue;
            }
            for (const char* s : {"weight_ih_l0.tensor", "weight_hh_l0.tensor", "bias_ih_l0.tensor", "bias_hh_l0.tensor"}) {
                n.push_back(p + s);
            }
        }
        const size_t layer = cfg.convs.size() + cfg.lstm_layers + 1;
        n.push_back(std::to_string(layer) + ".linear.weight.tensor");
        if (cfg.bias) {
            n.push_back(std::to_string(layer) + ".linear.bias.tensor");
        }
        if (cfg.out_features.has_value()) {
            n.push_back(std::to_string(layer + 1) + ".linear.weight.tensor");
        }
        return n;
    }

private:
    const config::BasecallModelConfig m_config;
    int m_device;
    b200_engine* m_engine{nullptr};
};

class B200ModelRunner final : public ModelRunnerBase {
public:
    B200ModelRunner(std::shared_ptr<B200Caller> caller, int batch_size, int chunk_size)
            : m_caller(std::move(caller)) {
        B200Caller::check(b200_runner_create(m_caller->engine(), batch_size, chunk_size, &m_runner));
        b200_decoder_options o;
        b200_default_decoder_options(&o);
        o.q_shift = m_caller->config().qbias;   // CudaCaller.cpp:159-160
        o.q_scale = m_caller->config().qscale;
        B200Caller::check(b200_runner_set_decoder_options(m_runner, &o));
        static std::atomic<int> ids{0};
        m_name = "B200ModelRunner_" + std::to_string(m_caller->device()) + "_" + std::to_string(ids++);
    }
    ~B200ModelRunner() override { b200_runner_destroy(m_runner); }

    void accept_chunk(int chunk_idx, const at::Tensor& chunk) final {
        const at::Tensor flat = chunk.reshape({-1}).contiguous();
        if (flat.scalar_type() == at::kHalf) {
            B200Caller::check(b200_runner_accept_chunk_f16(m_runner, chunk_idx,
                                                           reinterpret_cast<const uint16_t*>(flat.data_ptr<at::Half>()),
                                                           flat.numel()));
        } else {
            const at::Tensor f = flat.to(at::kFloat);
            B200Caller::check(b200_runner_accept_chunk_f32(m_runner, chunk_idx, f.data_ptr<float>(), f.numel()));
        }
    }

    // Raw-signal variant of accept_chunk (not part of ModelRunnerBase): `raw` is the read's whole int16 signal as the
    // DataLoader delivers it (ScalerNode.cpp:190 asserts kShort), shift/scale what ScalerNode computed for the read.
    // Scaling, slicing and repeat-padding run on the device (b200call.h: b200_runner_accept_raw_chunk), so ScalerNode's
    // in-place fp16 conversion and BasecallerNode's slice/concat (BasecallerNode.cpp:395-440) are skipped.
    void accept_raw_chunk(int chunk_idx, const at::Tensor& raw, size_t input_offset, float shift, float scale) {
        if (raw.scalar_type() != at::kShort || !raw.is_contiguous()) {
            throw std::invalid_argument("B200ModelRunner::accept_raw_chunk expects a contiguous int16 tensor");
        }
        b200_raw_chunk c{};
        c.raw = raw.data_ptr<int16_t>();
        c.num_samples = static_cast<uint64_t>(raw.numel());
        c.input_offset = static_cast<uint64_t>(input_offset);
        c.shift = shift;
        c.scale = scale;
        B200Caller::check(b200_runner_accept_raw_chunk(m_runner, chunk_idx, &c));
    }

    std::vector<decode::DecodedChunk> call_chunks(int num_chunks) final {
        b200_result r{};
        B200Caller::check(b200_runner_call_chunks(m_runner, num_chunks, &r));
        std::vector<decode::DecodedChunk> out(static_cast<size_t>(num_chunks));
        for (int i = 0; i < num_chunks; ++i) {
            const size_t off = static_cast<size_t>(i) * static_cast<size_t>(r.t_out);
            const auto n = static_cast<size_t>(r.n_bases[i]);
            out[i].sequence.assign(r.sequence + off, n);
            out[i].qstring.assign(r.qstring + off, n);
            out[i].moves.assign(r.moves + off, r.moves + off + r.t_out);
        }
        return out;
    }

    const config::BasecallModelConfig& config() const final { return m_caller->config(); }
    size_t chunk_size() const final { return static_cast<size_t>(b200_runner_chunk_size(m_runner)); }
    size_t batch_size() const final { return static_cast<size_t>(b200_runner_batch_size(m_runner)); }
    std::pair<int, int> batch_timeouts_ms() const final {  // CudaCaller.cpp:216-222
        int32_t first = 0, last = 0;
        B200Caller::check(b200_engine_batch_timeouts_ms(m_caller->engine(), &first, &last));
        return {first, last};
    }
    bool is_low_latency() const final { return b200_engine_is_low_latency(m_caller->engine()) != 0; }
    void terminate() final { B200Caller::check(b200_engine_terminate(m_caller->engine())); }  // CudaModelRunner.cpp:62
    void restart() final { B200Caller::check(b200_engine_restart(m_caller->engine())); }      // CudaModelRunner.cpp:64
    std::string get_name() const final { return m_name; }

    stats::NamedStats sample_stats() const final {
        stats::NamedStats s;
        b200_stats st{};
        if (b200_engine_get_stats(m_caller->engine(), &st) == B200_OK) {
            s["batches_called"] = static_cast<double>(st.batches_called);  // CudaCaller.cpp:316-321
            s["model_decode_ms"] = st.model_decode_ms;
        }
        return s;
    }

private:
    std::shared_ptr<B200Caller> m_caller;
    b200_runner* m_runner{nullptr};
    std::string m_name;
};

}  // namespace dorado::basecall
