// Parts of lstm_model.cu that other models reuse (modbase_model.cu): the fused conv1 + conv2 of a 1-channel signal, and
// the LSTM stack.  The stack owns how LSTM layers are laid out, planned and launched; its callers see neither the
// recurrence kernels nor their launch shapes, counters or error word.
#pragma once

#include "b200call.h"
#include "common.cuh"
#include "gemm.h"

#include <string>
#include <vector>

namespace b200 {

struct ProfileSink;

// conv1 (1 -> c1 <= 16 channels, w1) + conv2 (c1 -> 16, w2), both stride 1 with padding winlen / 2, fused on the FMA pipe
// (conv12_kernel): fp32 math, fp16 NTC output
constexpr int kConv12MaxWin = 9;
struct Conv12Params {
    const __half* x;  // [N][T]
    __half* out;      // [N][T_pad][16], row r <-> sample r - front_pad
    const float* w;   // packed: w1 [c1][w1] | b1 [16] | w2 [k][ci][co] (16x16 per tap) | b2 [16]
    int N, T, T_pad, front_pad;
    int c1, w1, w2, act1, act2;
    const int32_t* lens;  // optional per-chunk length in samples (variable chunk sizes): the chunk is zero beyond it
    int* tile_counter;    // conv12_tc_kernel: next tile to hand out (zeroed on the stream before every launch)
};
// torch-layout conv weights and biases -> the packed device array of Conv12Params::w (freed with cudaFree by the owner)
float* upload_conv12_weights(const b200_tensor& w1, const b200_tensor& b1, const b200_tensor& w2, const b200_tensor& b2,
                             const b200_conv_desc& c1, const b200_conv_desc& c2);
void launch_conv12(const Conv12Params& p, cudaStream_t stream);

// One LSTM layer's weights on the device.  lstm_size 96 (lstm_layer_kernel): W_ih [4C][C], W_hh and the bias with their
// gate rows permuted for the fused kernel.  Other sizes: PyTorch gate order (i | f | g | o), W_ih [4C][C padded to a
// multiple of 64] for the x-projection GEMM.
// The int8 form (upload_lstm_layer_int8; lstm_size 256 and 384): w_ih8 and w_hh8 [4C][C] int8, quantised together per gate
// row, inv [4C] the fp32 factor that dequantises a row's s32 accumulator, and the bias; w_ih and w_hh stay null.
struct LstmLayerWeights {
    __half* w_ih = nullptr;
    __half* w_hh = nullptr;  // [4C][C]
    float* bias = nullptr;   // [4C] b_ih + b_hh (fp32)
    int8_t* w_ih8 = nullptr;
    int8_t* w_hh8 = nullptr;
    float* inv = nullptr;
};
// fp32 PyTorch layouts (W_ih and W_hh [4C][C], b_ih and b_hh [4C]) -> the device layout for lstm_size C
LstmLayerWeights upload_lstm_layer(int C, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh);
LstmLayerWeights upload_lstm_layer_int8(int C, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh);
void free_lstm_layer(LstmLayerWeights& w);

struct LstmStackDesc {
    int C = 0;                   // lstm_size: 96, 128, 192, 256, 384, 768 or 1024
    int T = 0;                   // steps
    int Np = 0;                  // padded batch: a multiple of 16 (lstm_size 96) or 32
    int stride = 1;              // samples per step, for the chunk lengths of set_chunk_lengths
    int runners = 1;             // batches in flight: sizes the grid recurrence and caps the x-projection GEMM's CTAs
    bool reverse_first = false;  // layer 0 (and every other layer after it) runs reversed in time
    // int8 layers (lstm_size 256 and 384): seq holds int8 cvt.rni.sat.s8(kInt8ActScale * v), the x-projection and the
    // recurrence run on int8 operands with s32 accumulation (the int8 form of lstm_rec_kernel), gx stays fp16
    bool int8 = false;
    void* seq = nullptr;         // [T + 1][Np][C] fp16 (int8 if `int8`): the first layer's input, overwritten in place with h by every layer
    const LstmLayerWeights* layers = nullptr;  // kept by the caller for the stack's lifetime
    int num_layers = 0;
};
// The stack's slice of the caller's workspace: gx [T][Np][4C] (not for lstm_size 96), and for 768 / 1024 the group
// counters (one per 32 chunks and layer) and the error word of the grid recurrence
struct LstmStackBuffers {
    __half* gx = nullptr;
    unsigned int* counters = nullptr;
    size_t counter_bytes = 0;
    int* error = nullptr;
};
class Bump;
LstmStackBuffers carve_lstm_stack(Bump& b, int C, int num_layers, int T, int Np);

// Every layer is lstm_layer_kernel (lstm_size 96), or the x-projection GEMM followed by lstm_rec_kernel (128 - 384) or by
// one or more cooperative launches of lstm_grid_rec_kernel (768, 1024); int8 layers are the int8 x-projection GEMM followed
// by the int8 form of lstm_rec_kernel.  Built once per batch shape; reads
// B200_DEBUG_LSTM_LAYERS, B200_CLUSTER_CHUNKS, B200_GRID_CHUNKS and B200_GRID_GROUPS then.
class LstmStack {
public:
    LstmStack(const LstmStackDesc& d, const LstmStackBuffers& ws);  // ws: carved by carve_lstm_stack for the same shape
    ~LstmStack();
    LstmStack(const LstmStack&) = delete;
    LstmStack& operator=(const LstmStack&) = delete;
    // Enqueues the layers; false if B200_DEBUG_LSTM_LAYERS stopped the stack early (the sequence buffer then holds the
    // output of that many layers)
    bool run(cudaStream_t stream, ProfileSink* prof);
    // Variable chunk sizes: device array of per-chunk lengths in samples (lstm_size 128 and up)
    void set_chunk_lengths(const int32_t* d_lens) { m_lens = d_lens; }
    // After the stream has drained: throws if a group of the grid recurrence timed out at its step barrier
    void check_errors();
    std::string info() const;  // the launch shape: lstm_layer.*, lstm_rec.* or lstm_grid.* keys
    int launches() const;      // kernel launches per run

private:
    enum class Kind { Layer, Rec, Grid };
    Kind m_kind = Kind::Layer;
    LstmStackDesc m_d;
    int m_debug_layers = -1;  // >= 0: stop after that many layers
    // chunks per CTA / cluster / group, groups per launch, launches per layer, CTAs per group
    int m_nb = 0, m_groups = 0, m_launches = 1, m_group_ctas = 1;
    std::vector<GemmPlan> m_gx_gemm;  // per layer (not for lstm_size 96)
    // the counters are zeroed at the start of every run; a group whose step barrier timed out sets the error word
    LstmStackBuffers m_ws;
    const int32_t* m_lens = nullptr;
    int* m_error_host = nullptr;  // pinned copy of the error word, written at the end of every run
};

}  // namespace b200
