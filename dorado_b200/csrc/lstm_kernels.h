// Kernels of lstm_model.cu that other models reuse (modbase_model.cu): the fused conv1 + conv2 of a 1-channel signal, and
// the LSTM recurrences.  An LSTM layer is the x-projection GEMM (gemm.cu, gx = x W_ih^T + b_ih + b_hh, fp16 [T][N][4C])
// followed by one of the recurrences, which overwrite the sequence buffer [T][N][C] with h in place.
#pragma once

#include "b200call.h"
#include "common.cuh"

#include <vector>

namespace b200 {

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

// lstm_rec_kernel (lstm_size 192 and 384): a thread-block cluster per lstm_rec_chunks() chunks
struct LstmRecParams {
    __half* seq;          // [T][N][C] output h (in place over the layer input, which gx has consumed)
    const __half* gx;     // [T][N][4C]
    const __half* w_hh;   // [4C][C], PyTorch row order
    int T, N, reverse;
    const int32_t* lens;  // optional per-chunk length in samples (variable chunk sizes); stride = samples per step
    int stride;
};

// lstm_grid_rec_kernel (lstm_size 768 and 1024): groups of C / 16 CTAs that exchange h through L2
struct LstmGridParams {
    __half* seq;            // [T][N][C] output h (in place over the layer input, which gx has consumed)
    const __half* gx;       // [T][N][4C]
    const __half* w_hh;     // [4C][C], PyTorch row order
    int T, N, reverse;
    const int32_t* lens;    // optional per-chunk length in samples (variable chunk sizes); stride = samples per step
    int stride;
    int n_first;            // first chunk of this launch; group g owns chunks n_first + g NB ..
    unsigned int* counters; // one arrival counter per group of this launch, zero at launch
    int* error;             // set to 1 when a group barrier times out
};

// Chunks per cluster of lstm_rec_kernel for a padded batch of Np chunks (a multiple of 16), and the cluster size
int lstm_rec_chunks(int Np);
int lstm_rec_cluster_ctas(int C);
// Launches lstm_rec_kernel<C, cluster, nb> over `ctas` CTAs; throws Unsupported for a size without an instantiation
void launch_lstm_rec(int C, int nb, int ctas, const LstmRecParams& p, cudaStream_t stream);

// Launch shape of lstm_grid_rec_kernel for a padded batch of Np chunks (a multiple of 32) with `runners` batches in flight
struct LstmGridPlan {
    int nb = 0, groups = 0, launches = 0, ctas = 0;
    std::vector<int> launch_ctas;  // per launch (the last one may hold fewer groups)
};
LstmGridPlan plan_lstm_grid(int C, int Np, int runners);
// One cooperative launch of lstm_grid_rec_kernel<C, nb>
void launch_lstm_grid(int C, int nb, int ctas, const LstmGridParams& p, cudaStream_t stream);

}  // namespace b200
