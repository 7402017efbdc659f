// CRF decode entry points (device pointers). See decode.cu.
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "b200_crf_math.h"

namespace b200 {

struct DecodeArgs {
    const __half* scores;  // [N][T][4^(state_len+1)] fp16
    int N;
    int T;
    int state_len;
    float clamp_val;  // > 0: clamp scores to +-clamp_val on read (dorado/basecall/decode/Decoder.cpp:19)
    // DecoderOptions (dorado/basecall/include/basecall/DecodedChunk.h:15-23)
    int beam_width;
    float log_beam_cut;  // logf(beam_cut) or FLT_MAX when beam_cut <= 0 (beam_search.cpp:147-148)
    float blank;
    float q_shift;
    float q_scale;
    const b200_qtable* qtable;
    const int32_t* lens;  // optional per-chunk length in SAMPLES (variable chunk sizes); nullptr = every chunk has T blocks
    int stride;           // samples per block (only read with lens)
    int runners;          // batches in flight on the device (Model::num_runners_hint; < 1 means 1): sizes the state_len 3 grid
    long long* dbg;  // optional clock64 timeline of chunk 0, state_len 4 and 5 (B200_DEBUG_BEAM_TIMELINE, test hook only); nullptr in production
    // scratch
    float* bwd;   // carve_decode_scratch()
    uint2* beam;
    // outputs (device), rows of T
    uint8_t* moves;
    char* sequence;
    char* qstring;
    int32_t* n_bases;
};

size_t decode_max_blocks();  // largest T the traceback kernel's shared-memory plan holds
class Bump;
// The decoder's scratch for N chunks of T blocks: backward scores [N][T + 1][4^state_len] and beam records [N][T][32]
void carve_decode_scratch(Bump& b, int N, int T, int state_len, float** bwd, uint2** beam);
int decode_launches(int state_len);  // kernels one decode_scores call launches
struct ProfileSink;
void decode_scores(const DecodeArgs& args, cudaStream_t stream, ProfileSink* prof = nullptr);

}  // namespace b200
