// CRF decode for sm_90a: backward scan -> fused forward scan / posteriors / beam search -> traceback.
//
// Replaces the closed Koi kernels behind dorado/basecall/decode/CUDADecoder.cpp:76-104
// (host_back_guide_step, host_beam_search_step, host_compute_posts_step, host_run_decode) and the CPU
// slicing of CUDADecoder.cpp:115-173.  Semantics are those of the reference's open CPU decoder:
//   scans          dorado/basecall/decode/CPUDecoder.cpp:17-92
//   posteriors     CPUDecoder.cpp:130
//   beam search    dorado/basecall/decode/beam_search.cpp:125-520
//   sequence/qual  beam_search.cpp:54-102
// All floating point goes through include/b200_crf_math.h so results are bit-identical to the CPU
// oracle (oracle/crf_oracle.c).
//
// Data layout in HBM (per batch of N chunks, T blocks, S = 4^state_len states, C = 4S):
//   scores  fp16  [N][T][C]        read twice (once per scan direction), coalesced 32 B per thread
//   bwd     fp32  [N][T+1][S]      written by kernel 1, read once by kernel 2
//   beam    2 x 4 B [N][T][32]     two planes per kept element: meta {state:16, prev:8, stay:8} (all the traceback's pointer
//                                  chase reads) and the block probability f32 (before the ^0.4 of the qscore; read along the
//                                  chosen path only)
//   out     u8    moves/seq/qstr [N][T], n_bases i32 [N]
// Thread mapping: one thread per state in both scans (two states per thread for S = 1024 in the forward
// kernel); the forward kernel adds one beam-search warp per chunk that runs one block behind the scan.
#include "decode.h"

#include "b200_crf_math.h"
#include "common.cuh"
#include "engine.h"
#include "nvtx.h"

#include <string>

namespace b200 {

namespace {

constexpr int kBeamW = 32;
constexpr uint32_t kCrcPoly = 0x82f63b78u;
constexpr uint32_t kCrcSeed = 0x12345678u;

template <int SL>
struct Dims {
    static constexpr int S = 1 << (2 * SL);
    static constexpr int C = 4 * S;
};

// ------------------------------------------------------------------------------------------------
// Kernel 1: backward scan (CPUDecoder.cpp:69-92).  One thread per state.
//   bwd[t][v] = LSE( bwd[t+1][v] + blank, bwd[t+1][succ_j] + M[t][succ_j*4 + top(v)] , j = 0..3 )
// with v = q + top*S/4, succ_j = 4q + j.  The score row is staged through shared memory "transposed"
// ([i % 16][i / 16]) so that both the coalesced global read (4 fp16 per thread) and the per-state
// gather are bank-conflict free.
// ------------------------------------------------------------------------------------------------
template <int SL>
struct ScanCfg {
    static constexpr int S = Dims<SL>::S, C = Dims<SL>::C, P4 = S / 4;
    static constexpr int SPT = S > 512 ? S / 512 : 1;   // states per scan thread
    static constexpr int NT = S / SPT;                  // scan threads per chunk
    static constexpr int PITCH = P4 + 2;                // 4 * PITCH == 8 (mod 32): conflict-free staging
};

// Score clamp (Decoder.cpp:19): c <= 0 means no clamp.  min / max (two ALU-pipe instructions) instead of two compare + select
// pairs on the FMA pipe; identical for every non-NaN score.
__device__ __forceinline__ float clampf(float v, float c) {
    const float ce = c > 0.0f ? c : __int_as_float(0x7f800000);
    return fminf(fmaxf(v, -ce), ce);
}

template <int SL>
__global__ void __launch_bounds__(ScanCfg<SL>::S > 256 ? ScanCfg<SL>::S : 256)
        crf_bwd_scan_kernel(const __half* __restrict__ scores, float* __restrict__ bwd, int N, int T_pitch, float clamp_val,
                            float blank, const int32_t* __restrict__ lens, int stride) {
    using Cfg = ScanCfg<SL>;
    constexpr int S = Cfg::S, C = Cfg::C, P4 = Cfg::P4, PITCH = Cfg::PITCH;
    constexpr int CH = S >= 256 ? 1 : 256 / S;  // chunks per CTA
    constexpr int PF = 4;
    const int g = threadIdx.x / S;
    const int v = threadIdx.x % S;
    const int chunk = blockIdx.x * CH + g;
    __shared__ __align__(16) float a[CH][2][S];
    __shared__ float st[CH][2][16 * PITCH];
    const bool active = chunk < N;
    const int chunk_c = active ? chunk : N - 1;  // idle groups shadow the last chunk (no stores)
    // variable chunk sizes: this chunk has T of the T_pitch blocks its rows are laid out for
    const int T = lens ? min(T_pitch, __ldg(lens + chunk_c) / stride) : T_pitch;
    const uint2* srow = reinterpret_cast<const uint2*>(scores + (size_t)chunk_c * T_pitch * C) + v;
    constexpr int RS = C / 4;  // row stride in uint2
    float* out = bwd + (size_t)chunk_c * (T_pitch + 1) * S;
    const int q = v % P4, top = v / P4;
    const int st_row = 4 * (v & 3), st_col = v >> 2;

    uint2 pf[PF];
#pragma unroll
    for (int k = 0; k < PF; ++k) {
        const int tt = T - 1 - k;
        if (tt >= 0) pf[k] = __ldg(srow + (size_t)tt * RS);
    }
    auto stage = [&](int buf, const uint2& r) {
        const __half2 h0 = *reinterpret_cast<const __half2*>(&r.x), h1 = *reinterpret_cast<const __half2*>(&r.y);
        const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        float* d = &st[g][buf][st_row * PITCH + st_col];
        d[0] = clampf(f0.x, clamp_val);
        d[PITCH] = clampf(f0.y, clamp_val);
        d[2 * PITCH] = clampf(f1.x, clamp_val);
        d[3 * PITCH] = clampf(f1.y, clamp_val);
    };
    float own = 0.0f;
    a[g][0][v] = 0.0f;
    if (active) out[(size_t)T * S + v] = 0.0f;
    stage(0, pf[0]);
    if (T - 1 - PF >= 0) pf[0] = __ldg(srow + (size_t)(T - 1 - PF) * RS);
    if constexpr (S <= 32) __syncwarp(); else named_bar_sync(1 + g, S);

    int cur = 0;
    for (int t = T - 1; t >= 0; t -= PF) {
#pragma unroll
        for (int k = 0; k < PF; ++k) {
            const int tt = t - k;
            if (tt >= 0) {
                // stage the next block's scores while this block is computed
                if (tt - 1 >= 0) {
                    stage(cur ^ 1, pf[(k + 1) % PF]);
                    if (tt - 1 - PF >= 0) pf[(k + 1) % PF] = __ldg(srow + (size_t)(tt - 1 - PF) * RS);
                }
                const float4 nx = *reinterpret_cast<const float4*>(&a[g][cur][4 * q]);
                const float* sc = &st[g][cur][top * PITCH + q];
                own = b200_lse5(B200_ADD(own, blank), B200_ADD(nx.x, sc[0]), B200_ADD(nx.y, sc[4 * PITCH]),
                                B200_ADD(nx.z, sc[8 * PITCH]), B200_ADD(nx.w, sc[12 * PITCH]));
                a[g][cur ^ 1][v] = own;
                if (active) out[(size_t)tt * S + v] = own;
                if constexpr (S <= 32) __syncwarp(); else named_bar_sync(1 + g, S);
                cur ^= 1;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 2: forward scan + posteriors + beam search, pipelined.
// Per chunk: NT scan threads (one state each; two for S = 1024) produce, for block t, the clamped score row, the
// bwd[t+1] row and the posterior row into a double-buffered shared-memory slot; one beam warp (lane = beam
// element) consumes the slot one block behind, so the scan of block t+1 overlaps the beam step of block t.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t crc_bits(uint32_t crc, uint32_t nb, int nbits) {
    for (int i = 0; i < nbits; ++i) {
        const uint32_t b = (nb ^ crc) & 1u;
        crc >>= 1;
        if (b) crc ^= kCrcPoly;
        nb >>= 1;
    }
    return crc;
}

__device__ __forceinline__ uint32_t crc2(uint32_t crc, uint32_t nb) {
    uint32_t b = (nb ^ crc) & 1u;
    crc = (crc >> 1) ^ (b ? kCrcPoly : 0u);
    b = ((nb >> 1) ^ crc) & 1u;
    crc = (crc >> 1) ^ (b ? kCrcPoly : 0u);
    return crc;
}

// inverse of crc2 for known new bits: the hash a sequence must have had before `nb` was appended
__device__ __forceinline__ uint32_t crc2_inv(uint32_t crc, uint32_t nb) {
    uint32_t b = crc >> 31;  // the polynomial has bit 31 set, (x >> 1) does not
    uint32_t t = crc ^ (b ? kCrcPoly : 0u);
    crc = (t << 1) | (b ^ ((nb >> 1) & 1u));
    b = crc >> 31;
    t = crc ^ (b ? kCrcPoly : 0u);
    crc = (t << 1) | (b ^ (nb & 1u));
    return crc;
}

constexpr int kHashSlots = 1024;  // lane-id table over the low hash bits (stay/step merge lookup)

struct BeamSmem {
    __align__(16) float cand_score[5 * kBeamW];   // [prev][base] step candidates; stays at 4 * width + prev (replay path only)
    uint32_t cand_hash[5 * kBeamW];               // replay path only
    float new_score[kBeamW];
    uint32_t new_hash[kBeamW];
    uint32_t new_meta[kBeamW];  // state | prev << 16 | stay << 24
    __align__(16) uint32_t prev_hash[kBeamW];
    uint8_t slot_lane[kHashSlots];  // never cleared: an entry is only trusted after comparing the hash it points to
};

struct BeamLane {
    uint32_t hash;
    uint32_t state;
    float score;
};

__device__ __forceinline__ uint32_t float_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Initial beam: the W best states of bwd[0] in state order (beam_search.cpp:166-200).
template <int SL>
__device__ int beam_init(const float* bw_row, BeamSmem& bs, BeamLane& me, int W, int lane) {
    constexpr int S = Dims<SL>::S;
    constexpr int VPL = S >= 32 ? S / 32 : 1;
    uint32_t keys[VPL];
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
        const int s = lane * VPL + j;
        keys[j] = s < S ? float_key(bw_row[s]) : 0u;
    }
    uint32_t thr = 0u;  // key >= 0 always true: everything selected when W >= S
    if (W < S) {
        for (int bit = 31; bit >= 0; --bit) {
            const uint32_t cand = thr | (1u << bit);
            int c = 0;
#pragma unroll
            for (int j = 0; j < VPL; ++j) c += (lane * VPL + j < S) && (keys[j] >= cand);
            if (warp_sum_int(c) >= W) thr = cand;
        }
    }
    int c = 0;
#pragma unroll
    for (int j = 0; j < VPL; ++j) c += (lane * VPL + j < S) && (keys[j] >= thr);
    int incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    int pos = incl - c;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
        const int s = lane * VPL + j;
        if (s < S && keys[j] >= thr) {
            if (pos < W) bs.new_meta[pos] = (uint32_t)s;
            ++pos;
        }
    }
    __syncwarp();
    const int width = W < S ? W : S;
    if (lane < width) {
        me.state = bs.new_meta[lane] & 0xffffu;
        me.hash = crc_bits(kCrcSeed, me.state, 32);
        me.score = 0.0f;
    }
    __syncwarp();
    return width;
}

// Block probability of a kept element's kmer (beam_search.cpp:459-503, before the pow(p, 0.4) that the traceback kernel
// applies along the chosen path only): the posterior of the state plus those of its distinct shift neighbours, added in the
// reference's order L0, R0, L1, R1, ... (L_b = state >> 2 | b << (2k-2), R_b = (state << 2 | b) mod S).  The L's are mutually
// distinct and so are the R's, so a neighbour is skipped iff it equals the state or an earlier neighbour of the OTHER kind.
template <int SL>
__device__ __forceinline__ float kmer_block_prob(const float* post_row, int state) {
    constexpr int S = Dims<SL>::S;
    float prob = post_row[state];
    const int l = state >> 2;
    const int r = (state << 2) & (S - 1);
    constexpr int msb = S >> 2;
    // R_b' == L_b  <=>  r + b' == l + msb * b; with d = l - r:  b' - msb * b == d
    const int d = l - r;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        const int L = l + msb * b, R = r + b;
        // L_b against the state and R_0 .. R_{b-1}
        bool keepL = L != state;
#pragma unroll
        for (int bb = 0; bb < b; ++bb) keepL = keepL && (bb - msb * b != d);
        if (keepL) prob = B200_ADD(prob, post_row[L]);
        // R_b against the state and L_0 .. L_b
        bool keepR = R != state;
#pragma unroll
        for (int bb = 0; bb <= b; ++bb) keepR = keepR && (b - msb * bb != d);
        if (keepR) prob = B200_ADD(prob, post_row[R]);
    }
    return prob < 0.0f ? 0.0f : (prob > 1.0f ? 1.0f : prob);
}

// One block of the beam search for one chunk, executed by one warp (lane = beam element).
// Returns the new beam width; writes the kept elements (meta plane) and their block probabilities (prob plane).
//
// The decode kernels are bound by instruction issue -- the beam warp's block time is its instruction count times a few
// cycles -- so the step is written for few instructions: evaluating three levels of the beam-cut bisection at once
// (7 cutoffs per round) shortens the dependent chain but costs more instructions than it saves.
//   * stay/step merge: a stay i can only merge with the step (j, b_i) whose previous hash is crc2_inv(hash_i, b_i); that j is
//     found through a 1024-entry lane-id table over the low hash bits (one byte store, one byte load, one compare) instead of
//     comparing against all 32 hashes.  Lanes whose table entry was overwritten by another lane (a slot shared by two
//     hashes) are broadcast and compared directly, which also detects equal hashes -- the one case that needs the
//     reference's sequential order (replay path).
template <int SL>
__device__ int beam_step(const __half* sc_row,
                         const float* bw_row,
                         const float* post_row,
                         BeamSmem& bs,
                         BeamLane& me,
                         int width,
                         int W,
                         float log_beam_cut,
                         float blank,
                         bool last_block,
                         uint32_t* meta_row,
                         float* prob_row,
                         int lane,
                         long long* dbg) {
    constexpr int S = Dims<SL>::S;
    constexpr int SB = 2 * SL;
    if (dbg && lane == 0) dbg[0] = clock64();
    constexpr uint32_t mask = S - 1;
    const bool valid = lane < width;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const uint32_t vmask = width >= 32 ? 0xffffffffu : ((1u << width) - 1u);

    // --- candidates (beam_search.cpp:225-262) ---
    uint32_t ns[4], hs[4];
    float s[5];
    float lmax = B200_FLT_LOWEST;
    const uint32_t latest = me.state & 3u;
    const uint32_t target = crc2_inv(me.hash, latest);   // the hash a step's parent must have to merge with this stay
    const uint32_t own_slot = me.hash & (kHashSlots - 1);
    if (valid) {
        const uint32_t shifted = me.state << 2;
        const uint32_t dropped = shifted >> SB;
        const uint32_t nb = shifted & mask;
        const float4 bw4 = *reinterpret_cast<const float4*>(bw_row + nb);   // bwd of the four successor states
        const float bws = bw_row[me.state];
        const float bwv[4] = {bw4.x, bw4.y, bw4.z, bw4.w};
        bs.slot_lane[own_slot] = (uint8_t)lane;
        bs.prev_hash[lane] = me.hash;
#pragma unroll
        for (uint32_t b = 0; b < 4; ++b) {
            ns[b] = nb | b;
            const uint32_t move_idx = ((ns[b] << 2) + dropped) & 0xffffu;
            s[b] = B200_ADD(B200_ADD(me.score, __half2float(sc_row[move_idx])), bwv[b]);
            hs[b] = crc2(me.hash, b);
            lmax = b200_fmaxf(lmax, s[b]);
        }
        s[4] = B200_ADD(B200_ADD(me.score, blank), bws);
        lmax = b200_fmaxf(lmax, s[4]);
        *reinterpret_cast<float4*>(&bs.cand_score[lane * 4]) = make_float4(s[0], s[1], s[2], s[3]);
    }
    float max_score = warp_max(lmax);
    __syncwarp();
    if (dbg && lane == 0) dbg[1] = clock64();

    // --- merge stays with equal-hash steps (beam_search.cpp:264-305) ---
    int jm = -1;
    bool dup = false;
    {
        const uint32_t rb = valid ? bs.slot_lane[own_slot] : (uint32_t)lane;
        const uint32_t c = bs.slot_lane[target & (kHashSlots - 1)] & 31u;
        uint32_t ov = __ballot_sync(0xffffffffu, valid && rb != (uint32_t)lane);
        if (valid && ((vmask >> c) & 1u) && bs.prev_hash[c] == target) jm = (int)c;
        while (ov) {  // lanes not reachable through the table (warp-uniform loop, usually zero or one trip)
            const int j = __ffs(ov) - 1;
            ov &= ov - 1;
            const uint32_t hj = __shfl_sync(0xffffffffu, me.hash, j);
            if (valid && lane != j && me.hash == hj) dup = true;
            if (valid && target == hj) jm = j;
        }
    }
    if (!__any_sync(0xffffffffu, dup)) {
        float folded = B200_FLT_LOWEST;
        if (jm >= 0) {  // hashes are distinct: at most one parent matches
            const int pi = jm * 4 + (int)latest;
            const float st = s[4], sp = bs.cand_score[pi];
            folded = b200_log_sum_exp(st, sp);
            if (st > sp) {
                s[4] = folded;
                bs.cand_score[pi] = B200_FLT_LOWEST;
            } else {
                bs.cand_score[pi] = folded;
                s[4] = B200_FLT_LOWEST;
            }
        }
        max_score = b200_fmaxf(max_score, warp_max(folded));
        __syncwarp();
        if (valid) {
            const float4 r = *reinterpret_cast<const float4*>(&bs.cand_score[lane * 4]);
            s[0] = r.x; s[1] = r.y; s[2] = r.z; s[3] = r.w;
        }
    } else {
        // equal hashes among the beam elements (rare): replay the reference's sequential order
        if (valid) {
#pragma unroll
            for (int b = 0; b < 4; ++b) bs.cand_hash[lane * 4 + b] = hs[b];
            bs.cand_score[4 * width + lane] = s[4];
            bs.cand_hash[4 * width + lane] = me.hash;
        }
        bs.new_meta[lane] = valid ? latest : 0u;
        __syncwarp();
        float m2 = max_score;
        if (lane == 0) {
            for (int i = 0; i < width; ++i) {
                const int si = 4 * width + i;
                const int lt = (int)bs.new_meta[i];
                for (int j = 0; j < width; ++j) {
                    const int pi = j * 4 + lt;
                    if (bs.cand_hash[si] == bs.cand_hash[pi]) {
                        const float st = bs.cand_score[si], sp = bs.cand_score[pi];
                        const float folded = b200_log_sum_exp(st, sp);
                        if (st > sp) {
                            bs.cand_score[si] = folded;
                            bs.cand_score[pi] = B200_FLT_LOWEST;
                        } else {
                            bs.cand_score[pi] = folded;
                            bs.cand_score[si] = B200_FLT_LOWEST;
                        }
                        m2 = b200_fmaxf(m2, folded);
                    }
                }
            }
        }
        max_score = __shfl_sync(0xffffffffu, m2, 0);
        __syncwarp();
        if (valid) {
#pragma unroll
            for (int b = 0; b < 4; ++b) s[b] = bs.cand_score[lane * 4 + b];
            s[4] = bs.cand_score[4 * width + lane];
        }
        __syncwarp();
    }

    if (dbg && lane == 0) dbg[2] = clock64();
    // --- cutoff (beam_search.cpp:310-396) ---
    auto count_part = [&](float c) {  // this lane's share of count_ge(c)
        int n = 0;
        if (valid) {
#pragma unroll
            for (int k = 0; k < 5; ++k) n += (s[k] >= c);
        }
        return n;
    };
    float cutoff = B200_SUB(max_score, log_beam_cut);
    int cnt = warp_sum_int(count_part(cutoff));
    if (cnt > W) {
        const int min_w = (W * 8) / 10;
        float lo = cutoff, hi = max_score;
        int guesses = 1;
        while ((cnt > W || cnt < min_w) && guesses < 10) {
            if (cnt > W) {
                lo = cutoff;
                cutoff = B200_MUL(B200_ADD(cutoff, hi), 0.5f);  // == (cutoff + hi) / 2.0f bit for bit
            } else {
                hi = cutoff;
                cutoff = B200_MUL(B200_ADD(cutoff, lo), 0.5f);
            }
            cnt = warp_sum_int(count_part(cutoff));
            ++guesses;
        }
        if (guesses == 10) {
            cutoff = hi;
            cnt = warp_sum_int(count_part(cutoff));
        }
        if (cnt > W) cnt = W;
    }

    if (dbg && lane == 0) dbg[3] = clock64();
    // --- keep the first W candidates >= cutoff in candidate order (beam_search.cpp:398-409) ---
    bool f[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) f[k] = valid && (s[k] >= cutoff);
    const uint32_t b0 = __ballot_sync(0xffffffffu, f[0]), b1 = __ballot_sync(0xffffffffu, f[1]);
    const uint32_t b2 = __ballot_sync(0xffffffffu, f[2]), b3 = __ballot_sync(0xffffffffu, f[3]);
    const uint32_t b4 = __ballot_sync(0xffffffffu, f[4]);
    int pos = __popc(b0 & lt_mask) + __popc(b1 & lt_mask) + __popc(b2 & lt_mask) + __popc(b3 & lt_mask);
    const int steps_total = __popc(b0) + __popc(b1) + __popc(b2) + __popc(b3);
#pragma unroll
    for (int b = 0; b < 4; ++b) {
        if (f[b]) {
            if (pos < W) {
                bs.new_score[pos] = s[b];
                bs.new_hash[pos] = hs[b];
                bs.new_meta[pos] = ns[b] | ((uint32_t)lane << 16);
            }
            ++pos;
        }
    }
    if (f[4]) {
        const int sp = steps_total + __popc(b4 & lt_mask);
        if (sp < W) {
            bs.new_score[sp] = s[4];
            bs.new_hash[sp] = me.hash;
            bs.new_meta[sp] = me.state | ((uint32_t)lane << 16) | (1u << 24);
        }
    }
    __syncwarp();

    const bool nvalid = lane < cnt;
    uint32_t meta = 0;
    if (nvalid) {
        me.score = bs.new_score[lane];
        me.hash = bs.new_hash[lane];
        meta = bs.new_meta[lane];
        me.state = meta & 0xffffu;
    }

    if (dbg && lane == 0) dbg[4] = clock64();
    // --- last block: best element to slot 0 (beam_search.cpp:413-424) ---
    if (last_block) {
        const float best = warp_max(nvalid ? me.score : B200_FLT_LOWEST);
        // reference scans ascending with a strict '>' starting from lowest(): first index holding
        // the maximum, or index 0 if every score equals lowest()
        const uint32_t eq = __ballot_sync(0xffffffffu, nvalid && me.score == best && best > B200_FLT_LOWEST);
        const int bi = eq ? (__ffs(eq) - 1) : 0;
        const int src = lane == 0 ? bi : (lane == bi ? 0 : lane);
        const float sc2 = __shfl_sync(0xffffffffu, me.score, src);
        const uint32_t h2 = __shfl_sync(0xffffffffu, me.hash, src);
        const uint32_t m2 = __shfl_sync(0xffffffffu, meta, src);
        me.score = sc2;
        me.hash = h2;
        meta = m2;
        me.state = meta & 0xffffu;
    }
    if (nvalid) {
        me.score = B200_SUB(me.score, bw_row[me.state]);
        meta_row[lane] = meta;
        prob_row[lane] = kmer_block_prob<SL>(post_row, (int)me.state);
    }
    __syncwarp();  // the next step's shared-memory writes come after every lane's reads of this one
    if (dbg && lane == 0) {
        dbg[5] = clock64();
        dbg[6] = cnt;
    }
    return cnt;
}

// bar.arrive orders the arriving thread's earlier shared-memory accesses before the barrier completes (the PTX
// producer / consumer pattern: st.shared; bar.arrive  ||  bar.sync; ld.shared), so no membar is issued here -- the
// __threadfence_block() this used to carry cost a MEMBAR.CTA per block on both sides of the hand-over.
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

template <int SL>
struct FwdCfg {
    using Scan = ScanCfg<SL>;
    static constexpr int GT = Scan::NT + 32;                 // threads per chunk: scan threads + beam warp
    static constexpr int CH = GT <= 128 ? 2 : 1;             // chunks per CTA (barrier ids: 5 per chunk)
    static constexpr int THREADS = GT * CH;
};

template <int SL>
__global__ void __launch_bounds__(FwdCfg<SL>::THREADS) crf_fwd_beam_kernel(const __half* __restrict__ scores,
                                                                          const float* __restrict__ bwd,
                                                                          uint2* __restrict__ beam,
                                                                          int N,
                                                                          int T_pitch,
                                                                          float clamp_val,
                                                                          float blank,
                                                                          int W,
                                                                          float log_beam_cut,
                                                                          const int32_t* __restrict__ lens,
                                                                          int stride,
                                                                          long long* dbg) {
    using Cfg = ScanCfg<SL>;
    using F = FwdCfg<SL>;
    constexpr int S = Cfg::S, C = Cfg::C, P4 = Cfg::P4, SPT = Cfg::SPT, NT = Cfg::NT;
    constexpr int GT = F::GT, CH = F::CH;
    constexpr int NW = NT / 32;  // scan warps per chunk
    constexpr int PF = 4;

    const int g = threadIdx.x / GT;
    const int tid = threadIdx.x % GT;
    const int lane = threadIdx.x & 31;
    const int chunk = blockIdx.x * CH + g;
    // barrier ids of this chunk group.  SCAN: the scan threads among themselves (+ the beam warp for the two start-up
    // syncs); FULL[slot]: scan threads arrive, beam warp waits; EMPTY[slot]: beam warp arrives, scan threads wait.
    const int BAR_SCAN = 1 + 5 * g, BAR_FULL = 2 + 5 * g, BAR_EMPTY = 4 + 5 * g;

    __shared__ __align__(16) float fa[CH][2][S];
    __shared__ __align__(16) __half sc_row[CH][2][C];  // clamped scores (clamping fp16 values is exact in fp16)
    __shared__ __align__(16) float bw_row[CH][2][S];
    __shared__ __align__(16) float post_row[CH][2][S];
    __shared__ float red[CH][2][NW];
    __shared__ BeamSmem bsm[CH];

    if (chunk >= N) return;  // whole chunk groups exit together; every barrier below is per group
    const int T = lens ? min(T_pitch, __ldg(lens + chunk) / stride) : T_pitch;  // variable chunk sizes
    // beam history: two planes of [N][T][32] 4-byte words, meta = (state, prev, stay) and the block probability
    uint32_t* meta_out = reinterpret_cast<uint32_t*>(beam) + (size_t)chunk * T_pitch * kBeamW;
    float* prob_out = reinterpret_cast<float*>(beam) + ((size_t)N + chunk) * T_pitch * kBeamW;

    if (tid < NT) {
        // ================= scan threads =================
        const int v = tid;  // states SPT*v .. SPT*v + SPT-1
        const int wv = v >> 5;
        const __half* srow = scores + (size_t)chunk * T_pitch * C + (size_t)v * 4 * SPT;
        const float* brow = bwd + (size_t)chunk * (T_pitch + 1) * S + (size_t)v * SPT;
        // bwd[0] for the beam initialisation, forward guide 0
#pragma unroll
        for (int e = 0; e < SPT; ++e) {
            bw_row[g][1][SPT * v + e] = brow[e];
            fa[g][0][SPT * v + e] = 0.0f;
        }
        named_bar_sync(BAR_SCAN, GT);  // (a) bwd[0] visible to the beam warp
        named_bar_sync(BAR_SCAN, GT);  // (b) beam warp has consumed it; slot 1 may be reused
        uint2 pf[PF][SPT];
        float pb[PF][SPT];
#pragma unroll
        for (int k = 0; k < PF; ++k) {
            if (k < T) {
#pragma unroll
                for (int e = 0; e < SPT; ++e) {
                    pf[k][e] = __ldg(reinterpret_cast<const uint2*>(srow + (size_t)k * C) + e);
                    pb[k][e] = __ldg(brow + (size_t)(k + 1) * S + e);
                }
            }
        }
        float f[SPT];
#pragma unroll
        for (int e = 0; e < SPT; ++e) f[e] = 0.0f;
        int cur = 0;
        for (int t0 = 0; t0 < T; t0 += PF) {
#pragma unroll
            for (int k = 0; k < PF; ++k) {
                const int t = t0 + k;
                if (t < T) {
                    const int slot = t & 1;
                    long long* d = (dbg && chunk == 0 && tid == 0 && t >= 100 && t < 108) ? dbg + (t - 100) * 16 : nullptr;
                    if (d) d[8] = clock64();
                    if (t >= 2) named_bar_sync(BAR_EMPTY + slot, GT);  // beam warp is done with this slot
                    if (d) d[9] = clock64();
                    float vsum[SPT];
                    float lmax = B200_FLT_LOWEST;
#pragma unroll
                    for (int e = 0; e < SPT; ++e) {
                        const uint2 r = pf[k][e];
                        const float bw = pb[k][e];
                        if (t + PF < T) {
                            pf[k][e] = __ldg(reinterpret_cast<const uint2*>(srow + (size_t)(t + PF) * C) + e);
                            pb[k][e] = __ldg(brow + (size_t)(t + PF + 1) * S + e);
                        }
                        const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
                        const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
                        const float s0 = clampf(f0.x, clamp_val), s1 = clampf(f0.y, clamp_val);
                        const float s2 = clampf(f1.x, clamp_val), s3 = clampf(f1.y, clamp_val);
                        const int st = SPT * v + e;
                        {
                            const __half2 c0 = __floats2half2_rn(s0, s1), c1 = __floats2half2_rn(s2, s3);
                            uint2 pk;
                            pk.x = *reinterpret_cast<const uint32_t*>(&c0);
                            pk.y = *reinterpret_cast<const uint32_t*>(&c1);
                            *reinterpret_cast<uint2*>(&sc_row[g][slot][4 * st]) = pk;
                        }
                        bw_row[g][slot][st] = bw;
                        const int p = st >> 2;
                        f[e] = b200_lse5(B200_ADD(f[e], blank), B200_ADD(fa[g][cur][p], s0), B200_ADD(fa[g][cur][p + P4], s1),
                                         B200_ADD(fa[g][cur][p + 2 * P4], s2), B200_ADD(fa[g][cur][p + 3 * P4], s3));
                        fa[g][cur ^ 1][st] = f[e];
                        vsum[e] = B200_ADD(f[e], bw);  // fwd + bwd
                        lmax = b200_fmaxf(lmax, vsum[e]);
                    }
                    float mx = warp_max(lmax);
                    if constexpr (NW > 1) {
                        if (lane == 0) red[g][0][wv] = mx;
                        named_bar_sync(BAR_SCAN, NT);
                        mx = red[g][0][0];
#pragma unroll
                        for (int w = 1; w < NW; ++w) mx = b200_fmaxf(mx, red[g][0][w]);
                    }
                    // posterior normaliser in the contract's order: per-thread left-to-right, per-warp xor butterfly,
                    // warps left to right (oracle/crf_oracle.c posts_row)
                    float ex[SPT];
                    float part = 0.0f;
#pragma unroll
                    for (int e = 0; e < SPT; ++e) {
                        ex[e] = b200_expf_nonpos(B200_SUB(vsum[e], mx));
                        part = e == 0 ? ex[0] : B200_ADD(part, ex[e]);
                    }
#pragma unroll
                    for (int o = 16; o >= 1; o >>= 1) part = B200_ADD(part, __shfl_xor_sync(0xffffffffu, part, o));
                    float z = part;
                    if constexpr (NW > 1) {
                        if (lane == 0) red[g][1][wv] = part;
                        named_bar_sync(BAR_SCAN, NT);
                        z = red[g][1][0];
#pragma unroll
                        for (int w = 1; w < NW; ++w) z = B200_ADD(z, red[g][1][w]);
                    }
#pragma unroll
                    for (int e = 0; e < SPT; ++e) post_row[g][slot][SPT * v + e] = B200_DIV(ex[e], z);
                    named_bar_arrive(BAR_FULL + slot, GT);  // slot t is complete
                    if (d) d[10] = clock64();
                    cur ^= 1;
                }
            }
        }
    } else {
        // ================= beam warp =================
        named_bar_sync(BAR_SCAN, GT);  // (a)
        BeamLane me{0u, 0u, 0.0f};
        int width = beam_init<SL>(bw_row[g][1], bsm[g], me, W, lane);
        named_bar_sync(BAR_SCAN, GT);  // (b)
        for (int t = 0; t < T; ++t) {
            const int slot = t & 1;
            long long* d = (dbg && chunk == 0 && t >= 100 && t < 108) ? dbg + (t - 100) * 16 : nullptr;
            if (d && lane == 0) d[7] = clock64();
            named_bar_sync(BAR_FULL + slot, GT);
            width = beam_step<SL>(sc_row[g][slot], bw_row[g][slot], post_row[g][slot], bsm[g], me, width, W, log_beam_cut, blank,
                                  t == T - 1, meta_out + (size_t)t * kBeamW, prob_out + (size_t)t * kBeamW, lane, d);
            if (t + 2 < T) named_bar_arrive(BAR_EMPTY + slot, GT);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Kernel 3: traceback + sequence / qstring generation (beam_search.cpp:447-455, :54-102).
// One warp per chunk.  The pointer chase only needs the 4-byte (state, prev, stay) words, so the beam history is two planes
// (meta, prob) and the chase streams the meta plane alone, in tiles of 32 blocks: while lane 0 walks one tile in shared
// memory the next tile's 32 rows are already in flight (one register per row and lane).  The block probabilities are then
// gathered along the chosen path only (one 4-byte load per block, all independent).
// ------------------------------------------------------------------------------------------------
constexpr int kTbTile = 32;
constexpr int kTbWarps = 2;

__host__ __device__ constexpr size_t traceback_warp_bytes(int T) {
    return ((size_t)kTbTile * kBeamW * 4 + (size_t)((T + 3) & ~3) * (4 + 4 + 2) + 16 + 15) & ~(size_t)15;
}

__global__ void __launch_bounds__(kTbWarps * 32) crf_traceback_kernel(const uint32_t* __restrict__ beam_meta,
                                                                      const float* __restrict__ beam_prob,
                                                                      int N,
                                                                      int T_pitch,
                                                                      const int32_t* __restrict__ lens,
                                                                      int stride,
                                                                      const b200_qtable* __restrict__ qtable,
                                                                      uint8_t* __restrict__ moves_out,
                                                                      char* __restrict__ seq_out,
                                                                      char* __restrict__ qstr_out,
                                                                      int32_t* __restrict__ n_bases_out) {
    extern __shared__ __align__(16) unsigned char tb_smem[];
    __shared__ b200_qtable qt;  // quality-character quantiser (bin edges placed by the host, b200_crf_math.h)
    for (int i = threadIdx.x; i < (int)(sizeof(b200_qtable) / 4); i += blockDim.x) {
        reinterpret_cast<uint32_t*>(&qt)[i] = reinterpret_cast<const uint32_t*>(qtable)[i];
    }
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunk = blockIdx.x * kTbWarps + w;
    if (chunk >= N) return;
    const int T = lens ? min(T_pitch, __ldg(lens + chunk) / stride) : T_pitch;  // variable chunk sizes
    const int Tp = (T_pitch + 3) & ~3;
    // per-warp carve-up
    unsigned char* base = tb_smem + (size_t)w * traceback_warp_bytes(T_pitch);
    uint32_t* tile = reinterpret_cast<uint32_t*>(base);                         // [32 blocks][32 elements]
    uint32_t* path = tile + kTbTile * kBeamW;                                   // state | move << 16 | element << 24
    float* pprob = reinterpret_cast<float*>(path + Tp);
    uint16_t* bstart = reinterpret_cast<uint16_t*>(pprob + Tp);

    const uint32_t* mrow = beam_meta + (size_t)chunk * T_pitch * kBeamW + lane;
    uint32_t nxt[kTbTile];
    auto load_tile = [&](int t_hi) {  // rows t_hi-32 .. t_hi-1 (those >= 0), row r of the tile in nxt[r]
        const int t_lo = t_hi - kTbTile;
#pragma unroll
        for (int r = 0; r < kTbTile; ++r) {
            const int t = t_lo + r;
            nxt[r] = t >= 0 ? __ldg(mrow + (size_t)t * kBeamW) : 0u;
        }
    };
    if (T > 0) load_tile(T);
    uint32_t ei = 0;
    for (int t_hi = T; t_hi > 0; t_hi -= kTbTile) {
#pragma unroll
        for (int r = 0; r < kTbTile; ++r) tile[r * kBeamW + lane] = nxt[r];
        __syncwarp();
        if (t_hi - kTbTile > 0) load_tile(t_hi - kTbTile);  // in flight during the walk below
        if (lane == 0) {
            const int t_lo = t_hi - kTbTile;
            const int r_lo = t_lo < 0 ? -t_lo : 0;
            for (int r = kTbTile - 1; r >= r_lo; --r) {
                const uint32_t e = tile[r * kBeamW + ei];
                path[t_lo + r] = (e & 0xffffu) | ((((e >> 24) & 1u) ^ 1u) << 16) | (ei << 24);
                ei = (e >> 16) & 0xffu;
            }
        }
        __syncwarp();
    }
    if (lane == 0 && T > 0) path[0] |= 1u << 16;  // always step in the first block
    __syncwarp();
    {
        const float* prow = beam_prob + (size_t)chunk * T_pitch * kBeamW;
        for (int t = lane; t < T; t += 32) {  // "power fudge factor", beam_search.cpp:503
            pprob[t] = b200_pow0p4f(__ldg(prow + (size_t)t * kBeamW + (path[t] >> 24)));
        }
    }
    __syncwarp();

    // base start blocks
    int nb = 0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const int t = t0 + lane;
        const bool m = t < T && ((path[t] >> 16) & 1u);
        const uint32_t bal = __ballot_sync(0xffffffffu, m);
        if (m) bstart[nb + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)t;
        nb += __popc(bal);
    }
    if (lane == 0) bstart[nb] = (uint16_t)T;
    __syncwarp();

    uint8_t* mo = moves_out + (size_t)chunk * T_pitch;
    char* so = seq_out + (size_t)chunk * T_pitch;
    char* qo = qstr_out + (size_t)chunk * T_pitch;
    for (int t = lane; t < T_pitch; t += 32) mo[t] = t < T ? (uint8_t)((path[t] >> 16) & 1u) : 0;
    for (int p = lane; p < T_pitch; p += 32) {
        char sc = 0, qc = 0;
        if (p < nb) {
            const int b0 = bstart[p], b1 = bstart[p + 1];
            float bp = 0.0f, tp = 0.0f;
            int base = 0;
            for (int blk = b0; blk < b1; ++blk) {
                base = path[blk] & 3;
                const float prob = pprob[blk];
                const float wrong = B200_DIV(B200_SUB(1.0f, prob), 3.0f);
                bp = B200_ADD(bp, prob);
#pragma unroll
                for (int k = 0; k < 4; ++k) tp = B200_ADD(tp, k == base ? prob : wrong);
            }
            sc = "ACGT"[path[b0] & 3];
            qc = b200_qtable_lookup(&qt, bp, tp);
        }
        so[p] = sc;
        qo[p] = qc;
    }
    if (lane == 0) n_bases_out[chunk] = nb;
}

size_t traceback_smem_bytes(int T) { return kTbWarps * traceback_warp_bytes(T); }

template <int SL>
void launch_decode(const DecodeArgs& a, cudaStream_t stream, ProfileSink* prof) {
    {
        constexpr int S = Dims<SL>::S;
        constexpr int CH = S >= 256 ? 1 : 256 / S;
        const int grid = (a.N + CH - 1) / CH;
        NvtxRange r("back_guides");
        crf_bwd_scan_kernel<SL><<<grid, S * CH, 0, stream>>>(a.scores, a.bwd, a.N, a.T, a.clamp_val, a.blank, a.lens, a.stride);
        if (prof) prof->mark("crf_bwd_scan", stream);
    }
    {
        using F = FwdCfg<SL>;
        const int grid = (a.N + F::CH - 1) / F::CH;
        NvtxRange r("beam_search");  // forward scan + posteriors (the reference's "compute_posts") are fused in
        crf_fwd_beam_kernel<SL><<<grid, F::THREADS, 0, stream>>>(a.scores, a.bwd, a.beam, a.N, a.T, a.clamp_val, a.blank,
                                                                   a.beam_width, a.log_beam_cut, a.lens, a.stride, a.dbg);
        if (prof) prof->mark("crf_fwd_beam", stream);
    }
    {
        const size_t smem = traceback_smem_bytes(a.T);
        if (smem > 48 * 1024) ensure_dynamic_smem(crf_traceback_kernel, 200 * 1024);
        const int grid = (a.N + kTbWarps - 1) / kTbWarps;
        NvtxRange r("decode");
        const uint32_t* meta = reinterpret_cast<const uint32_t*>(a.beam);
        const float* prob = reinterpret_cast<const float*>(a.beam) + (size_t)a.N * a.T * kBeamW;
        crf_traceback_kernel<<<grid, kTbWarps * 32, smem, stream>>>(meta, prob, a.N, a.T, a.lens, a.stride, a.qtable, a.moves,
                                                                    a.sequence, a.qstring, a.n_bases);
        if (prof) prof->mark("crf_traceback", stream);
    }
    B200_CUDA(cudaGetLastError());
}

}  // namespace

size_t decode_max_blocks() {
    int T = 65535;
    while (traceback_smem_bytes(T) > 200 * 1024) T -= 64;
    return (size_t)T;
}

size_t decode_scratch_bytes(int N, int T, int state_len, size_t* bwd_bytes, size_t* beam_bytes) {
    const size_t S = (size_t)1 << (2 * state_len);
    const size_t b1 = ((size_t)N * (T + 1) * S * sizeof(float) + 255) & ~(size_t)255;
    const size_t b2 = ((size_t)N * T * kBeamW * sizeof(uint2) + 255) & ~(size_t)255;
    if (bwd_bytes) *bwd_bytes = b1;
    if (beam_bytes) *beam_bytes = b2;
    return b1 + b2;
}

void decode_scores(const DecodeArgs& a, cudaStream_t stream, ProfileSink* prof) {
    if (a.beam_width < 1 || a.beam_width > kBeamW) {
        throw std::invalid_argument("b200 decode: beam_width must be in [1, 32]");
    }
    if (a.T < 1 || a.T > 65535 || a.N < 1) {
        throw std::invalid_argument("b200 decode: need 1 <= T <= 65535 and N >= 1");
    }
    if (!a.qtable) throw std::invalid_argument("b200 decode: quality table missing");
    if (a.lens && a.stride < 1) throw std::invalid_argument("b200 decode: chunk lengths need the model stride");
    if (traceback_smem_bytes(a.T) > 200 * 1024) {
        throw std::invalid_argument("b200 decode: " + std::to_string(a.T) + " blocks per chunk exceed what the traceback kernel "
                                    "holds in shared memory (about 10 700); use a smaller chunk size");
    }
    switch (a.state_len) {
        case 3: launch_decode<3>(a, stream, prof); break;
        case 4: launch_decode<4>(a, stream, prof); break;
        case 5: launch_decode<5>(a, stream, prof); break;
        default: throw std::invalid_argument("b200 decode: state_len must be 3, 4 or 5");
    }
}

}  // namespace b200
