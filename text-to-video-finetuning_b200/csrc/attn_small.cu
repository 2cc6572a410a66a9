// Self-attention along the frame axis for TransformerTemporalModel: attn_small (L <= 32, a warp per sequence) and attn_long
// (L <= 256, a CTA per sequence, below).
//
// The reference permutes (B,C,F,H,W) -> (B*H*W, F, C) before this attention (diffusers TransformerTemporalModel,
// wired at unet_3d_blocks.py:331-340,491-500 and unet_3d_condition.py:147-152).  Here activations stay in the
// frames-major token order [B][F][H*W][C]; a sequence is addressed with strides instead (SeqAddr), so both permute
// copies disappear, and q / k / v may be column slices of one fused [rows][3C] projection.
//
// One warp owns one (sequence, head).  The tiles are 16 x 64 (L x D): far below one wgmma instruction (M = 64), so
// the four small products run on warp-level tensor-core MMAs (mma.sync m16n8k16, bf16 in / fp32 accumulate) fed by
// ldmatrix from shared memory; softmax and its gradient stay in the accumulator registers.  Global traffic is 16-byte
// coalesced in both directions (q, k, v, dO read once; o / dq, dk, dv written once): the kernel is HBM-bound.
#include "common.h"
#include "mma_sync.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cuda_bf16.h>

namespace t2v {
using namespace wmma16;   // ldmatrix / mma.sync fragment helpers (mma_sync.cuh)

constexpr int kMaxL = 32;

// Sequence addressing in ROWS of a token matrix; q/k/v (and their gradients) have row pitch ld_in - which lets them be
// column slices of one fused [rows][3C] QKV projection - while o / dO have row pitch ld_out.
struct SeqAddr {
    int64_t outer_rows, inner_rows, seq_rows;
    int64_t ld_in, ld_out;
    int32_t inner;
};

__device__ __forceinline__ int64_t seq_row(const SeqAddr& a, int64_t z) {
    return (z / a.inner) * a.outer_rows + (z % a.inner) * a.inner_rows;
}


// global [L rows x D] (row stride `stride` elements) -> shared [LP][D + 8] bf16; rows >= L stay zero (filled once at start)
template <int D>
__device__ __forceinline__ void load_tile(const __nv_bfloat16* __restrict__ g, int64_t base, int64_t stride, int L, uint8_t* sm, int lane) {
    constexpr int CPT = D / 8, PITCH = (D + 8) * 2;
    const int total = L * CPT;
#pragma unroll 4
    for (int idx = lane; idx < total; idx += 32) {
        const int t = idx / CPT, c = idx % CPT;
        *reinterpret_cast<uint4*>(sm + t * PITCH + c * 16) = __ldg(reinterpret_cast<const uint4*>(g + base + t * stride) + c);
    }
}
template <int D>
__device__ __forceinline__ void store_tile(__nv_bfloat16* __restrict__ g, int64_t base, int64_t stride, int L, const uint8_t* sm, int lane) {
    constexpr int CPT = D / 8, PITCH = (D + 8) * 2;
    const int total = L * CPT;
#pragma unroll 4
    for (int idx = lane; idx < total; idx += 32) {
        const int t = idx / CPT, c = idx % CPT;
        *(reinterpret_cast<uint4*>(g + base + t * stride) + c) = *reinterpret_cast<const uint4*>(sm + t * PITCH + c * 16);
    }
}
// accumulator tile (rows m0.. of a [LP][N] result) -> bf16 staging
template <int N>
__device__ __forceinline__ void stage_acc(const float (&acc)[N / 8][4], uint8_t* sm, int pitch, int m0, int lane) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < N / 8; ++nt) {
        *reinterpret_cast<uint32_t*>(sm + (m0 + g) * pitch + (nt * 8 + 2 * t) * 2) = pack_bf16(acc[nt][0], acc[nt][1]);
        *reinterpret_cast<uint32_t*>(sm + (m0 + g + 8) * pitch + (nt * 8 + 2 * t) * 2) = pack_bf16(acc[nt][2], acc[nt][3]);
    }
}

// Row softmax of a 16 x LP score tile held in accumulator layout (columns >= L masked); returns P in place.
template <int LP>
__device__ __forceinline__ void softmax_rows(float (&s)[LP / 8][4], int L, float scale, int lane) {
    const int t = lane & 3;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < LP / 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int j = nt * 8 + 2 * t + (e & 1);
            s[nt][e] = j < L ? s[nt][e] * scale : -INFINITY;
            mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
        }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < LP / 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            s[nt][e] = __expf(s[nt][e] - mx[e >> 1]);
            sum[e >> 1] += s[nt][e];
        }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
        sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
        sum[h] = 1.0f / sum[h];
    }
#pragma unroll
    for (int nt = 0; nt < LP / 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[nt][e] *= sum[e >> 1];
}

template <int D, int LP>
struct AttnSmem {
    static constexpr int kTilePitch = (D + 8) * 2;            // bytes per row of a [LP][D] tile (conflict-free ldmatrix)
    static constexpr int kTileBytes = LP * kTilePitch;
    static constexpr int kProbPitch = (LP + 8) * 2;
    static constexpr int kProbBytes = LP * kProbPitch;
    static constexpr int kFwdBytes = 4 * kTileBytes;                    // q, k, v, staging
    static constexpr int kBwdBytes = 5 * kTileBytes + 2 * kProbBytes;   // q, k, v, dO, staging, P, dS
};

template <int D, int LP>
__global__ void attn_small_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                      const __nv_bfloat16* __restrict__ v, __nv_bfloat16* __restrict__ o, SeqAddr a, int64_t nseq,
                                      int heads, int L, float scale) {
    pdl_sync();
    using S = AttnSmem<D, LP>;
    extern __shared__ __align__(16) uint8_t sm_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* sq = sm_all + warp * S::kFwdBytes;
    uint8_t* sk = sq + S::kTileBytes;
    uint8_t* sv = sk + S::kTileBytes;
    uint8_t* so = sv + S::kTileBytes;
    for (int i = lane; i < S::kFwdBytes / 16; i += 32) reinterpret_cast<uint4*>(sq)[i] = make_uint4(0, 0, 0, 0);
    const uint32_t aq = smem_u32(sq), ak = smem_u32(sk), av = smem_u32(sv);
    const int nwarps = blockDim.x >> 5;
    const int64_t total = nseq * heads;
    for (int64_t w = blockIdx.x * int64_t(nwarps) + warp; w < total; w += int64_t(gridDim.x) * nwarps) {
        const int64_t z = w / heads;
        const int h = int(w % heads);
        const int64_t row0 = seq_row(a, z);
        const int64_t base = row0 * a.ld_in + int64_t(h) * D, sstr = a.seq_rows * a.ld_in;
        const int64_t obase = row0 * a.ld_out + int64_t(h) * D, ostr = a.seq_rows * a.ld_out;
        __syncwarp();
        load_tile<D>(q, base, sstr, L, sq, lane);
        load_tile<D>(k, base, sstr, L, sk, lane);
        load_tile<D>(v, base, sstr, L, sv, lane);
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < LP / 16; ++mt) {
            if (mt * 16 >= L) break;
            float s[LP / 8][4];
#pragma unroll
            for (int nt = 0; nt < LP / 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            warp_mma<LP, D, false, false>(s, aq, S::kTilePitch, mt * 16, ak, S::kTilePitch, lane);  // S = Q K^T
            softmax_rows<LP>(s, L, scale, lane);
            float oacc[D / 8][4];
#pragma unroll
            for (int nt = 0; nt < D / 8; ++nt) oacc[nt][0] = oacc[nt][1] = oacc[nt][2] = oacc[nt][3] = 0.f;
#pragma unroll
            for (int kt = 0; kt < LP / 16; ++kt) {  // O = P V: the score accumulators ARE the A fragments of P
                uint32_t pa[4];
                pa[0] = pack_bf16(s[2 * kt][0], s[2 * kt][1]);
                pa[1] = pack_bf16(s[2 * kt][2], s[2 * kt][3]);
                pa[2] = pack_bf16(s[2 * kt + 1][0], s[2 * kt + 1][1]);
                pa[3] = pack_bf16(s[2 * kt + 1][2], s[2 * kt + 1][3]);
#pragma unroll
                for (int np = 0; np < D / 16; ++np) {
                    uint32_t b[4];
                    load_b2<true>(av, S::kTilePitch, np * 16, kt * 16, lane, b);
                    mma_bf16(oacc[2 * np], pa, b[0], b[1]);
                    mma_bf16(oacc[2 * np + 1], pa, b[2], b[3]);
                }
            }
            stage_acc<D>(oacc, so, S::kTilePitch, mt * 16, lane);
        }
        __syncwarp();
        store_tile<D>(o, obase, ostr, L, so, lane);
    }
}

// Backward: per 16-row block recompute P, form dP = dO V^T and dS = P o (dP - rowsum(P o dP)) * scale in registers, park
// P and dS (bf16) in shared memory, then dQ = dS K, dK = dS^T Q, dV = P^T dO (transposed operands via ldmatrix.trans).
template <int D, int LP>
__global__ void attn_small_bwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                      const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ dout,
                                      __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv,
                                      SeqAddr a, int64_t nseq, int heads, int L, float scale) {
    pdl_sync();
    using S = AttnSmem<D, LP>;
    extern __shared__ __align__(16) uint8_t sm_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* sq = sm_all + warp * S::kBwdBytes;
    uint8_t* sk = sq + S::kTileBytes;
    uint8_t* sv = sk + S::kTileBytes;
    uint8_t* sd = sv + S::kTileBytes;
    uint8_t* so = sd + S::kTileBytes;
    uint8_t* sp = so + S::kTileBytes;
    uint8_t* ss = sp + S::kProbBytes;
    for (int i = lane; i < S::kBwdBytes / 16; i += 32) reinterpret_cast<uint4*>(sq)[i] = make_uint4(0, 0, 0, 0);
    const uint32_t aq = smem_u32(sq), ak = smem_u32(sk), av = smem_u32(sv), ad = smem_u32(sd), ap = smem_u32(sp), as = smem_u32(ss);
    const int nwarps = blockDim.x >> 5;
    const int64_t total = nseq * heads;
    const int g = lane >> 2, t = lane & 3;
    for (int64_t w = blockIdx.x * int64_t(nwarps) + warp; w < total; w += int64_t(gridDim.x) * nwarps) {
        const int64_t z = w / heads;
        const int h = int(w % heads);
        const int64_t row0 = seq_row(a, z);
        const int64_t base = row0 * a.ld_in + int64_t(h) * D, sstr = a.seq_rows * a.ld_in;
        const int64_t obase = row0 * a.ld_out + int64_t(h) * D, ostr = a.seq_rows * a.ld_out;
        __syncwarp();
        load_tile<D>(q, base, sstr, L, sq, lane);
        load_tile<D>(k, base, sstr, L, sk, lane);
        load_tile<D>(v, base, sstr, L, sv, lane);
        load_tile<D>(dout, obase, ostr, L, sd, lane);
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < LP / 16; ++mt) {
            float s[LP / 8][4], dp[LP / 8][4];
#pragma unroll
            for (int nt = 0; nt < LP / 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) s[nt][e] = dp[nt][e] = 0.f;
            warp_mma<LP, D, false, false>(s, aq, S::kTilePitch, mt * 16, ak, S::kTilePitch, lane);   // S  = Q K^T
            warp_mma<LP, D, false, false>(dp, ad, S::kTilePitch, mt * 16, av, S::kTilePitch, lane);  // dP = dO V^T
            softmax_rows<LP>(s, L, scale, lane);
            float dot[2] = {0.f, 0.f};
#pragma unroll
            for (int nt = 0; nt < LP / 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) dot[e >> 1] += s[nt][e] * dp[nt][e];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                dot[hh] += __shfl_xor_sync(0xffffffffu, dot[hh], 1);
                dot[hh] += __shfl_xor_sync(0xffffffffu, dot[hh], 2);
            }
#pragma unroll
            for (int nt = 0; nt < LP / 8; ++nt) {
                const int col = (nt * 8 + 2 * t) * 2;
                const int r0 = (mt * 16 + g) * S::kProbPitch, r1 = (mt * 16 + g + 8) * S::kProbPitch;
                *reinterpret_cast<uint32_t*>(sp + r0 + col) = pack_bf16(s[nt][0], s[nt][1]);
                *reinterpret_cast<uint32_t*>(sp + r1 + col) = pack_bf16(s[nt][2], s[nt][3]);
                *reinterpret_cast<uint32_t*>(ss + r0 + col) =
                    pack_bf16(s[nt][0] * (dp[nt][0] - dot[0]) * scale, s[nt][1] * (dp[nt][1] - dot[0]) * scale);
                *reinterpret_cast<uint32_t*>(ss + r1 + col) =
                    pack_bf16(s[nt][2] * (dp[nt][2] - dot[1]) * scale, s[nt][3] * (dp[nt][3] - dot[1]) * scale);
            }
        }
        __syncwarp();
        // three [LP x D] results, each staged to shared memory and written with coalesced 16-byte stores
#pragma unroll
        for (int which = 0; which < 3; ++which) {
#pragma unroll
            for (int mt = 0; mt < LP / 16; ++mt) {
                if (mt * 16 >= L) break;
                float acc[D / 8][4];
#pragma unroll
                for (int nt = 0; nt < D / 8; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
                if (which == 0) warp_mma<D, LP, false, true>(acc, as, S::kProbPitch, mt * 16, ak, S::kTilePitch, lane);      // dQ = dS K
                else if (which == 1) warp_mma<D, LP, true, true>(acc, as, S::kProbPitch, mt * 16, aq, S::kTilePitch, lane);  // dK = dS^T Q
                else warp_mma<D, LP, true, true>(acc, ap, S::kProbPitch, mt * 16, ad, S::kTilePitch, lane);                  // dV = P^T dO
                stage_acc<D>(acc, so, S::kTilePitch, mt * 16, lane);
            }
            __syncwarp();
            store_tile<D>(which == 0 ? dq : (which == 1 ? dk : dv), base, sstr, L, so, lane);
            __syncwarp();
        }
    }
}

// ---------------------------------------------------------------------------------------------- long sequences (L <= 256)
// One CTA owns one (sequence, head); the whole sequence sits in shared memory as [LP][D + 8] tiles with LP = L rounded up to
// 64 (rows >= L are zero).  Each warp owns 16-row blocks; the other operand is walked in 64-row tiles so the register count
// does not depend on L.  Scores are kept in the log2 domain (s * scale * log2 e); lse is the natural-log row logsumexp.
constexpr int kLongMaxL = 256;
constexpr int kLongWarps = 8;
constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;

// global [L rows x D] -> shared [.][D + 8], all threads of the CTA
template <int D>
__device__ __forceinline__ void cta_load_tile(const __nv_bfloat16* __restrict__ g, int64_t base, int64_t stride, int L, uint8_t* sm) {
    constexpr int CPT = D / 8, PITCH = (D + 8) * 2;
    const int total = L * CPT;
    for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
        const int t = idx / CPT, c = idx % CPT;
        *reinterpret_cast<uint4*>(sm + t * PITCH + c * 16) = __ldg(reinterpret_cast<const uint4*>(g + base + t * stride) + c);
    }
}

// 16 x 64 score / probability accumulators -> the four A fragments of a k = 64 product (as in attn_small_fwd_kernel)
__device__ __forceinline__ void acc_to_a(const float (&s)[8][4], int kk, uint32_t (&pa)[4]) {
    pa[0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
    pa[1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
    pa[2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
    pa[3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
}

template <int D>
struct LongSmem {
    static constexpr int kPitch = (D + 8) * 2;
    __host__ __device__ static int tile(int LP) { return LP * kPitch; }
    __host__ __device__ static int fwd(int LP) { return 3 * tile(LP); }   // q (then o), k, v
    __host__ __device__ static int bwd(int LP, int warps) {                // q, k, v, dO, lse, delta, dK/dV staging
        return 4 * tile(LP) + 2 * LP * 4 + warps * 16 * kPitch;
    }
};

// Forward: per 16-query block, online softmax over 64-key tiles; O is staged into the block's own q rows.
template <int D>
__global__ void __launch_bounds__(kLongWarps * 32) attn_long_fwd_kernel(
    const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
    __nv_bfloat16* __restrict__ o, float* __restrict__ lse, SeqAddr a, int64_t nseq, int heads, int L, int LP, float scale_log2) {
    pdl_sync();
    constexpr int PITCH = LongSmem<D>::kPitch;
    extern __shared__ __align__(16) uint8_t sm_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int t = lane & 3, g = lane >> 2;
    uint8_t* sq = sm_all;
    uint8_t* sk = sq + LP * PITCH;
    uint8_t* sv = sk + LP * PITCH;
    for (int i = threadIdx.x; i < LongSmem<D>::fwd(LP) / 16; i += blockDim.x) reinterpret_cast<uint4*>(sm_all)[i] = make_uint4(0, 0, 0, 0);
    const uint32_t aq = smem_u32(sq), ak = smem_u32(sk), av = smem_u32(sv);
    const int nq = (L + 15) / 16, nk = (L + 63) / 64;
    const int64_t total = nseq * heads;
    for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
        const int64_t z = w / heads;
        const int h = int(w % heads);
        const int64_t row0 = seq_row(a, z);
        const int64_t base = row0 * a.ld_in + int64_t(h) * D, sstr = a.seq_rows * a.ld_in;
        const int64_t obase = row0 * a.ld_out + int64_t(h) * D, ostr = a.seq_rows * a.ld_out;
        __syncthreads();
        cta_load_tile<D>(q, base, sstr, L, sq);
        cta_load_tile<D>(k, base, sstr, L, sk);
        cta_load_tile<D>(v, base, sstr, L, sv);
        __syncthreads();
        for (int mt = warp; mt < nq; mt += nwarps) {
            float oacc[D / 8][4];
#pragma unroll
            for (int nt = 0; nt < D / 8; ++nt) oacc[nt][0] = oacc[nt][1] = oacc[nt][2] = oacc[nt][3] = 0.f;
            float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
            for (int kt = 0; kt < nk; ++kt) {
                float s[8][4];
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
                warp_mma<64, D, false, false>(s, aq, PITCH, mt * 16, ak + kt * 64 * PITCH, PITCH, lane);   // S = Q K^T
                float mx[2] = {m[0], m[1]};
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int j = kt * 64 + nt * 8 + 2 * t + (e & 1);
                        s[nt][e] = j < L ? s[nt][e] * scale_log2 : -INFINITY;
                        mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
                    }
                float corr[2];
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
                    mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
                    corr[hh] = exp2f(m[hh] - mx[hh]);   // 0 on the first tile (m = -inf); every tile has a valid key
                    m[hh] = mx[hh];
                    l[hh] *= corr[hh];
                }
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        s[nt][e] = exp2f(s[nt][e] - m[e >> 1]);
                        l[e >> 1] += s[nt][e];
                    }
#pragma unroll
                for (int nt = 0; nt < D / 8; ++nt) {
                    oacc[nt][0] *= corr[0], oacc[nt][1] *= corr[0];
                    oacc[nt][2] *= corr[1], oacc[nt][3] *= corr[1];
                }
                const uint32_t avt = av + kt * 64 * PITCH;
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {   // O += P V
                    uint32_t pa[4];
                    acc_to_a(s, kk, pa);
#pragma unroll
                    for (int np = 0; np < D / 16; ++np) {
                        uint32_t b[4];
                        load_b2<true>(avt, PITCH, np * 16, kk * 16, lane, b);
                        mma_bf16(oacc[2 * np], pa, b[0], b[1]);
                        mma_bf16(oacc[2 * np + 1], pa, b[2], b[3]);
                    }
                }
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
                l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
            }
            const float inv0 = 1.0f / l[0], inv1 = 1.0f / l[1];
#pragma unroll
            for (int nt = 0; nt < D / 8; ++nt) {
                oacc[nt][0] *= inv0, oacc[nt][1] *= inv0;
                oacc[nt][2] *= inv1, oacc[nt][3] *= inv1;
            }
            const int r = mt * 16 + g;
            if (t == 0 && r < L) lse[w * L + r] = (m[0] + __log2f(l[0])) * kLn2;
            if (t == 0 && r + 8 < L) lse[w * L + r + 8] = (m[1] + __log2f(l[1])) * kLn2;
            __syncwarp();   // this warp's q rows are dead: stage O over them
            stage_acc<D>(oacc, sq, PITCH, mt * 16, lane);
            __syncwarp();
            store_tile<D>(o, obase + int64_t(mt * 16) * ostr, ostr, min(16, L - mt * 16), sq + mt * 16 * PITCH, lane);
        }
    }
}

// Backward, one pass over HBM and no atomics.  delta = rowsum(dO o O) is read from the forward's O (one extra L x D read,
// instead of a second P V product per row block).
//   phase 1, per 16-key block:   P^T = exp2(K Q^T - lse), dS^T = P^T o (V dO^T - delta) * scale over 64-query tiles;
//                                dV = P^T dO, dK = dS^T Q accumulate in registers, staged per warp and written.
//   phase 2, per 16-query block: P, dS the same way over 64-key tiles; dQ = dS K, staged over the block's own q rows.
// Padding rows (>= L) of q / dO get lse = +inf (P = 0); those of k / v are zero, so masked keys contribute nothing to dQ.
template <int D>
__global__ void __launch_bounds__(kLongWarps * 32) attn_long_bwd_kernel(
    const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v,
    const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
    __nv_bfloat16* __restrict__ dq, __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv, SeqAddr a, int64_t nseq,
    int heads, int L, int LP, float scale, float scale_log2) {
    pdl_sync();
    constexpr int PITCH = LongSmem<D>::kPitch, TPR = D / 8;
    extern __shared__ __align__(16) uint8_t sm_all[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int t = lane & 3, g = lane >> 2;
    uint8_t* sq = sm_all;
    uint8_t* sk = sq + LP * PITCH;
    uint8_t* sv = sk + LP * PITCH;
    uint8_t* sd = sv + LP * PITCH;
    float* slse = reinterpret_cast<float*>(sd + LP * PITCH);   // lse * log2 e
    float* sdel = slse + LP;
    uint8_t* sst = reinterpret_cast<uint8_t*>(sdel + LP) + warp * 16 * PITCH;
    for (int i = threadIdx.x; i < LongSmem<D>::bwd(LP, nwarps) / 16; i += blockDim.x)
        reinterpret_cast<uint4*>(sm_all)[i] = make_uint4(0, 0, 0, 0);
    const uint32_t aq = smem_u32(sq), ak = smem_u32(sk), av = smem_u32(sv), ad = smem_u32(sd);
    const int n16 = (L + 15) / 16, n64 = (L + 63) / 64;
    const int64_t total = nseq * heads;
    for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
        const int64_t z = w / heads;
        const int h = int(w % heads);
        const int64_t row0 = seq_row(a, z);
        const int64_t base = row0 * a.ld_in + int64_t(h) * D, sstr = a.seq_rows * a.ld_in;
        const int64_t obase = row0 * a.ld_out + int64_t(h) * D, ostr = a.seq_rows * a.ld_out;
        __syncthreads();
        cta_load_tile<D>(q, base, sstr, L, sq);
        cta_load_tile<D>(k, base, sstr, L, sk);
        cta_load_tile<D>(v, base, sstr, L, sv);
        cta_load_tile<D>(dout, obase, ostr, L, sd);
        // delta and lse: TPR threads per row, 8 columns each (rows are warp-uniform per iteration, so the shuffles are safe)
        for (int r0 = 0; r0 < LP; r0 += blockDim.x / TPR) {
            const int r = r0 + int(threadIdx.x) / TPR, c = int(threadIdx.x) % TPR;
            float acc = 0.f;
            if (r < L) {
                const int64_t off = obase + int64_t(r) * ostr + c * 8;
                const uint4 ov = __ldg(reinterpret_cast<const uint4*>(o + off)), dv4 = __ldg(reinterpret_cast<const uint4*>(dout + off));
                const __nv_bfloat162* o2 = reinterpret_cast<const __nv_bfloat162*>(&ov);
                const __nv_bfloat162* d2 = reinterpret_cast<const __nv_bfloat162*>(&dv4);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 of = __bfloat1622float2(o2[i]), df = __bfloat1622float2(d2[i]);
                    acc = fmaf(of.x, df.x, fmaf(of.y, df.y, acc));
                }
            }
#pragma unroll
            for (int off = 1; off < TPR; off <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
            if (c == 0 && r < LP) {
                sdel[r] = acc;
                slse[r] = r < L ? lse[w * L + r] * kLog2e : INFINITY;
            }
        }
        __syncthreads();
        // ---- phase 1: dK, dV per 16-key block
        for (int bt = warp; bt < n16; bt += nwarps) {
            const int n0 = bt * 16;
            float dka[D / 8][4], dva[D / 8][4];
#pragma unroll
            for (int nt = 0; nt < D / 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) dka[nt][e] = dva[nt][e] = 0.f;
            for (int qt = 0; qt < n64; ++qt) {
                float st[8][4], dpt[8][4];
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) st[nt][e] = dpt[nt][e] = 0.f;
                const uint32_t aqt = aq + qt * 64 * PITCH, adt = ad + qt * 64 * PITCH;
                warp_mma<64, D, false, false>(st, ak, PITCH, n0, aqt, PITCH, lane);    // S^T  = K Q^T
                warp_mma<64, D, false, false>(dpt, av, PITCH, n0, adt, PITCH, lane);   // dP^T = V dO^T
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int i = qt * 64 + nt * 8 + 2 * t + (e & 1);
                        const float p = exp2f(st[nt][e] * scale_log2 - slse[i]);
                        st[nt][e] = p;
                        dpt[nt][e] = p * (dpt[nt][e] - sdel[i]) * scale;
                    }
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    uint32_t pa[4], da[4];
                    acc_to_a(st, kk, pa);
                    acc_to_a(dpt, kk, da);
#pragma unroll
                    for (int np = 0; np < D / 16; ++np) {
                        uint32_t b[4];
                        load_b2<true>(adt, PITCH, np * 16, kk * 16, lane, b);   // dV += P^T dO
                        mma_bf16(dva[2 * np], pa, b[0], b[1]);
                        mma_bf16(dva[2 * np + 1], pa, b[2], b[3]);
                        load_b2<true>(aqt, PITCH, np * 16, kk * 16, lane, b);   // dK += dS^T Q
                        mma_bf16(dka[2 * np], da, b[0], b[1]);
                        mma_bf16(dka[2 * np + 1], da, b[2], b[3]);
                    }
                }
            }
            const int rows = min(16, L - n0);
            stage_acc<D>(dka, sst, PITCH, 0, lane);
            __syncwarp();
            store_tile<D>(dk, base + int64_t(n0) * sstr, sstr, rows, sst, lane);
            __syncwarp();
            stage_acc<D>(dva, sst, PITCH, 0, lane);
            __syncwarp();
            store_tile<D>(dv, base + int64_t(n0) * sstr, sstr, rows, sst, lane);
            __syncwarp();
        }
        __syncthreads();   // phase 1 reads every q row; phase 2 overwrites them with dQ
        // ---- phase 2: dQ per 16-query block
        for (int mt = warp; mt < n16; mt += nwarps) {
            const int m0 = mt * 16;
            const float lse0 = slse[m0 + g], lse1 = slse[m0 + g + 8], del0 = sdel[m0 + g], del1 = sdel[m0 + g + 8];
            float dqa[D / 8][4];
#pragma unroll
            for (int nt = 0; nt < D / 8; ++nt) dqa[nt][0] = dqa[nt][1] = dqa[nt][2] = dqa[nt][3] = 0.f;
            for (int kt = 0; kt < n64; ++kt) {
                float s[8][4], dp[8][4];
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) s[nt][e] = dp[nt][e] = 0.f;
                const uint32_t akt = ak + kt * 64 * PITCH;
                warp_mma<64, D, false, false>(s, aq, PITCH, m0, akt, PITCH, lane);                       // S  = Q K^T
                warp_mma<64, D, false, false>(dp, ad, PITCH, m0, av + kt * 64 * PITCH, PITCH, lane);     // dP = dO V^T
#pragma unroll
                for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float p = exp2f(s[nt][e] * scale_log2 - (e < 2 ? lse0 : lse1));
                        s[nt][e] = p * (dp[nt][e] - (e < 2 ? del0 : del1)) * scale;
                    }
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {   // dQ += dS K
                    uint32_t da[4];
                    acc_to_a(s, kk, da);
#pragma unroll
                    for (int np = 0; np < D / 16; ++np) {
                        uint32_t b[4];
                        load_b2<true>(akt, PITCH, np * 16, kk * 16, lane, b);
                        mma_bf16(dqa[2 * np], da, b[0], b[1]);
                        mma_bf16(dqa[2 * np + 1], da, b[2], b[3]);
                    }
                }
            }
            __syncwarp();
            stage_acc<D>(dqa, sq, PITCH, m0, lane);
            __syncwarp();
            store_tile<D>(dq, base + int64_t(m0) * sstr, sstr, min(16, L - m0), sq + m0 * PITCH, lane);
        }
    }
}

}  // namespace t2v

using namespace t2v;

namespace {

int check_args(int L, int D, int64_t ld_in, int64_t ld_out) {
    if (L < 1 || L > kMaxL) return fail(-2, "attn_small: L=%d out of range (1..%d)", L, kMaxL);
    if (D != 64 && D != 32) return fail(-2, "attn_small: head_dim %d unsupported (32 or 64)", D);
    if (ld_in % 8 || ld_out % 8) return fail(-2, "attn_small: row pitches must be multiples of 8 elements");
    return 0;
}

// warps per block so that a block stays near 64 KB of shared memory (3 blocks per SM)
int warps_for(int per_warp_bytes) { return std::max(1, std::min(8, (64 * 1024) / per_warp_bytes)); }

template <typename Kernel>
void set_smem_once(Kernel kernel, bool& done) {
    if (done) return;
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    done = true;
}

template <int D, int LP>
int launch_fwd(const void* q, const void* k, const void* v, void* o, const SeqAddr& a, int64_t nseq, int heads, int L, cudaStream_t st) {
    static bool done = false;
    set_smem_once(attn_small_fwd_kernel<D, LP>, done);
    const int per_warp = AttnSmem<D, LP>::kFwdBytes;
    const int warps = warps_for(per_warp);
    const int64_t total = nseq * heads;
    const int grid = int(std::min<int64_t>((total + warps - 1) / warps, int64_t(device_sm_count()) * 8));
    return int(launch_pdl(attn_small_fwd_kernel<D, LP>, dim3(grid), dim3(warps * 32), size_t(per_warp) * warps, st,
                          static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(v),
                          static_cast<__nv_bfloat16*>(o), a, nseq, heads, L, 1.0f / sqrtf(float(D))));
}

template <int D, int LP>
int launch_bwd(const void* q, const void* k, const void* v, const void* dout, void* dq, void* dk, void* dv, const SeqAddr& a,
               int64_t nseq, int heads, int L, cudaStream_t st) {
    static bool done = false;
    set_smem_once(attn_small_bwd_kernel<D, LP>, done);
    const int per_warp = AttnSmem<D, LP>::kBwdBytes;
    const int warps = warps_for(per_warp);
    const int64_t total = nseq * heads;
    const int grid = int(std::min<int64_t>((total + warps - 1) / warps, int64_t(device_sm_count()) * 8));
    auto B = [](const void* p) { return static_cast<const __nv_bfloat16*>(p); };
    auto W = [](void* p) { return static_cast<__nv_bfloat16*>(p); };
    return int(launch_pdl(attn_small_bwd_kernel<D, LP>, dim3(grid), dim3(warps * 32), size_t(per_warp) * warps, st, B(q), B(k), B(v),
                          B(dout), W(dq), W(dk), W(dv), a, nseq, heads, L, 1.0f / sqrtf(float(D))));
}

int check_long_args(int L, int D, int64_t ld_in, int64_t ld_out) {
    if (L < 1 || L > kLongMaxL) return fail(-2, "attn_long: L=%d out of range (1..%d)", L, kLongMaxL);
    if (D != 64 && D != 32) return fail(-2, "attn_long: head_dim %d unsupported (32 or 64)", D);
    if (ld_in % 8 || ld_out % 8) return fail(-2, "attn_long: row pitches must be multiples of 8 elements");
    return 0;
}

// one CTA per (sequence, head), a warp per 16-row block up to kLongWarps; the grid loops when there are more pairs than fit
struct LongLaunch {
    int LP, warps, grid;
    LongLaunch(int L, int64_t total)
        : LP((L + 63) / 64 * 64), warps(std::min(kLongWarps, (L + 15) / 16)),
          grid(int(std::min<int64_t>(total, int64_t(device_sm_count()) * 32))) {}
};

template <int D>
int launch_long_fwd(const void* q, const void* k, const void* v, void* o, float* lse, const SeqAddr& a, int64_t nseq, int heads, int L,
                    cudaStream_t st) {
    static bool done = false;
    set_smem_once(attn_long_fwd_kernel<D>, done);
    const LongLaunch c(L, nseq * heads);
    const float scale = 1.0f / sqrtf(float(D));
    return int(launch_pdl(attn_long_fwd_kernel<D>, dim3(c.grid), dim3(c.warps * 32), size_t(LongSmem<D>::fwd(c.LP)), st,
                          static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k), static_cast<const __nv_bfloat16*>(v),
                          static_cast<__nv_bfloat16*>(o), lse, a, nseq, heads, L, c.LP, scale * kLog2e));
}

template <int D>
int launch_long_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse, void* dq, void* dk,
                    void* dv, const SeqAddr& a, int64_t nseq, int heads, int L, cudaStream_t st) {
    static bool done = false;
    set_smem_once(attn_long_bwd_kernel<D>, done);
    const LongLaunch c(L, nseq * heads);
    const float scale = 1.0f / sqrtf(float(D));
    auto B = [](const void* p) { return static_cast<const __nv_bfloat16*>(p); };
    auto W = [](void* p) { return static_cast<__nv_bfloat16*>(p); };
    return int(launch_pdl(attn_long_bwd_kernel<D>, dim3(c.grid), dim3(c.warps * 32), size_t(LongSmem<D>::bwd(c.LP, c.warps)), st, B(q),
                          B(k), B(v), B(o), B(dout), lse, W(dq), W(dk), W(dv), a, nseq, heads, L, c.LP, scale, scale * kLog2e));
}

}  // namespace

extern "C" {

int t2v_attn_small_fwd(const void* q, const void* k, const void* v, void* o, int64_t nseq, int32_t inner, int64_t outer_rows,
                       int64_t inner_rows, int64_t seq_rows, int64_t ld_in, int64_t ld_out, int32_t heads, int32_t L, int32_t D,
                       void* stream) {
    if (int r = check_args(L, D, ld_in, ld_out)) return r;
    const SeqAddr a{outer_rows, inner_rows, seq_rows, ld_in, ld_out, inner};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc;
    if (D == 64) rc = L <= 16 ? launch_fwd<64, 16>(q, k, v, o, a, nseq, heads, L, st) : launch_fwd<64, 32>(q, k, v, o, a, nseq, heads, L, st);
    else rc = L <= 16 ? launch_fwd<32, 16>(q, k, v, o, a, nseq, heads, L, st) : launch_fwd<32, 32>(q, k, v, o, a, nseq, heads, L, st);
    return launch_checked(rc, "attn_small_fwd");
}

int t2v_attn_small_bwd(const void* q, const void* k, const void* v, const void* dout, void* dq, void* dk, void* dv, int64_t nseq,
                       int32_t inner, int64_t outer_rows, int64_t inner_rows, int64_t seq_rows, int64_t ld_in, int64_t ld_out,
                       int32_t heads, int32_t L, int32_t D, void* stream) {
    if (int r = check_args(L, D, ld_in, ld_out)) return r;
    const SeqAddr a{outer_rows, inner_rows, seq_rows, ld_in, ld_out, inner};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc;
    if (D == 64)
        rc = L <= 16 ? launch_bwd<64, 16>(q, k, v, dout, dq, dk, dv, a, nseq, heads, L, st)
                     : launch_bwd<64, 32>(q, k, v, dout, dq, dk, dv, a, nseq, heads, L, st);
    else
        rc = L <= 16 ? launch_bwd<32, 16>(q, k, v, dout, dq, dk, dv, a, nseq, heads, L, st)
                     : launch_bwd<32, 32>(q, k, v, dout, dq, dk, dv, a, nseq, heads, L, st);
    return launch_checked(rc, "attn_small_bwd");
}

int t2v_attn_long_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int64_t nseq, int32_t inner, int64_t outer_rows,
                      int64_t inner_rows, int64_t seq_rows, int64_t ld_in, int64_t ld_out, int32_t heads, int32_t L, int32_t D,
                      void* stream) {
    if (int r = check_long_args(L, D, ld_in, ld_out)) return r;
    const SeqAddr a{outer_rows, inner_rows, seq_rows, ld_in, ld_out, inner};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = D == 64 ? launch_long_fwd<64>(q, k, v, o, lse, a, nseq, heads, L, st) : launch_long_fwd<32>(q, k, v, o, lse, a, nseq, heads, L, st);
    return launch_checked(rc, "attn_long_fwd");
}

int t2v_attn_long_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse, void* dq, void* dk,
                      void* dv, int64_t nseq, int32_t inner, int64_t outer_rows, int64_t inner_rows, int64_t seq_rows, int64_t ld_in,
                      int64_t ld_out, int32_t heads, int32_t L, int32_t D, void* stream) {
    if (int r = check_long_args(L, D, ld_in, ld_out)) return r;
    const SeqAddr a{outer_rows, inner_rows, seq_rows, ld_in, ld_out, inner};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = D == 64 ? launch_long_bwd<64>(q, k, v, o, dout, lse, dq, dk, dv, a, nseq, heads, L, st)
                           : launch_long_bwd<32>(q, k, v, o, dout, lse, dq, dk, dv, a, nseq, heads, L, st);
    return launch_checked(rc, "attn_long_bwd");
}

}  // extern "C"
