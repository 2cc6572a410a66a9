// Fused AdamW + global-norm clipping over the flat parameter arena (SURVEY 8(f) row 1; the reference builds
// torch.optim.AdamW at train.py:616-623 and clips with accelerator.clip_grad_norm_ at :868-876).
//
// Three kernels per optimizer step, all free of host-side scalars so that the step can sit inside the CUDA graph of the
// training step (learning rate, step count and clip factor live in device memory):
//   sqnorm   one read of the trainable gradient ranges -> sum of squares (fp64 accumulation)             4 B / param
//   prepare  one thread: step += 1, bias corrections, clip factor min(1, max_norm / (norm + 1e-6))       -
//   update   reads p, g, m, v, writes p, m, v, the bf16 compute shadow of p (kernel layout == master layout, so the
//            per-step cast kernel disappears) and zero into g (so the per-step gradient memset disappears)  34 B / param
// HBM-bound; algorithmic bytes = 38 per trainable parameter with clipping, 34 without.
// The blockwise 8-bit update (adamw8bit_chunks) replaces the 16 B of fp32 m, v traffic by 2 B of codes and 16 B per
// 256-element block of absmax: 26 B + 1/16 B per parameter with clipping.
//
// The trainable set is described by a CHUNK TABLE (int64 pairs: offset, length; offsets and lengths are multiples of 64
// elements, a chunk never straddles the matrix/vector boundary of the arena): one launch covers every parameter of a
// hyper-parameter set, however fragmented (LoRA: 1,148 small matrices between frozen base weights).
//
// Semantics = torch.optim.AdamW (decoupled weight decay, no amsgrad):
//   p *= 1 - lr * wd;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
// with g pre-multiplied by the clip factor.
#include "common.h"
#include "gemm_tc.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cmath>
#include <cuda_bf16.h>

namespace t2v {

// hp layout (floats): [0] lr [1] beta1 [2] beta2 [3] eps [4] weight_decay [5] bias_c1 [6] sqrt(bias_c2) [7] grad_scale
constexpr int kHp = 8;

struct AdamWArgs {
    float lr, beta1, beta2, eps, weight_decay, bias_c1, bias_c2_sqrt, grad_scale;
};

__device__ __forceinline__ void adamw_one(float& p, float g, float& m, float& v, const AdamWArgs& a) {
    g *= a.grad_scale;
    p *= 1.0f - a.lr * a.weight_decay;
    m = a.beta1 * m + (1.0f - a.beta1) * g;
    v = a.beta2 * v + (1.0f - a.beta2) * g * g;
    const float denom = sqrtf(v) / a.bias_c2_sqrt + a.eps;
    p -= (a.lr / a.bias_c1) * (m / denom);
}

__device__ __forceinline__ AdamWArgs load_hp(const float* hp) {
    AdamWArgs a;
    a.lr = hp[0]; a.beta1 = hp[1]; a.beta2 = hp[2]; a.eps = hp[3]; a.weight_decay = hp[4];
    a.bias_c1 = hp[5]; a.bias_c2_sqrt = hp[6]; a.grad_scale = hp[7];
    return a;
}

// Exponential moving average of the updated weights (diffusers' EMAModel with its default arguments).  k = the step count
// after this step's increment (adamw_prepare): d_1 = 0, d_k = min(decay, k / (9 + k)) for k >= 2, computed in fp64; the
// kernels use 1 - d_k rounded to fp32.  The lerp is EMAModel.step's `s -= (1 - d) * (s - p)`, each operation rounded on its
// own (no FMA contraction), so it restates torch's fp32 arithmetic exactly.
__device__ __forceinline__ float ema_one_minus_decay(const int64_t* __restrict__ step, float decay) {
    const double k = double(*step);
    const double d = k <= 1.0 ? 0.0 : fmin(double(decay), k / (9.0 + k));
    return float(1.0 - d);
}

__device__ __forceinline__ void ema_lerp(float4& e, const float4& p, float omd) {
    e.x = __fsub_rn(e.x, __fmul_rn(omd, __fsub_rn(e.x, p.x)));
    e.y = __fsub_rn(e.y, __fmul_rn(omd, __fsub_rn(e.y, p.y)));
    e.z = __fsub_rn(e.z, __fmul_rn(omd, __fsub_rn(e.z, p.z)));
    e.w = __fsub_rn(e.w, __fmul_rn(omd, __fsub_rn(e.w, p.w)));
}

// One chunk with fp32 state, the block's threads striding over it: elements [off, off + len) of p, g, shadow (written when sh)
// and g16 (may be NULL), state elements [soff, soff + len) of m and v.  kEma: then also the EMA elements [eoff, eoff + len),
// lerped towards the new p with omd = 1 - d_k.
template <bool kEma>
__device__ __forceinline__ void adamw_chunk_f32(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                __nv_bfloat16* __restrict__ shadow, bool sh, const __nv_bfloat16* __restrict__ g16,
                                                int64_t off, int64_t soff, int64_t len, const AdamWArgs& a, int zero_grad,
                                                float* __restrict__ ema, int64_t eoff, float omd) {
    float4* p4 = reinterpret_cast<float4*>(p + off);
    float4* g4 = reinterpret_cast<float4*>(g + off);
    float4* m4 = reinterpret_cast<float4*>(m + soff);
    float4* v4 = reinterpret_cast<float4*>(v + soff);
    uint2* s2 = reinterpret_cast<uint2*>(shadow + off);
    const uint2* h2 = reinterpret_cast<const uint2*>(g16 + off);
    const int nv = int(len >> 2);
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        float4 pp = p4[i];
        float4 gg;
        if (g16) {
            const uint2 h = __ldg(h2 + i);
            gg = make_float4(bf16_lo(h.x), bf16_hi(h.x), bf16_lo(h.y), bf16_hi(h.y));
        } else {
            gg = g4[i];
        }
        float4 mm = m4[i];
        float4 vv = v4[i];
        adamw_one(pp.x, gg.x, mm.x, vv.x, a);
        adamw_one(pp.y, gg.y, mm.y, vv.y, a);
        adamw_one(pp.z, gg.z, mm.z, vv.z, a);
        adamw_one(pp.w, gg.w, mm.w, vv.w, a);
        p4[i] = pp;
        m4[i] = mm;
        v4[i] = vv;
        if constexpr (kEma) {
            float4* e4 = reinterpret_cast<float4*>(ema + eoff);
            float4 ee = e4[i];
            ema_lerp(ee, pp, omd);
            e4[i] = ee;
        }
        if (sh) {
            uint2 q;
            q.x = pack_bf16(pp.x, pp.y);
            q.y = pack_bf16(pp.z, pp.w);
            s2[i] = q;
        }
        if (zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// g16 != NULL: the gradient comes from the bf16 communication buffer (the all-reduced, averaged gradient of a data-parallel
// step); the fp32 accumulation buffer g is then only zeroed.  Chunk rows: (offset, length), or with kEma (offset, length,
// EMA offset).
template <bool kEma>
__device__ __forceinline__ void adamw_chunks_body(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                  __nv_bfloat16* __restrict__ shadow, int64_t n_shadow, const int64_t* __restrict__ chunks,
                                                  int n_chunks, const float* __restrict__ hp, int zero_grad,
                                                  const __nv_bfloat16* __restrict__ g16, float* __restrict__ ema,
                                                  const int64_t* __restrict__ step, float ema_decay) {
    constexpr int kCols = kEma ? 3 : 2;
    pdl_sync();
    const AdamWArgs a = load_hp(hp);
    float omd = 0.f;
    if constexpr (kEma) omd = ema_one_minus_decay(step, ema_decay);
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int64_t off = chunks[kCols * c], len = chunks[kCols * c + 1];
        const bool sh = shadow != nullptr && off < n_shadow;
        adamw_chunk_f32<kEma>(p, g, m, v, shadow, sh, g16, off, off, len, a, zero_grad, ema, kEma ? chunks[kCols * c + kCols - 1] : 0, omd);
    }
}

__global__ void __launch_bounds__(256) adamw_chunks_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                                           float* __restrict__ v, __nv_bfloat16* __restrict__ shadow, int64_t n_shadow,
                                                           const int64_t* __restrict__ chunks, int n_chunks, const float* __restrict__ hp,
                                                           int zero_grad, const __nv_bfloat16* __restrict__ g16) {
    adamw_chunks_body<false>(p, g, m, v, shadow, n_shadow, chunks, n_chunks, hp, zero_grad, g16, nullptr, nullptr, 0.f);
}

__global__ void __launch_bounds__(256) adamw_ema_chunks_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                                               float* __restrict__ v, __nv_bfloat16* __restrict__ shadow, int64_t n_shadow,
                                                               const int64_t* __restrict__ chunks, int n_chunks, const float* __restrict__ hp,
                                                               int zero_grad, const __nv_bfloat16* __restrict__ g16, float* __restrict__ ema,
                                                               const int64_t* __restrict__ step, float ema_decay) {
    adamw_chunks_body<true>(p, g, m, v, shadow, n_shadow, chunks, n_chunks, hp, zero_grad, g16, ema, step, ema_decay);
}

// Blockwise 8-bit AdamW (optim.AdamW8bit; Dettmers et al., ICLR 2022).  Chunk rows are int64 quadruples (arena offset, length,
// state offset, bits).  bits == 32: fp32 m32 / v32 at the state offset, exactly adamw_chunks' update.  bits == 8: the row's
// 256-element blocks (the last one may hold 64, 128 or 192) each keep one uint8 code per element and one fp32 absmax per
// moment; m uses the signed map qmaps[0..255], v the unsigned map qmaps[256..511].  Per block (one warp, 8 elements per lane):
// dequantise (map[code] * absmax), adamw_one on the unquantised moments, new absmax = block max |m| (|v|), new code = nearest
// map entry: the smallest i with x <= 0.5f * (map[i] + map[i+1]).  A block whose absmax is 0 stores the code of 0.0.
// The 255 midpoints are searched as an implicit (Eytzinger) binary tree in shared memory: level d of the tree is 2^d
// consecutive floats, so the lanes of a warp hit distinct banks on the first six of the eight levels.
constexpr int kQBlock = 256;

__device__ __forceinline__ uint32_t quantize(float x, float absmax, const float* tree, uint32_t zero_code) {
    if (absmax == 0.f) return zero_code;
    x = x / absmax;
    uint32_t k = 1;
#pragma unroll
    for (int l = 0; l < 8; ++l) k = 2 * k + (x > tree[k] ? 1u : 0u);
    return k - 256;
}

// kEma: rows carry a fifth column, the EMA offset; both the 32-bit and the 8-bit rows lerp the fp32 EMA towards the new p.
template <bool kEma>
__device__ __forceinline__ void adamw8bit_chunks_body(float* __restrict__ p, float* __restrict__ g, __nv_bfloat16* __restrict__ shadow,
                                                      int64_t n_shadow, const int64_t* __restrict__ chunks, int n_chunks,
                                                      const float* __restrict__ hp, const float* __restrict__ qmaps, float* __restrict__ m32,
                                                      float* __restrict__ v32, uint8_t* __restrict__ qm, uint8_t* __restrict__ qv,
                                                      float* __restrict__ absmax_m, float* __restrict__ absmax_v, int zero_grad,
                                                      const __nv_bfloat16* __restrict__ g16, float* __restrict__ ema,
                                                      const int64_t* __restrict__ step, float ema_decay) {
    constexpr int kCols = kEma ? 5 : 4;
    __shared__ float map_m[256], map_v[256], tree_m[256], tree_v[256];
    __shared__ uint32_t zero_m;
    pdl_sync();
    const int t = threadIdx.x;
    map_m[t] = qmaps[t];
    map_v[t] = qmaps[256 + t];
    __syncthreads();
    if (t > 0) {   // tree node t at depth d holds the midpoint of in-order rank ((2 (t - 2^d) + 1) << (7 - d)) - 1
        const int d = 31 - __clz(t);
        const int i = ((2 * (t - (1 << d)) + 1) << (7 - d)) - 1;
        tree_m[t] = 0.5f * (map_m[i] + map_m[i + 1]);
        tree_v[t] = 0.5f * (map_v[i] + map_v[i + 1]);
    }
    if (map_m[t] == 0.f) zero_m = uint32_t(t);
    __syncthreads();
    const uint32_t zm = zero_m, zv = 0;   // the unsigned map starts at 0.0
    const AdamWArgs a = load_hp(hp);
    float omd = 0.f;
    if constexpr (kEma) omd = ema_one_minus_decay(step, ema_decay);
    const int lane = t & 31, warp = t >> 5;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int64_t off = chunks[kCols * c], len = chunks[kCols * c + 1], soff = chunks[kCols * c + 2];
        const int64_t eoff = kEma ? chunks[kCols * c + kCols - 1] : 0;
        const bool sh = shadow != nullptr && off < n_shadow;
        if (chunks[kCols * c + 3] != 8) {   // uniform across the thread block
            adamw_chunk_f32<kEma>(p, g, m32, v32, shadow, sh, g16, off, soff, len, a, zero_grad, ema, eoff, omd);
            continue;
        }
        const int nblk = int((len + kQBlock - 1) / kQBlock);
        for (int b = warp; b < nblk; b += blockDim.x >> 5) {
            const int64_t e0 = int64_t(b) * kQBlock;          // element of the row where this block starts
            const int nb = int(min(int64_t(kQBlock), len - e0));  // 64, 128, 192 or 256
            const int64_t qb = soff / kQBlock + b;             // block index into absmax
            const float am_old = absmax_m[qb], av_old = absmax_v[qb];
            float pe[8], me[8], ve[8];
            bool ok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {   // lane owns elements h*128 + 4*lane .. +3 of the block: two 16-byte loads
                const int j = h * 128 + 4 * lane;
                ok[h] = j < nb;
                if (!ok[h]) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) pe[4 * h + u] = me[4 * h + u] = ve[4 * h + u] = 0.f;
                    continue;
                }
                const int64_t e = off + e0 + j;
                const float4 pp = *reinterpret_cast<const float4*>(p + e);
                float4 gg;
                if (g16) {
                    const uint2 hh = __ldg(reinterpret_cast<const uint2*>(g16 + e));
                    gg = make_float4(bf16_lo(hh.x), bf16_hi(hh.x), bf16_lo(hh.y), bf16_hi(hh.y));
                } else {
                    gg = *reinterpret_cast<const float4*>(g + e);
                }
                const uint32_t cm = *reinterpret_cast<const uint32_t*>(qm + soff + e0 + j);
                const uint32_t cv = *reinterpret_cast<const uint32_t*>(qv + soff + e0 + j);
                const float gl[4] = {gg.x, gg.y, gg.z, gg.w};
                pe[4 * h] = pp.x; pe[4 * h + 1] = pp.y; pe[4 * h + 2] = pp.z; pe[4 * h + 3] = pp.w;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    float& m = me[4 * h + u];
                    float& v = ve[4 * h + u];
                    m = map_m[(cm >> (8 * u)) & 0xFF] * am_old;
                    v = map_v[(cv >> (8 * u)) & 0xFF] * av_old;
                    adamw_one(pe[4 * h + u], gl[u], m, v, a);
                }
            }
            uint32_t mx_m = 0, mx_v = 0;   // |x| of finite floats orders like its bit pattern
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                mx_m = max(mx_m, __float_as_uint(fabsf(me[u])));
                mx_v = max(mx_v, __float_as_uint(fabsf(ve[u])));
            }
            const float am = __uint_as_float(__reduce_max_sync(0xffffffffu, mx_m));
            const float av = __uint_as_float(__reduce_max_sync(0xffffffffu, mx_v));
            if (lane == 0) {
                absmax_m[qb] = am;
                absmax_v[qb] = av;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!ok[h]) continue;
                const int j = h * 128 + 4 * lane;
                const int64_t e = off + e0 + j;
                uint32_t cm = 0, cv = 0;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    cm |= quantize(me[4 * h + u], am, tree_m, zm) << (8 * u);
                    cv |= quantize(ve[4 * h + u], av, tree_v, zv) << (8 * u);
                }
                *reinterpret_cast<uint32_t*>(qm + soff + e0 + j) = cm;
                *reinterpret_cast<uint32_t*>(qv + soff + e0 + j) = cv;
                const float4 pn = make_float4(pe[4 * h], pe[4 * h + 1], pe[4 * h + 2], pe[4 * h + 3]);
                *reinterpret_cast<float4*>(p + e) = pn;
                if constexpr (kEma) {
                    float4* e4 = reinterpret_cast<float4*>(ema + eoff + e0 + j);
                    float4 ee = *e4;
                    ema_lerp(ee, pn, omd);
                    *e4 = ee;
                }
                if (sh)
                    *reinterpret_cast<uint2*>(shadow + e) =
                        make_uint2(pack_bf16(pe[4 * h], pe[4 * h + 1]), pack_bf16(pe[4 * h + 2], pe[4 * h + 3]));
                if (zero_grad) *reinterpret_cast<float4*>(g + e) = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
    }
}

__global__ void __launch_bounds__(256) adamw8bit_chunks_kernel(float* __restrict__ p, float* __restrict__ g, __nv_bfloat16* __restrict__ shadow,
                                                               int64_t n_shadow, const int64_t* __restrict__ chunks, int n_chunks,
                                                               const float* __restrict__ hp, const float* __restrict__ qmaps, float* __restrict__ m32,
                                                               float* __restrict__ v32, uint8_t* __restrict__ qm, uint8_t* __restrict__ qv,
                                                               float* __restrict__ absmax_m, float* __restrict__ absmax_v, int zero_grad,
                                                               const __nv_bfloat16* __restrict__ g16) {
    adamw8bit_chunks_body<false>(p, g, shadow, n_shadow, chunks, n_chunks, hp, qmaps, m32, v32, qm, qv, absmax_m, absmax_v, zero_grad, g16,
                                 nullptr, nullptr, 0.f);
}

__global__ void __launch_bounds__(256) adamw8bit_ema_chunks_kernel(float* __restrict__ p, float* __restrict__ g, __nv_bfloat16* __restrict__ shadow,
                                                                   int64_t n_shadow, const int64_t* __restrict__ chunks, int n_chunks,
                                                                   const float* __restrict__ hp, const float* __restrict__ qmaps,
                                                                   float* __restrict__ m32, float* __restrict__ v32, uint8_t* __restrict__ qm,
                                                                   uint8_t* __restrict__ qv, float* __restrict__ absmax_m,
                                                                   float* __restrict__ absmax_v, int zero_grad,
                                                                   const __nv_bfloat16* __restrict__ g16, float* __restrict__ ema,
                                                                   const int64_t* __restrict__ step, float ema_decay) {
    adamw8bit_chunks_body<true>(p, g, shadow, n_shadow, chunks, n_chunks, hp, qmaps, m32, v32, qm, qv, absmax_m, absmax_v, zero_grad, g16,
                                ema, step, ema_decay);
}

// Exchanges p and the EMA over (arena offset, length, EMA offset) rows and rewrites the bf16 shadow of the rows below n_shadow
// from the new p, rounded as the update kernels round it: a second call restores p, the EMA and the shadow bit for bit.
__global__ void __launch_bounds__(256) ema_swap_chunks_kernel(float* __restrict__ p, float* __restrict__ ema, __nv_bfloat16* __restrict__ shadow,
                                                              int64_t n_shadow, const int64_t* __restrict__ rows, int n_rows) {
    pdl_sync();
    for (int c = blockIdx.x; c < n_rows; c += gridDim.x) {
        const int64_t off = rows[3 * c], len = rows[3 * c + 1], eoff = rows[3 * c + 2];
        const bool sh = shadow != nullptr && off < n_shadow;
        float4* p4 = reinterpret_cast<float4*>(p + off);
        float4* e4 = reinterpret_cast<float4*>(ema + eoff);
        uint2* s2 = reinterpret_cast<uint2*>(shadow + off);
        const int nv = int(len >> 2);
        for (int i = threadIdx.x; i < nv; i += blockDim.x) {
            const float4 pp = p4[i], ee = e4[i];
            p4[i] = ee;
            e4[i] = pp;
            if (sh) s2[i] = make_uint2(pack_bf16(ee.x, ee.y), pack_bf16(ee.z, ee.w));
        }
    }
}

__global__ void __launch_bounds__(256) sqnorm_chunks_kernel(const float* __restrict__ g, const int64_t* __restrict__ chunks, int n_chunks,
                                                            double* __restrict__ out, const __nv_bfloat16* __restrict__ g16) {
    pdl_sync();
    double acc = 0.0;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int64_t off = chunks[2 * c], len = chunks[2 * c + 1];
        const float4* g4 = reinterpret_cast<const float4*>(g + off);
        const uint2* h2 = reinterpret_cast<const uint2*>(g16 + off);
        const int nv = int(len >> 2);
        float part = 0.f;  // one chunk is at most 64 K elements: 64 fp32 terms per thread, then fp64
        for (int i = threadIdx.x; i < nv; i += blockDim.x) {
            float4 q;
            if (g16) {
                const uint2 h = __ldg(h2 + i);
                q = make_float4(bf16_lo(h.x), bf16_hi(h.x), bf16_lo(h.y), bf16_hi(h.y));
            } else {
                q = __ldg(g4 + i);
            }
            part += q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
        }
        acc += double(part);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double wsum[8];
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += wsum[w];
        atomicAdd(out, t);
    }
}

// hp_in: n_sets x 5 floats (lr, beta1, beta2, eps, weight_decay) written by the host before the step; hp: n_sets x kHp.
// state: [0] optimizer step count (int64)  ;  sq: [0] sum of squared gradients of this step (consumed and reset here),
// [1] the gradient norm of the last step (kept for logging)
__global__ void adamw_prepare_kernel(const float* __restrict__ hp_in, float* __restrict__ hp, int n_sets, int64_t* __restrict__ state,
                                     double* __restrict__ sq, float max_norm) {
    pdl_sync();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int64_t step = state[0] + 1;
    state[0] = step;
    const double norm = sqrt(sq[0]);
    sq[1] = norm;
    sq[0] = 0.0;
    float scale = 1.0f;
    if (max_norm > 0.f) scale = fminf(1.0f, max_norm / (float(norm) + 1e-6f));
    for (int s = 0; s < n_sets; ++s) {
        const float* in = hp_in + 5 * s;
        float* o = hp + kHp * s;
        o[0] = in[0]; o[1] = in[1]; o[2] = in[2]; o[3] = in[3]; o[4] = in[4];
        o[5] = float(1.0 - pow(double(in[1]), double(step)));
        o[6] = float(sqrt(1.0 - pow(double(in[2]), double(step))));
        o[7] = scale;
    }
}

__global__ void counter_add_kernel(int64_t* p, int64_t v) {
    pdl_sync();
    if (threadIdx.x == 0 && blockIdx.x == 0) *p += v;
}

}  // namespace t2v

using namespace t2v;

extern "C" {

static int chunk_grid(int n_chunks) { return std::max(1, std::min(n_chunks, device_sm_count() * 8)); }

int t2v_sqnorm_chunks(const float* g, const void* g_bf16, const int64_t* chunks, int32_t n_chunks, double* out, void* stream) {
    if (n_chunks <= 0) return 0;
    const int rc = int(launch_pdl(sqnorm_chunks_kernel, dim3(chunk_grid(n_chunks)), dim3(256), size_t(0), static_cast<cudaStream_t>(stream), g,
                                  chunks, int(n_chunks), out, static_cast<const __nv_bfloat16*>(g_bf16)));
    return launch_checked(rc, "sqnorm_chunks");
}

int t2v_adamw_prepare(const float* hp_in, float* hp, int32_t n_sets, int64_t* state, double* sq, float max_norm, void* stream) {
    if (n_sets <= 0) return fail(-2, "adamw_prepare: no hyper-parameter sets");
    const int rc = int(launch_pdl(adamw_prepare_kernel, dim3(1), dim3(32), size_t(0), static_cast<cudaStream_t>(stream), hp_in, hp, int(n_sets),
                                  state, sq, max_norm));
    return launch_checked(rc, "adamw_prepare");
}

int t2v_adamw_chunks(float* p, float* g, const void* g_bf16, float* m, float* v, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks,
                     int32_t n_chunks, const float* hp, int32_t zero_grad, void* stream) {
    if (n_chunks <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15u)
        return fail(-2, "adamw_chunks: p, g, m, v must be 16-byte aligned");
    if (shadow_bf16 && (reinterpret_cast<uintptr_t>(shadow_bf16) & 7u)) return fail(-2, "adamw_chunks: shadow must be 8-byte aligned");
    const int rc = int(launch_pdl(adamw_chunks_kernel, dim3(chunk_grid(n_chunks)), dim3(256), size_t(0), static_cast<cudaStream_t>(stream), p, g, m,
                                  v, static_cast<__nv_bfloat16*>(shadow_bf16), n_shadow, chunks, int(n_chunks), hp, int(zero_grad),
                                  static_cast<const __nv_bfloat16*>(g_bf16)));
    return launch_checked(rc, "adamw_chunks");
}

int t2v_adamw8bit_chunks(float* p, float* g, const void* g_bf16, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks, int32_t n_chunks,
                         const float* hp, const float* qmaps, float* m32, float* v32, void* code_m, void* code_v, float* absmax_m,
                         float* absmax_v, int32_t zero_grad, void* stream) {
    if (n_chunks <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m32) | reinterpret_cast<uintptr_t>(v32)) &
        15u)
        return fail(-2, "adamw8bit_chunks: p, g, m32, v32 must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(code_m) | reinterpret_cast<uintptr_t>(code_v)) & 3u)
        return fail(-2, "adamw8bit_chunks: code_m, code_v must be 4-byte aligned");
    if (shadow_bf16 && (reinterpret_cast<uintptr_t>(shadow_bf16) & 7u)) return fail(-2, "adamw8bit_chunks: shadow must be 8-byte aligned");
    const int rc = int(launch_pdl(adamw8bit_chunks_kernel, dim3(chunk_grid(n_chunks)), dim3(256), size_t(0), static_cast<cudaStream_t>(stream), p,
                                  g, static_cast<__nv_bfloat16*>(shadow_bf16), n_shadow, chunks, int(n_chunks), hp, qmaps, m32, v32,
                                  static_cast<uint8_t*>(code_m), static_cast<uint8_t*>(code_v), absmax_m, absmax_v, int(zero_grad),
                                  static_cast<const __nv_bfloat16*>(g_bf16)));
    return launch_checked(rc, "adamw8bit_chunks");
}

static int check_ema(const float* ema, const int64_t* step, float ema_decay, const char* who) {
    if (!ema || !step) return fail(-2, "%s: ema and step must not be NULL", who);
    if (reinterpret_cast<uintptr_t>(ema) & 15u) return fail(-2, "%s: ema must be 16-byte aligned", who);
    if (!(ema_decay >= 0.f && ema_decay <= 1.f)) return fail(-2, "%s: ema_decay must lie in [0, 1]", who);
    return 0;
}

int t2v_adamw_ema_chunks(float* p, float* g, const void* g_bf16, float* m, float* v, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks,
                         int32_t n_chunks, const float* hp, int32_t zero_grad, float* ema, const int64_t* step, float ema_decay, void* stream) {
    if (n_chunks <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15u)
        return fail(-2, "adamw_ema_chunks: p, g, m, v must be 16-byte aligned");
    if (shadow_bf16 && (reinterpret_cast<uintptr_t>(shadow_bf16) & 7u)) return fail(-2, "adamw_ema_chunks: shadow must be 8-byte aligned");
    if (const int rc = check_ema(ema, step, ema_decay, "adamw_ema_chunks")) return rc;
    const int rc = int(launch_pdl(adamw_ema_chunks_kernel, dim3(chunk_grid(n_chunks)), dim3(256), size_t(0), static_cast<cudaStream_t>(stream), p, g,
                                  m, v, static_cast<__nv_bfloat16*>(shadow_bf16), n_shadow, chunks, int(n_chunks), hp, int(zero_grad),
                                  static_cast<const __nv_bfloat16*>(g_bf16), ema, step, ema_decay));
    return launch_checked(rc, "adamw_ema_chunks");
}

int t2v_adamw8bit_ema_chunks(float* p, float* g, const void* g_bf16, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks, int32_t n_chunks,
                             const float* hp, const float* qmaps, float* m32, float* v32, void* code_m, void* code_v, float* absmax_m,
                             float* absmax_v, int32_t zero_grad, float* ema, const int64_t* step, float ema_decay, void* stream) {
    if (n_chunks <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m32) | reinterpret_cast<uintptr_t>(v32)) &
        15u)
        return fail(-2, "adamw8bit_ema_chunks: p, g, m32, v32 must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(code_m) | reinterpret_cast<uintptr_t>(code_v)) & 3u)
        return fail(-2, "adamw8bit_ema_chunks: code_m, code_v must be 4-byte aligned");
    if (shadow_bf16 && (reinterpret_cast<uintptr_t>(shadow_bf16) & 7u)) return fail(-2, "adamw8bit_ema_chunks: shadow must be 8-byte aligned");
    if (const int rc = check_ema(ema, step, ema_decay, "adamw8bit_ema_chunks")) return rc;
    const int rc = int(launch_pdl(adamw8bit_ema_chunks_kernel, dim3(chunk_grid(n_chunks)), dim3(256), size_t(0), static_cast<cudaStream_t>(stream),
                                  p, g, static_cast<__nv_bfloat16*>(shadow_bf16), n_shadow, chunks, int(n_chunks), hp, qmaps, m32, v32,
                                  static_cast<uint8_t*>(code_m), static_cast<uint8_t*>(code_v), absmax_m, absmax_v, int(zero_grad),
                                  static_cast<const __nv_bfloat16*>(g_bf16), ema, step, ema_decay));
    return launch_checked(rc, "adamw8bit_ema_chunks");
}

int t2v_ema_swap_chunks(float* p, float* ema, void* shadow_bf16, int64_t n_shadow, const int64_t* rows, int32_t n_rows, void* stream) {
    if (n_rows <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(ema)) & 15u) return fail(-2, "ema_swap_chunks: p, ema must be 16-byte aligned");
    if (shadow_bf16 && (reinterpret_cast<uintptr_t>(shadow_bf16) & 7u)) return fail(-2, "ema_swap_chunks: shadow must be 8-byte aligned");
    const int rc = int(launch_pdl(ema_swap_chunks_kernel, dim3(chunk_grid(n_rows)), dim3(256), size_t(0), static_cast<cudaStream_t>(stream), p, ema,
                                  static_cast<__nv_bfloat16*>(shadow_bf16), n_shadow, rows, int(n_rows)));
    return launch_checked(rc, "ema_swap_chunks");
}

int t2v_counter_add(int64_t* counter, int64_t value, void* stream) {
    const int rc = int(launch_pdl(counter_add_kernel, dim3(1), dim3(32), size_t(0), static_cast<cudaStream_t>(stream), counter, value));
    return launch_checked(rc, "counter_add");
}

}  // extern "C"
