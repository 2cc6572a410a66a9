// HBM-bound glue kernels of the finetune step: layout conversion at the latent boundary (fused with add_noise / MSE),
// GEGLU, SiLU, nearest up-sampling, channel concat/split, bias gradients, softmax, casts.
// All use 128-bit accesses on channels-last bf16 data and grid-stride loops sized in multiples of the SM count.
#include "common.h"
#include "ptx.cuh"

#include <algorithm>
#include <cmath>
#include <cuda_bf16.h>

namespace t2v {

__device__ __forceinline__ void unpack8e(const uint4& q, float* v) {
    v[0] = bf16_lo(q.x); v[1] = bf16_hi(q.x); v[2] = bf16_lo(q.y); v[3] = bf16_hi(q.y);
    v[4] = bf16_lo(q.z); v[5] = bf16_hi(q.z); v[6] = bf16_lo(q.w); v[7] = bf16_hi(q.w);
}
__device__ __forceinline__ uint4 pack8e(const float* v) {
    uint4 q;
    q.x = pack_bf16(v[0], v[1]); q.y = pack_bf16(v[2], v[3]); q.z = pack_bf16(v[4], v[5]); q.w = pack_bf16(v[6], v[7]);
    return q;
}
__device__ __forceinline__ float sigm(float z) { return 1.0f / (1.0f + __expf(-z)); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_erf_grad(float x) {
    return 0.5f * (1.0f + erff(x * 0.70710678118654752f)) + x * 0.39894228040143268f * __expf(-0.5f * x * x);
}

static inline int ew_grid(int64_t n, int threads = 256) {
    return int(std::min<int64_t>((n + threads - 1) / threads, int64_t(device_sm_count()) * 16));
}
#define GRID_STRIDE(i, n) for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < (n); i += int64_t(gridDim.x) * blockDim.x)

// ------------------------------------------------------------------------------------------------ latent boundary
// (B, C<=8, F, H, W) fp32  ->  [B*F][H][W][8] bf16 (zero-padded channels), optionally fused with DDPM add_noise:
//   x_t = sqrt(abar[t_b]) x0 + sqrt(1 - abar[t_b]) eps        (train.py:760)
__global__ void to_nhwc8_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const float* __restrict__ abar,
                                const int64_t* __restrict__ t, __nv_bfloat16* __restrict__ out, int B, int C, int F, int HW) {
    pdl_sync();
    const int64_t npix = int64_t(B) * F * HW;
    GRID_STRIDE(i, npix) {
        const int hw = int(i % HW);
        const int f = int((i / HW) % F);
        const int b = int(i / (int64_t(HW) * F));
        float sa = 1.f, sb = 0.f;
        if (noise) {
            const float a = abar[t[b]];
            sa = sqrtf(a);
            sb = sqrtf(1.f - a);
        }
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float x = 0.f;
            if (c < C) {
                const int64_t src = ((int64_t(b) * C + c) * F + f) * HW + hw;
                x = sa * x0[src];
                if (noise) x += sb * noise[src];
            }
            v[c] = x;
        }
        reinterpret_cast<uint4*>(out)[i] = pack8e(v);
    }
}

// [B*F][H][W][8] bf16 -> (B, C, F, H, W) fp32
__global__ void from_nhwc8_kernel(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, int B, int C, int F, int HW) {
    pdl_sync();
    const int64_t npix = int64_t(B) * F * HW;
    GRID_STRIDE(i, npix) {
        const int hw = int(i % HW);
        const int f = int((i / HW) % F);
        const int b = int(i / (int64_t(HW) * F));
        float v[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(in) + i), v);
        for (int c = 0; c < C; ++c) out[((int64_t(b) * C + c) * F + f) * HW + hw] = v[c];
    }
}

// MSE forward: loss += sum (pred - target)^2 / numel ; backward: dpred = g * 2 (pred - target) / numel
// target is (B, C, F, H, W) fp32.  With x0 given it is the noise of a v-prediction step and the regression target is the
// velocity, formed per element and never stored:  v = sqrt(abar[t_b]) eps - sqrt(1 - abar[t_b]) x0  (DDPMScheduler.get_velocity,
// train.py:796-797).  abar and t are read on the device, so a replayed CUDA graph uses each step's timesteps.
// Six blocks per SM holds the kernel at the 40 registers the noise-target-only version used (no spills); left free, ptxas
// keeps all sixteen loads of the velocity path in flight and takes 42, which drops a block per SM for both objectives.
//
// The same body computes the weighted and robust objectives of t2v_diffusion_loss: FORM picks the per-element loss psi and
// WEIGHTED the Min-SNR-gamma sample weight w_b; loss += sum w_b psi(e) / numel, dpred = g w_b psi'(e) / numel.  w_b and the
// Huber scale c_b come from abar[t[b]] on the device, like the velocity, so a replayed graph uses each step's timesteps.
// mse_kernel<kL2, false> is the plain MSE above: its body is unchanged, and `terms` is never read.
enum LossForm { kL2 = 0, kHuber = 1, kSmoothL1 = 2 };   // = T2V_LOSS_*
struct LossTerms {
    float huber_c;      // c of T2V_HUBER_CONSTANT, and the floor of T2V_HUBER_SNR
    float log_c_per_t;  // ln(huber_c) / T: T2V_HUBER_EXPONENTIAL's c_b = exp(t_b ln(huber_c) / T)
    float snr_gamma;
    int schedule;       // T2V_HUBER_*
};

// Min-SNR-gamma weight, snr = a / (1 - a), written without dividing by 1 - a:
//   epsilon  min(snr, gamma) / snr       = min(1, gamma (1 - a) / a), whose limit at a = 0 (snr = 0) is 1;
//   v        min(snr, gamma) / (snr + 1) = min(a, gamma (1 - a)), which is 0 at a = 0 without a special case.
__device__ __forceinline__ float min_snr_weight(float a, float gamma, bool velocity) {
    if (velocity) return fminf(a, gamma * (1.f - a));
    return a > 0.f ? fminf(1.f, __fdividef(gamma * (1.f - a), a)) : 1.f;   // a in (0, 1]: both operands finite
}
// Huber scale of sample b.  T2V_HUBER_SNR: (1 - c) / (1 + sigma)^2 + c with sigma = sqrt((1 - a) / a) is
// (1 - c) a / (sqrt(a) + sqrt(1 - a))^2 + c, whose denominator is >= 1: finite at a = 0, where it is c.
__device__ __forceinline__ float huber_scale(const LossTerms& lt, float a, int64_t tb) {
    if (lt.schedule == T2V_HUBER_EXPONENTIAL) return expf(float(tb) * lt.log_c_per_t);
    if (lt.schedule == T2V_HUBER_SNR) {
        const float s = sqrtf(a) + sqrtf(1.f - a);
        return __fdividef((1.f - lt.huber_c) * a, s * s) + lt.huber_c;
    }
    return lt.huber_c;
}
// psi(e) and psi'(e) of the pseudo-Huber forms.  sqrt(e^2 + c^2) - c is formed as e^2 / (sqrt(e^2 + c^2) + c), which keeps
// its relative precision for |e| << c.  c >= huber_c > 0, so both denominators are positive and finite.
template <int FORM>
__device__ __forceinline__ void huber_terms(float e, float c, float& psi, float& dpsi) {
    const float q = fmaxf(fmaf(e, e, c * c), 1e-30f);   // c^2 underflows only for c < 1e-19
    const float r = rsqrtf(q);                 // 1 / sqrt(e^2 + c^2)
    const float k = FORM == kHuber ? 2.f * c : 2.f;
    psi = __fdividef(k * e * e, fmaf(q, r, c));
    dpsi = k * e * r;
}

template <int FORM, bool WEIGHTED>
__global__ void __launch_bounds__(256, 6) mse_kernel(const __nv_bfloat16* __restrict__ pred, const float* __restrict__ target, float* __restrict__ loss,
                           const float* __restrict__ gout, __nv_bfloat16* __restrict__ dpred, int B, int C, int F, int HW,
                           const float* __restrict__ x0, const float* __restrict__ abar, const int64_t* __restrict__ t,
                           LossTerms terms) {
    constexpr bool kPlain = FORM == kL2 && !WEIGHTED;
    pdl_sync();
    const int64_t npix = int64_t(B) * F * HW;
    const float inv = 1.0f / (float(npix) * C);
    const float g = (dpred && gout) ? *gout : 1.0f;
    float acc = 0.f;
    GRID_STRIDE(i, npix) {
        const int hw = int(i % HW);
        const int f = int((i / HW) % F);
        const int b = int(i / (int64_t(HW) * F));
        const int64_t src = (int64_t(b) * C * F + f) * HW + hw, cstride = int64_t(F) * HW;
        float sa = 1.f, sb = 0.f, a = 0.f, hc = 1.f;
        if constexpr (kPlain) {
            if (x0) {
                const float a = abar[t[b]];
                sa = sqrtf(a);
                sb = sqrtf(1.f - a);
            }
        } else {
            const int64_t tb = t[b];
            a = abar[tb];
            if (x0) {
                sa = sqrtf(a);
                sb = sqrtf(1.f - a);
            }
            if constexpr (FORM != kL2) hc = huber_scale(terms, a, tb);
        }
        float v[8], d[8], px = 0.f;   // px: sum of psi over the pixel's channels, weighted once below
        unpack8e(__ldg(reinterpret_cast<const uint4*>(pred) + i), v);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float e = 0.f;
            if (c < C) {
                float y = target[src + c * cstride];
                if (x0) y = sa * y - sb * x0[src + c * cstride];
                e = v[c] - y;
            }
            if constexpr (kPlain) {
                acc += e * e;
                d[c] = 2.f * e * inv * g;
            } else if constexpr (FORM == kL2) {
                px += e * e;
                d[c] = 2.f * e;
            } else {
                huber_terms<FORM>(e, hc, v[c], d[c]);   // v[c] <- psi, d[c] <- psi'
                px += v[c];
            }
        }
        if constexpr (!kPlain) {
            const float w = WEIGHTED ? min_snr_weight(a, terms.snr_gamma, x0 != nullptr) : 1.f;
            const float wg = w * inv * g;
#pragma unroll
            for (int c = 0; c < 8; ++c) d[c] *= wg;
            acc = fmaf(w, px, acc);
        }
        if (dpred) reinterpret_cast<uint4*>(dpred)[i] = pack8e(d);
    }
    if (loss) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        __shared__ float ws[32];
        if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x < 32) {
            float a = threadIdx.x < (blockDim.x >> 5) ? ws[threadIdx.x] : 0.f;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
            if (threadIdx.x == 0) atomicAdd(loss, a * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------ activations
// GEGLU: proj [M][2I] -> out [M][I] = h * gelu(gate)   (diffusers GEGLU; exact erf GELU)
__global__ void geglu_fwd_kernel(const __nv_bfloat16* __restrict__ proj, __nv_bfloat16* __restrict__ out, int64_t M, int I) {
    pdl_sync();
    const int V = I >> 3;
    GRID_STRIDE(i, M * V) {
        const int64_t m = i / V;
        const int cv = int(i % V);
        float h[8], g[8];
        const uint4* row = reinterpret_cast<const uint4*>(proj + m * 2 * I);
        unpack8e(__ldg(row + cv), h);
        unpack8e(__ldg(row + V + cv), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] *= gelu_erf(g[j]);
        reinterpret_cast<uint4*>(out)[i] = pack8e(h);
    }
}
// y = gelu(x) (exact erf form, or CLIP's quick_gelu x * sigmoid(1.702 x)): the MLP activation of the frozen text encoder
__global__ void gelu_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t nvec, int quick) {
    pdl_sync();
    GRID_STRIDE(i, nvec) {
        float v[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(x) + i), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = quick ? v[j] / (1.f + __expf(-1.702f * v[j])) : gelu_erf(v[j]);
        reinterpret_cast<uint4*>(y)[i] = pack8e(v);
    }
}
// dx = dy * gelu'(x): the backward of gelu_kernel, both forms (text-encoder LoRA training).  x is the saved fc1 output.
//   quick_gelu: d/dx [x s(1.702 x)] = s + 1.702 x s (1 - s)
__global__ void gelu_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx,
                                int64_t nvec, int quick) {
    pdl_sync();
    GRID_STRIDE(i, nvec) {
        float v[8], d[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(x) + i), v);
        unpack8e(__ldg(reinterpret_cast<const uint4*>(dy) + i), d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float g;
            if (quick) {
                const float s = sigm(1.702f * v[j]);
                g = s + 1.702f * v[j] * s * (1.f - s);
            } else {
                g = gelu_erf_grad(v[j]);
            }
            d[j] *= g;
        }
        reinterpret_cast<uint4*>(dx)[i] = pack8e(d);
    }
}
// out[b*L + l][:] = tok_emb[ids[b][l]][:] + pos_emb[l][:]   (fp32 tables -> bf16 activations; CLIPTextEmbeddings)
__global__ void embed_tokens_kernel(const int64_t* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                                    __nv_bfloat16* __restrict__ out, int64_t rows, int L, int C, int vocab) {
    pdl_sync();
    const int V = C >> 3;
    GRID_STRIDE(i, rows * V) {
        const int64_t r = i / V;
        const int cv = int(i % V);
        int64_t id = ids[r];
        id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
        const float4* t4 = reinterpret_cast<const float4*>(tok + id * C) + 2 * cv;
        const float4* p4 = reinterpret_cast<const float4*>(pos + (r % L) * C) + 2 * cv;
        const float4 a = __ldg(t4), b = __ldg(t4 + 1), c = __ldg(p4), d = __ldg(p4 + 1);
        const float v[8] = {a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w, b.x + d.x, b.y + d.y, b.z + d.z, b.w + d.w};
        reinterpret_cast<uint4*>(out)[i] = pack8e(v);
    }
}
// Backward of embed_tokens_kernel, accumulated into the fp32 tables' gradients without atomics, so the sums are the same on
// every launch.  Blocks [0, n_tok) are token blocks, one per row r: a block whose (clamped) id already occurs in an earlier row
// exits, so exactly one block owns each id; it sums the rows with that id in row order and adds the sum to dtok[id] once.
// Padded prompts repeat one id dozens of times, so most rows exit after the scan.  Blocks [n_tok, n_tok + n_pos) are
// position blocks, one per l: dpos[l] += sum over b of dy[b*L + l], in b order.
__global__ void embed_tokens_bwd_kernel(const int64_t* __restrict__ ids, const __nv_bfloat16* __restrict__ dy, float* __restrict__ dtok,
                                        float* __restrict__ dpos, int64_t rows, int L, int C, int vocab, int n_tok) {
    pdl_sync();
    const int V = C >> 3;
    auto clamp_id = [&](int64_t r) {
        const int64_t id = __ldg(ids + r);
        return id < 0 ? int64_t(0) : (id >= vocab ? int64_t(vocab - 1) : id);
    };
    if (int(blockIdx.x) < n_tok) {
        const int64_t r = blockIdx.x;
        const int64_t id = clamp_id(r);
        int seen = 0;
        for (int64_t j = threadIdx.x; j < r && !seen; j += blockDim.x) seen = clamp_id(j) == id;
        if (__syncthreads_or(seen)) return;
        for (int cv = threadIdx.x; cv < V; cv += blockDim.x) {
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            for (int64_t j = r; j < rows; ++j) {
                if (clamp_id(j) != id) continue;
                float v[8];
                unpack8e(__ldg(reinterpret_cast<const uint4*>(dy + j * C) + cv), v);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] += v[k];
            }
            float4* g = reinterpret_cast<float4*>(dtok + id * C) + 2 * cv;
            float4 a = g[0], b = g[1];
            a.x += acc[0]; a.y += acc[1]; a.z += acc[2]; a.w += acc[3];
            b.x += acc[4]; b.y += acc[5]; b.z += acc[6]; b.w += acc[7];
            g[0] = a;
            g[1] = b;
        }
        return;
    }
    const int l = int(blockIdx.x) - n_tok;
    for (int cv = threadIdx.x; cv < V; cv += blockDim.x) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int64_t j = l; j < rows; j += L) {
            float v[8];
            unpack8e(__ldg(reinterpret_cast<const uint4*>(dy + j * C) + cv), v);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += v[k];
        }
        float4* g = reinterpret_cast<float4*>(dpos + int64_t(l) * C) + 2 * cv;
        float4 a = g[0], b = g[1];
        a.x += acc[0]; a.y += acc[1]; a.z += acc[2]; a.w += acc[3];
        b.x += acc[4]; b.y += acc[5]; b.z += acc[6]; b.w += acc[7];
        g[0] = a;
        g[1] = b;
    }
}
__global__ void geglu_bwd_kernel(const __nv_bfloat16* __restrict__ proj, const __nv_bfloat16* __restrict__ dout,
                                 __nv_bfloat16* __restrict__ dproj, int64_t M, int I) {
    pdl_sync();
    const int V = I >> 3;
    GRID_STRIDE(i, M * V) {
        const int64_t m = i / V;
        const int cv = int(i % V);
        float h[8], g[8], d[8], dh[8], dg[8];
        const uint4* row = reinterpret_cast<const uint4*>(proj + m * 2 * I);
        unpack8e(__ldg(row + cv), h);
        unpack8e(__ldg(row + V + cv), g);
        unpack8e(__ldg(reinterpret_cast<const uint4*>(dout) + i), d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            dh[j] = d[j] * gelu_erf(g[j]);
            dg[j] = d[j] * h[j] * gelu_erf_grad(g[j]);
        }
        uint4* orow = reinterpret_cast<uint4*>(dproj + m * 2 * I);
        orow[cv] = pack8e(dh);
        orow[V + cv] = pack8e(dg);
    }
}

// SiLU on a small fp32 tensor (time embedding path): y_bf16 = silu(x_f32);  backward: dx_f32 = dy_f32 * silu'(x)
__global__ void silu_f32_to_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t n, int apply) {
    pdl_sync();
    GRID_STRIDE(i, n) {
        const float v = x[i];
        y[i] = __float2bfloat16_rn(apply ? v * sigm(v) : v);
    }
}
__global__ void silu_bwd_f32_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, int64_t n,
                                    int accumulate) {
    pdl_sync();
    GRID_STRIDE(i, n) {
        const float v = x[i], s = sigm(v);
        const float g = dy[i] * s * (1.f + v * (1.f - s));
        dx[i] = accumulate ? dx[i] + g : g;
    }
}

__global__ void silu_bf16_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int64_t n) {
    pdl_sync();
    GRID_STRIDE(i, n) {
        const float v = __bfloat162float(x[i]);
        y[i] = __float2bfloat16_rn(v * sigm(v));
    }
}
__global__ void silu_bf16_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                                     __nv_bfloat16* __restrict__ dx, int64_t n) {
    pdl_sync();
    GRID_STRIDE(i, n) {
        const float v = __bfloat162float(x[i]), s = sigm(v);
        dx[i] = __float2bfloat16_rn(__bfloat162float(dy[i]) * s * (1.f + v * (1.f - s)));
    }
}

// out = a + b (+ c)   (gradient fan-in)
__global__ void add_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b,
                           const __nv_bfloat16* __restrict__ c, __nv_bfloat16* __restrict__ out, int64_t nvec) {
    pdl_sync();
    GRID_STRIDE(i, nvec) {
        float x[8], y[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(a) + i), x);
        unpack8e(__ldg(reinterpret_cast<const uint4*>(b) + i), y);
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] += y[j];
        if (c) {
            unpack8e(__ldg(reinterpret_cast<const uint4*>(c) + i), y);
#pragma unroll
            for (int j = 0; j < 8; ++j) x[j] += y[j];
        }
        reinterpret_cast<uint4*>(out)[i] = pack8e(x);
    }
}
__global__ void scale_bf16_kernel(const __nv_bfloat16* __restrict__ a, __nv_bfloat16* __restrict__ out, int64_t nvec, float alpha) {
    pdl_sync();
    GRID_STRIDE(i, nvec) {
        float x[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(a) + i), x);
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] *= alpha;
        reinterpret_cast<uint4*>(out)[i] = pack8e(x);
    }
}
__global__ void add_f32_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int64_t n) {
    pdl_sync();
    GRID_STRIDE(i, n) out[i] = a[i] + b[i];
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int64_t n) {
    pdl_sync();
    const int64_t nv = n >> 3;
    GRID_STRIDE(i, nv) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(src) + 2 * i);
        const float4 b = __ldg(reinterpret_cast<const float4*>(src) + 2 * i + 1);
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        reinterpret_cast<uint4*>(dst)[i] = pack8e(v);
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 7)) dst[(nv << 3) + threadIdx.x] = __float2bfloat16_rn(src[(nv << 3) + threadIdx.x]);
}

// Data pipeline (SURVEY 8(f) row 3; reference utils/dataset.py:22-41 normalize_input + the decoder's resize): decoded RGB frames
// uint8 [F][H0][W0][3] -> bilinear resize (half-pixel centres, as F.interpolate(align_corners=False)) -> x / 127.5 - 1 ->
// bf16 channels-last [F][h][w][8] (channels 3..7 zero): exactly the tensor AutoencoderKL.encode consumes, in one pass.
// One output pixel (x, y) of the frame at `base` [H0][W0][3]; sy = H0 / h, sx = W0 / w.  Both resize kernels below call this,
// so a clip resized inside a ragged batch is bitwise equal to the same clip resized alone.
__device__ __forceinline__ uint4 bilinear_px8(const uint8_t* __restrict__ base, int H0, int W0, float sy, float sx, int x, int y) {
    const float fy = fmaxf((y + 0.5f) * sy - 0.5f, 0.f), fx = fmaxf((x + 0.5f) * sx - 0.5f, 0.f);
    const int y0 = min(int(fy), H0 - 1), x0 = min(int(fx), W0 - 1);
    const int y1 = min(y0 + 1, H0 - 1), x1 = min(x0 + 1, W0 - 1);
    const float wy = fy - float(y0), wx = fx - float(x0);
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float p00 = base[(int64_t(y0) * W0 + x0) * 3 + c], p01 = base[(int64_t(y0) * W0 + x1) * 3 + c];
        const float p10 = base[(int64_t(y1) * W0 + x0) * 3 + c], p11 = base[(int64_t(y1) * W0 + x1) * 3 + c];
        const float top = p00 + (p01 - p00) * wx, bot = p10 + (p11 - p10) * wx;
        v[c] = (top + (bot - top) * wy) * (1.0f / 127.5f) - 1.0f;
    }
    return pack8e(v);
}

__global__ void frames_u8_to_nhwc8_kernel(const uint8_t* __restrict__ src, __nv_bfloat16* __restrict__ dst, int F, int H0, int W0, int h, int w) {
    pdl_sync();
    const int64_t total = int64_t(F) * h * w;
    const float sy = float(H0) / float(h), sx = float(W0) / float(w);
    GRID_STRIDE(i, total) {
        const int x = int(i % w), y = int((i / w) % h);
        const int f = int(i / (int64_t(w) * h));
        reinterpret_cast<uint4*>(dst)[i] = bilinear_px8(src + int64_t(f) * H0 * W0 * 3, H0, W0, sy, sx, x, y);
    }
}

// The same resize for a ragged batch of clips in ONE launch: clip k has F_k frames of its own native size H0_k x W0_k, stored
// at byte `offset_k` of one packed buffer; table = int64 [n_clips][4] (offset, F, H0, W0).  Output bf16 [sum F_k][h][w][8],
// clip after clip.  Every block stages the table in shared memory with the clips' first output frames (prefix sum of F) and
// scales, then walks output pixels grid-stride; a pixel finds its clip by binary search over the first frames.  Idx: the pixel
// index type - 32-bit whenever the output has < 2^31 pixels (every training batch), which turns the index divisions into
// 32-bit ones; 64-bit otherwise.
constexpr int kRaggedMaxClips = 256;
template <typename Idx>
__global__ void __launch_bounds__(256) frames_u8_to_nhwc8_ragged_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ table,
                                                                        int n_clips, int64_t total_frames, __nv_bfloat16* __restrict__ dst,
                                                                        int h, int w) {
    __shared__ int64_t s_off[kRaggedMaxClips];
    __shared__ int s_first[kRaggedMaxClips + 1], s_h0[kRaggedMaxClips], s_w0[kRaggedMaxClips];
    __shared__ float s_sy[kRaggedMaxClips], s_sx[kRaggedMaxClips];
    pdl_sync();
    for (int k = threadIdx.x; k < n_clips; k += blockDim.x) {
        const int64_t* row = table + 4 * k;
        s_off[k] = row[0];
        s_first[k + 1] = int(row[1]);   // frame count; turned into a prefix sum below
        s_h0[k] = int(row[2]);
        s_w0[k] = int(row[3]);
        s_sy[k] = float(s_h0[k]) / float(h);
        s_sx[k] = float(s_w0[k]) / float(w);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        s_first[0] = 0;
        for (int k = 0; k < n_clips; ++k) s_first[k + 1] += s_first[k];
    }
    __syncthreads();
    const Idx total = Idx(total_frames * h * w), W = Idx(w), HW = Idx(h) * Idx(w);
    for (Idx i = Idx(blockIdx.x) * Idx(blockDim.x) + Idx(threadIdx.x); i < total; i += Idx(gridDim.x) * Idx(blockDim.x)) {
        const Idx fi = i / HW, r = i - fi * HW;
        const int f = int(fi), y = int(r / W), x = int(r - (r / W) * W);
        int lo = 0, hi = n_clips - 1;   // last clip k with s_first[k] <= f
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (s_first[mid] <= f) lo = mid; else hi = mid - 1;
        }
        const int H0 = s_h0[lo], W0 = s_w0[lo];
        const uint8_t* base = src + s_off[lo] + int64_t(f - s_first[lo]) * H0 * W0 * 3;
        reinterpret_cast<uint4*>(dst)[i] = bilinear_px8(base, H0, W0, s_sy[lo], s_sx[lo], x, y);
    }
}

// Gradient compression for the data-parallel all-reduce: dst (bf16) = alpha * src (fp32); and its inverse (widening).
__global__ void scale_cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int64_t n, float alpha) {
    pdl_sync();
    const int64_t nv = n >> 3;
    GRID_STRIDE(i, nv) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(src) + 2 * i);
        const float4 b = __ldg(reinterpret_cast<const float4*>(src) + 2 * i + 1);
        const float v[8] = {a.x * alpha, a.y * alpha, a.z * alpha, a.w * alpha, b.x * alpha, b.y * alpha, b.z * alpha, b.w * alpha};
        reinterpret_cast<uint4*>(dst)[i] = pack8e(v);
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 7)) dst[(nv << 3) + threadIdx.x] = __float2bfloat16_rn(alpha * src[(nv << 3) + threadIdx.x]);
}
__global__ void cast_bf16_f32_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, int64_t n) {
    pdl_sync();
    const int64_t nv = n >> 3;
    GRID_STRIDE(i, nv) {
        float v[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(src) + i), v);
        reinterpret_cast<float4*>(dst)[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4*>(dst)[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 7)) dst[(nv << 3) + threadIdx.x] = __bfloat162float(src[(nv << 3) + threadIdx.x]);
}

// ------------------------------------------------------------------------------------------------ resampling / concat
// nearest-neighbour resize [N][H][W][C] -> [N][Ho][Wo][C]  (src = floor(dst * in / out), F.interpolate 'nearest')
__global__ void upsample_nearest_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int N, int H,
                                            int W, int Ho, int Wo, int C) {
    pdl_sync();
    const int V = C >> 3;
    const int64_t total = int64_t(N) * Ho * Wo * V;
    GRID_STRIDE(i, total) {
        const int cv = int(i % V);
        int64_t r = i / V;
        const int wo = int(r % Wo);
        r /= Wo;
        const int ho = int(r % Ho);
        const int n = int(r / Ho);
        const int hi = min(H - 1, int(int64_t(ho) * H / Ho)), wi = min(W - 1, int(int64_t(wo) * W / Wo));
        reinterpret_cast<uint4*>(y)[i] = __ldg(reinterpret_cast<const uint4*>(x) + ((int64_t(n) * H + hi) * W + wi) * V + cv);
    }
}
// backward of the nearest resize: dx[h][w] = sum of dy over the output pixels that read (h, w)
__global__ void upsample_nearest_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int N, int H,
                                            int W, int Ho, int Wo, int C) {
    pdl_sync();
    const int V = C >> 3;
    const int64_t total = int64_t(N) * H * W * V;
    GRID_STRIDE(i, total) {
        const int cv = int(i % V);
        int64_t r = i / V;
        const int w = int(r % W);
        r /= W;
        const int h = int(r % H);
        const int n = int(r / H);
        // floor(ho * H / Ho) == h  <=>  ceil(h Ho / H) <= ho < ceil((h+1) Ho / H)
        const int ho0 = int((int64_t(h) * Ho + H - 1) / H), ho1 = int((int64_t(h + 1) * Ho + H - 1) / H);
        const int wo0 = int((int64_t(w) * Wo + W - 1) / W), wo1 = int((int64_t(w + 1) * Wo + W - 1) / W);
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int a = ho0; a < ho1; ++a)
            for (int b = wo0; b < wo1; ++b) {
                float v[8];
                unpack8e(__ldg(reinterpret_cast<const uint4*>(dy) + ((int64_t(n) * Ho + a) * Wo + b) * V + cv), v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
            }
        reinterpret_cast<uint4*>(dx)[i] = pack8e(acc);
    }
}

// strided 2-D copy of bf16 rows: dst[m][dst_off + c] = src[m][src_off + c], c < C  (concat / split of channels)
__global__ void copy_cols_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int64_t M, int C,
                                 int src_ld, int src_off, int dst_ld, int dst_off) {
    pdl_sync();
    const int V = C >> 3;
    GRID_STRIDE(i, M * V) {
        const int64_t m = i / V;
        const int cv = int(i % V);
        *reinterpret_cast<uint4*>(dst + m * dst_ld + dst_off + cv * 8) =
            __ldg(reinterpret_cast<const uint4*>(src + m * src_ld + src_off + cv * 8));
    }
}

// ------------------------------------------------------------------------------------------------ reductions
// Segmented column sum: out[s][c] (+)= sum_p x[s][p][c].  Grid (chunks, S); per-thread 8-channel vectors.
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, int64_t P, int C, int chunk_rows,
                              int ld, int col0) {
    pdl_sync();  // C = width of this column block, ld = full row length, col0 = first column
    extern __shared__ float sh[];  // [C]
    const int s = blockIdx.y;
    const int V = C >> 3;
    const int lanes = blockDim.x / V;
    const int cv = threadIdx.x % V, pl = threadIdx.x / V;
    for (int i = threadIdx.x; i < C; i += blockDim.x) sh[i] = 0.f;
    __syncthreads();
    if (pl < lanes) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int64_t p0 = int64_t(blockIdx.x) * chunk_rows, p1 = min(P, p0 + chunk_rows);
        const uint4* xs = reinterpret_cast<const uint4*>(x + int64_t(s) * P * ld + col0) + cv;
        const int LV = ld >> 3;
        int64_t p = p0 + pl;
        for (; p + 3 * lanes < p1; p += 4 * lanes) {  // four 16-byte loads in flight per thread
            uint4 q[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) q[u] = __ldg(xs + (p + u * lanes) * LV);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float v[8];
                unpack8e(q[u], v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
            }
        }
        for (; p < p1; p += lanes) {
            float v[8];
            unpack8e(__ldg(xs + p * LV), v);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += v[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(&sh[cv * 8 + j], acc[j]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(out + int64_t(s) * ld + col0 + c, sh[c]);
}
// out[c] += sum_s x[s][c] for a small fp32 matrix
__global__ void colsum_f32_kernel(const float* __restrict__ x, float* __restrict__ out, int S, int C) {
    pdl_sync();
    GRID_STRIDE(c, C) {
        float a = 0.f;
        for (int s = 0; s < S; ++s) a += x[int64_t(s) * C + c];
        out[c] += a;
    }
}

// Row softmax over fp32 scores -> bf16 probabilities; columns >= n_valid (padding up to ld_out) are written as 0.
// causal_period > 0: row r attends to columns <= r % causal_period (CLIP text encoder's causal mask).
__global__ void softmax_fwd_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ p, int64_t rows, int n_valid_all, int ld_in,
                                   int ld_out, int causal_period) {
    pdl_sync();
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
    for (int64_t r = warp; r < rows; r += nwarps) {
        const int n_valid = causal_period > 0 ? min(n_valid_all, int(r % causal_period) + 1) : n_valid_all;
        const float* sr = s + r * ld_in;
        float mx = -INFINITY;
        for (int c = lane; c < n_valid; c += 32) mx = fmaxf(mx, sr[c]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
        for (int c = lane; c < n_valid; c += 32) sum += __expf(sr[c] - mx);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float inv = 1.f / sum;
        __nv_bfloat16* pr = p + r * ld_out;
        for (int c = lane; c < ld_out; c += 32) pr[c] = __float2bfloat16_rn(c < n_valid ? __expf(sr[c] - mx) * inv : 0.f);
    }
}
// dS = P * (dP - rowsum(dP * P)) * scale  -> bf16 (padding columns zero)
__global__ void softmax_bwd_kernel(const __nv_bfloat16* __restrict__ p, const float* __restrict__ dp, __nv_bfloat16* __restrict__ ds,
                                   int64_t rows, int n_valid, int ld_p, int ld_dp, float scale) {
    pdl_sync();
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
    for (int64_t r = warp; r < rows; r += nwarps) {
        const __nv_bfloat16* pr = p + r * ld_p;
        const float* dr = dp + r * ld_dp;
        float dot = 0.f;
        for (int c = lane; c < n_valid; c += 32) dot += __bfloat162float(pr[c]) * dr[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        __nv_bfloat16* o_ = ds + r * ld_p;
        for (int c = lane; c < ld_p; c += 32)
            o_[c] = __float2bfloat16_rn(c < n_valid ? __bfloat162float(pr[c]) * (dr[c] - dot) * scale : 0.f);
    }
}

// out = base + scale * x * mask / (1 - p), mask ~ Bernoulli(1 - p) from a counter-based generator keyed by
// (seed, element index): the backward pass regenerates the same mask instead of storing it.
__device__ __forceinline__ uint32_t mix32(uint64_t seed, uint64_t idx) {
    uint64_t z = seed + idx * 0x9E3779B97F4A7C15ull;  // splitmix64 finaliser: counter-based, stateless
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return uint32_t((z ^ (z >> 31)) >> 32);
}
__global__ void dropout_scale_add_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ base,
                                         __nv_bfloat16* __restrict__ out, int64_t nvec, float p, float scale, uint64_t seed,
                                         const int64_t* __restrict__ epoch) {
    pdl_sync();
    // `epoch` (device memory, bumped once per training step) keeps the masks of a replayed CUDA graph fresh: the host seed
    // is baked into the captured launch, the epoch is read when the kernel runs
    if (epoch) seed ^= uint64_t(*epoch) * 0xD1342543DE82EF95ull;
    const uint32_t thresh = uint32_t(double(p) * 4294967296.0);
    const float k = scale / (1.f - p);
    GRID_STRIDE(i, nvec) {
        float v[8], b[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(x) + i), v);
        if (base) unpack8e(__ldg(reinterpret_cast<const uint4*>(base) + i), b);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const bool keep = mix32(seed, uint64_t(i) * 8 + j) >= thresh;
            v[j] = (keep ? v[j] * k : 0.f) + (base ? b[j] : 0.f);
        }
        reinterpret_cast<uint4*>(out)[i] = pack8e(v);
    }
}

// DiagonalGaussianDistribution.sample() fused with tensor_to_vae_latent's rearrange and * 0.18215 (train.py:343-345):
// moments [B*F][HW][8] bf16 (mean = ch 0..3, logvar = ch 4..7)  ->  latents (B, 4, F, HW) fp32
__global__ void vae_sample_kernel(const __nv_bfloat16* __restrict__ mom, const float* __restrict__ eps, float* __restrict__ out,
                                  int B, int F, int HW, float scale) {
    pdl_sync();
    const int64_t npix = int64_t(B) * F * HW;
    GRID_STRIDE(i, npix) {
        const int hw = int(i % HW);
        const int f = int((i / HW) % F);
        const int b = int(i / (int64_t(HW) * F));
        float v[8];
        unpack8e(__ldg(reinterpret_cast<const uint4*>(mom) + i), v);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int64_t o = ((int64_t(b) * 4 + c) * F + f) * HW + hw;
            const float lv = fminf(fmaxf(v[4 + c], -30.f), 20.f);
            out[o] = (v[c] + expf(0.5f * lv) * eps[o]) * scale;
        }
    }
}

// Timesteps(dim, flip_sin_to_cos=True, shift=0): [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(10000) i / half)  -> bf16 [B][dim]
__global__ void timestep_embed_kernel(const int64_t* __restrict__ t, __nv_bfloat16* __restrict__ out, int B, int dim) {
    pdl_sync();
    const int half = dim >> 1;
    GRID_STRIDE(i, int64_t(B) * half) {
        const int b = int(i / half), k = int(i % half);
        const float f = expf(-9.210340371976184f * float(k) / float(half));
        const float a = float(t[b]) * f;
        out[int64_t(b) * dim + k] = __float2bfloat16_rn(cosf(a));
        out[int64_t(b) * dim + half + k] = __float2bfloat16_rn(sinf(a));
    }
}

}  // namespace t2v

using namespace t2v;
#define ST static_cast<cudaStream_t>(stream)
#define BF(p) static_cast<const __nv_bfloat16*>(p)
#define BFW(p) static_cast<__nv_bfloat16*>(p)

extern "C" {

int t2v_latents_to_nhwc8(const float* x0, const float* noise, const float* alphas_cumprod, const int64_t* timesteps, void* out,
                         int32_t B, int32_t C, int32_t F, int32_t HW, void* stream) {
    if (C > 8) return fail(-2, "latents_to_nhwc8: C=%d > 8", C);
    const int64_t n = int64_t(B) * F * HW;
    launch_pdl(to_nhwc8_kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, x0, noise, alphas_cumprod, timesteps, BFW(out), B, C, F, HW);
    return launch_checked(int(cudaGetLastError()), "latents_to_nhwc8");
}
int t2v_nhwc8_to_latents(const void* in, float* out, int32_t B, int32_t C, int32_t F, int32_t HW, void* stream) {
    const int64_t n = int64_t(B) * F * HW;
    launch_pdl(from_nhwc8_kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, BF(in), out, B, C, F, HW);
    return launch_checked(int(cudaGetLastError()), "nhwc8_to_latents");
}
int t2v_mse_loss(const void* pred, const float* target, float* loss, const float* gout, void* dpred, int32_t B, int32_t C,
                 int32_t F, int32_t HW, void* stream) {
    const int64_t n = int64_t(B) * F * HW;
    if (loss) cudaMemsetAsync(loss, 0, sizeof(float), ST);
    launch_pdl(mse_kernel<kL2, false>, dim3(ew_grid(n)), dim3(256), size_t(0), ST, BF(pred), target, loss, gout, BFW(dpred), B, C, F,
               HW, (const float*)nullptr, (const float*)nullptr, (const int64_t*)nullptr, LossTerms{});
    return launch_checked(int(cudaGetLastError()), "mse_loss");
}
int t2v_velocity_mse_loss(const void* pred, const float* x0, const float* noise, const float* alphas_cumprod, const int64_t* timesteps,
                          float* loss, const float* gout, void* dpred, int32_t B, int32_t C, int32_t F, int32_t HW, void* stream) {
    if (!x0 || !noise || !alphas_cumprod || !timesteps) return fail(-2, "velocity_mse_loss: x0, noise, alphas_cumprod and timesteps are required");
    if (C > 8) return fail(-2, "velocity_mse_loss: C=%d > 8", C);
    const int64_t n = int64_t(B) * F * HW;
    if (loss) cudaMemsetAsync(loss, 0, sizeof(float), ST);
    launch_pdl(mse_kernel<kL2, false>, dim3(ew_grid(n)), dim3(256), size_t(0), ST, BF(pred), noise, loss, gout, BFW(dpred), B, C, F,
               HW, x0, alphas_cumprod, timesteps, LossTerms{});
    return launch_checked(int(cudaGetLastError()), "velocity_mse_loss");
}
int t2v_diffusion_loss(const void* pred, const float* noise, const float* x0, const float* alphas_cumprod, const int64_t* timesteps,
                       const T2VLossParams* params, float* loss, const float* gout, void* dpred, int32_t B, int32_t C, int32_t F,
                       int32_t HW, void* stream) {
    if (!params) return fail(-2, "diffusion_loss: params is required");
    const T2VLossParams& p = *params;
    if (!noise || !alphas_cumprod || !timesteps) return fail(-2, "diffusion_loss: noise, alphas_cumprod and timesteps are required");
    if (p.prediction != T2V_PRED_EPSILON && p.prediction != T2V_PRED_V) return fail(-2, "diffusion_loss: prediction %d", p.prediction);
    if (p.prediction == T2V_PRED_V && !x0) return fail(-2, "diffusion_loss: v-prediction needs x0");
    if (p.loss < T2V_LOSS_L2 || p.loss > T2V_LOSS_SMOOTH_L1) return fail(-2, "diffusion_loss: loss %d", p.loss);
    if (p.loss != T2V_LOSS_L2) {
        if (p.huber_schedule < T2V_HUBER_CONSTANT || p.huber_schedule > T2V_HUBER_SNR)
            return fail(-2, "diffusion_loss: huber_schedule %d", p.huber_schedule);
        if (!(p.huber_c > 0.f)) return fail(-2, "diffusion_loss: huber_c = %g must be > 0", double(p.huber_c));
        if (p.huber_schedule == T2V_HUBER_EXPONENTIAL && (p.huber_c > 1.f || p.num_timesteps <= 0))
            return fail(-2, "diffusion_loss: the exponential schedule needs 0 < huber_c <= 1 and T > 0");
    }
    if (C > 8) return fail(-2, "diffusion_loss: C=%d > 8", C);
    const LossTerms lt{p.huber_c, p.num_timesteps > 0 ? float(std::log(double(p.huber_c)) / p.num_timesteps) : 0.f, p.snr_gamma,
                       p.huber_schedule};
    const float* v0 = p.prediction == T2V_PRED_V ? x0 : nullptr;   // the kernel forms the velocity when x0 is given
    const bool weighted = p.snr_gamma > 0.f;
    void (*kernel)(const __nv_bfloat16*, const float*, float*, const float*, __nv_bfloat16*, int, int, int, int, const float*,
                   const float*, const int64_t*, LossTerms) =
        p.loss == T2V_LOSS_HUBER     ? (weighted ? mse_kernel<kHuber, true> : mse_kernel<kHuber, false>)
        : p.loss == T2V_LOSS_SMOOTH_L1 ? (weighted ? mse_kernel<kSmoothL1, true> : mse_kernel<kSmoothL1, false>)
                                       : (weighted ? mse_kernel<kL2, true> : mse_kernel<kL2, false>);
    const int64_t n = int64_t(B) * F * HW;
    if (loss) cudaMemsetAsync(loss, 0, sizeof(float), ST);
    launch_pdl(kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, BF(pred), noise, loss, gout, BFW(dpred), B, C, F, HW, v0,
               alphas_cumprod, timesteps, lt);
    return launch_checked(int(cudaGetLastError()), "diffusion_loss");
}
int t2v_geglu_fwd(const void* proj, void* out, int64_t M, int32_t I, void* stream) {
    if (I % 8) return fail(-2, "geglu: inner dim %d not a multiple of 8", I);
    launch_pdl(geglu_fwd_kernel, dim3(ew_grid(M * (I / 8))), dim3(256), size_t(0), ST, BF(proj), BFW(out), M, I);
    return launch_checked(int(cudaGetLastError()), "geglu_fwd");
}
int t2v_geglu_bwd(const void* proj, const void* dout, void* dproj, int64_t M, int32_t I, void* stream) {
    if (I % 8) return fail(-2, "geglu: inner dim %d not a multiple of 8", I);
    launch_pdl(geglu_bwd_kernel, dim3(ew_grid(M * (I / 8))), dim3(256), size_t(0), ST, BF(proj), BF(dout), BFW(dproj), M, I);
    return launch_checked(int(cudaGetLastError()), "geglu_bwd");
}
int t2v_frames_u8_to_nhwc8(const uint8_t* src, void* dst, int32_t F, int32_t H0, int32_t W0, int32_t h, int32_t w, void* stream) {
    if (F <= 0 || H0 <= 0 || W0 <= 0 || h <= 0 || w <= 0) return fail(-2, "frames_u8_to_nhwc8: bad shape");
    launch_pdl(frames_u8_to_nhwc8_kernel, dim3(ew_grid(int64_t(F) * h * w)), dim3(256), size_t(0), ST, src, BFW(dst), F, H0, W0, h, w);
    return launch_checked(int(cudaGetLastError()), "frames_u8_to_nhwc8");
}
int t2v_frames_u8_to_nhwc8_ragged(const uint8_t* src, const int64_t* table, int32_t n_clips, int64_t total_frames, void* dst, int32_t h,
                                  int32_t w, void* stream) {
    if (n_clips <= 0 || n_clips > kRaggedMaxClips) return fail(-2, "frames_u8_to_nhwc8_ragged: %d clips (1..%d)", n_clips, kRaggedMaxClips);
    if (total_frames < n_clips || total_frames > INT32_MAX || h <= 0 || w <= 0) return fail(-2, "frames_u8_to_nhwc8_ragged: bad shape");
    const int64_t total = total_frames * h * w;
    // 32-bit indices need total + the grid's stride < 2^31 (the stride is at most 16 blocks of 256 per SM)
    if (total + int64_t(ew_grid(total)) * 256 < INT32_MAX)
        launch_pdl(frames_u8_to_nhwc8_ragged_kernel<int32_t>, dim3(ew_grid(total)), dim3(256), size_t(0), ST, src, table, int(n_clips),
                   total_frames, BFW(dst), int(h), int(w));
    else
        launch_pdl(frames_u8_to_nhwc8_ragged_kernel<int64_t>, dim3(ew_grid(total)), dim3(256), size_t(0), ST, src, table, int(n_clips),
                   total_frames, BFW(dst), int(h), int(w));
    return launch_checked(int(cudaGetLastError()), "frames_u8_to_nhwc8_ragged");
}
int t2v_gelu_bf16(const void* x, void* y, int64_t n, int32_t quick, void* stream) {
    if (n % 8) return fail(-2, "gelu: n must be a multiple of 8");
    launch_pdl(gelu_kernel, dim3(ew_grid(n / 8)), dim3(256), size_t(0), ST, BF(x), BFW(y), n / 8, quick);
    return launch_checked(int(cudaGetLastError()), "gelu_bf16");
}
int t2v_gelu_bwd_bf16(const void* x, const void* dy, void* dx, int64_t n, int32_t quick, void* stream) {
    if (n % 8) return fail(-2, "gelu_bwd: n must be a multiple of 8");
    launch_pdl(gelu_bwd_kernel, dim3(ew_grid(n / 8)), dim3(256), size_t(0), ST, BF(x), BF(dy), BFW(dx), n / 8, quick);
    return launch_checked(int(cudaGetLastError()), "gelu_bwd_bf16");
}
int t2v_embed_tokens(const int64_t* ids, const float* tok_emb, const float* pos_emb, void* out, int64_t rows, int32_t L, int32_t C,
                     int32_t vocab, void* stream) {
    if (C % 8) return fail(-2, "embed_tokens: C=%d must be a multiple of 8", C);
    launch_pdl(embed_tokens_kernel, dim3(ew_grid(rows * (C / 8))), dim3(256), size_t(0), ST, ids, tok_emb, pos_emb, BFW(out), rows, L, C, vocab);
    return launch_checked(int(cudaGetLastError()), "embed_tokens");
}
int t2v_embed_tokens_bwd(const int64_t* ids, const void* dy, float* dtok, float* dpos, int64_t rows, int32_t L, int32_t C, int32_t vocab,
                         void* stream) {
    if (C % 8) return fail(-2, "embed_tokens_bwd: C=%d must be a multiple of 8", C);
    if (rows <= 0 || L <= 0 || rows % L || vocab <= 0) return fail(-2, "embed_tokens_bwd: rows=%lld, L=%d, vocab=%d", (long long)rows, L, vocab);
    if (rows > INT32_MAX) return fail(-2, "embed_tokens_bwd: rows=%lld too large", (long long)rows);
    const int n_tok = dtok ? int(rows) : 0, n_pos = dpos ? L : 0;
    if (n_tok + n_pos == 0) return 0;
    launch_pdl(embed_tokens_bwd_kernel, dim3(n_tok + n_pos), dim3(128), size_t(0), ST, ids, BF(dy), dtok, dpos, rows, L, C, vocab, n_tok);
    return launch_checked(int(cudaGetLastError()), "embed_tokens_bwd");
}
int t2v_silu_f32_to_bf16(const float* x, void* y, int64_t n, int32_t apply_silu, void* stream) {
    launch_pdl(silu_f32_to_bf16_kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, x, BFW(y), n, apply_silu);
    return launch_checked(int(cudaGetLastError()), "silu_f32_to_bf16");
}
int t2v_silu_bwd_f32(const float* x, const float* dy, float* dx, int64_t n, int32_t accumulate, void* stream) {
    launch_pdl(silu_bwd_f32_kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, x, dy, dx, n, accumulate);
    return launch_checked(int(cudaGetLastError()), "silu_bwd_f32");
}
int t2v_silu_bf16(const void* x, void* y, int64_t n, void* stream) {
    launch_pdl(silu_bf16_kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, BF(x), BFW(y), n);
    return launch_checked(int(cudaGetLastError()), "silu_bf16");
}
int t2v_silu_bf16_bwd(const void* x, const void* dy, void* dx, int64_t n, void* stream) {
    launch_pdl(silu_bf16_bwd_kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, BF(x), BF(dy), BFW(dx), n);
    return launch_checked(int(cudaGetLastError()), "silu_bf16_bwd");
}
int t2v_add_bf16(const void* a, const void* b, const void* c, void* out, int64_t n, void* stream) {
    if (n % 8) return fail(-2, "add_bf16: n must be a multiple of 8");
    launch_pdl(add_kernel, dim3(ew_grid(n / 8)), dim3(256), size_t(0), ST, BF(a), BF(b), BF(c), BFW(out), n / 8);
    return launch_checked(int(cudaGetLastError()), "add_bf16");
}
int t2v_scale_bf16(const void* a, void* out, int64_t n, float alpha, void* stream) {
    if (n % 8) return fail(-2, "scale_bf16: n must be a multiple of 8");
    launch_pdl(scale_bf16_kernel, dim3(ew_grid(n / 8)), dim3(256), size_t(0), ST, BF(a), BFW(out), n / 8, alpha);
    return launch_checked(int(cudaGetLastError()), "scale_bf16");
}
int t2v_add_f32(const float* a, const float* b, float* out, int64_t n, void* stream) {
    launch_pdl(add_f32_kernel, dim3(ew_grid(n)), dim3(256), size_t(0), ST, a, b, out, n);
    return launch_checked(int(cudaGetLastError()), "add_f32");
}
int t2v_scale_cast_f32_bf16(const float* src, void* dst, int64_t n, float alpha, void* stream) {
    if ((reinterpret_cast<uintptr_t>(src) & 15u) || (reinterpret_cast<uintptr_t>(dst) & 15u)) return fail(-2, "scale_cast_f32_bf16: 16-byte alignment");
    launch_pdl(scale_cast_f32_bf16_kernel, dim3(ew_grid(std::max<int64_t>(n / 8, 1))), dim3(256), size_t(0), ST, src, BFW(dst), n, alpha);
    return launch_checked(int(cudaGetLastError()), "scale_cast_f32_bf16");
}
int t2v_cast_bf16_f32(const void* src, float* dst, int64_t n, void* stream) {
    if ((reinterpret_cast<uintptr_t>(src) & 15u) || (reinterpret_cast<uintptr_t>(dst) & 15u)) return fail(-2, "cast_bf16_f32: 16-byte alignment");
    launch_pdl(cast_bf16_f32_kernel, dim3(ew_grid(std::max<int64_t>(n / 8, 1))), dim3(256), size_t(0), ST, BF(src), dst, n);
    return launch_checked(int(cudaGetLastError()), "cast_bf16_f32");
}
int t2v_cast_f32_bf16(const float* src, void* dst, int64_t n, void* stream) {
    launch_pdl(cast_f32_bf16_kernel, dim3(ew_grid(std::max<int64_t>(n / 8, 1))), dim3(256), size_t(0), ST, src, BFW(dst), n);
    return launch_checked(int(cudaGetLastError()), "cast_f32_bf16");
}
int t2v_upsample_nearest_fwd(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t Ho, int32_t Wo, int32_t C, void* stream) {
    if (C % 8) return fail(-2, "upsample: C %% 8 != 0");
    launch_pdl(upsample_nearest_fwd_kernel, dim3(ew_grid(int64_t(N) * Ho * Wo * (C / 8))), dim3(256), size_t(0), ST, BF(x), BFW(y), N, H, W, Ho, Wo, C);
    return launch_checked(int(cudaGetLastError()), "upsample_nearest_fwd");
}
int t2v_upsample_nearest_bwd(const void* dy, void* dx, int32_t N, int32_t H, int32_t W, int32_t Ho, int32_t Wo, int32_t C, void* stream) {
    if (C % 8) return fail(-2, "upsample: C %% 8 != 0");
    launch_pdl(upsample_nearest_bwd_kernel, dim3(ew_grid(int64_t(N) * H * W * (C / 8))), dim3(256), size_t(0), ST, BF(dy), BFW(dx), N, H, W, Ho, Wo, C);
    return launch_checked(int(cudaGetLastError()), "upsample_nearest_bwd");
}
int t2v_copy_cols(const void* src, void* dst, int64_t M, int32_t C, int32_t src_ld, int32_t src_off, int32_t dst_ld, int32_t dst_off,
                  void* stream) {
    if (C % 8 || src_ld % 8 || src_off % 8 || dst_ld % 8 || dst_off % 8) return fail(-2, "copy_cols: all extents must be multiples of 8");
    launch_pdl(copy_cols_kernel, dim3(ew_grid(M * (C / 8))), dim3(256), size_t(0), ST, BF(src), BFW(dst), M, C, src_ld, src_off, dst_ld, dst_off);
    return launch_checked(int(cudaGetLastError()), "copy_cols");
}
int t2v_colsum(const void* x, float* out, int32_t S, int64_t P, int32_t C, void* stream) {
    if (C % 8) return fail(-2, "colsum: C=%d must be a multiple of 8", C);
    // ~2 blocks of 512 threads per SM: the final red.global.add per channel is only ~300 deep, and every thread keeps four
    // 16-byte loads in flight
    const int64_t want = std::max<int64_t>(1, (2 * int64_t(device_sm_count()) + S - 1) / S);
    const int chunk = int(std::min<int64_t>(P, std::max<int64_t>(16, (P + want - 1) / want)));
    const int chunks = int((P + chunk - 1) / chunk);
    for (int col0 = 0; col0 < C; col0 += 4096) {  // column blocks of <= 4096 channels (512 vectors per block row)
        const int cw = std::min(4096, C - col0);
        int bs = 512;
        while (bs < cw / 8) bs += 32;
        launch_pdl(colsum_kernel, dim3(dim3(chunks, S)), dim3(bs), size_t(cw * sizeof(float)), ST, BF(x), out, P, cw, chunk, C, col0);
        if (col0) count_launch();
    }
    return launch_checked(int(cudaGetLastError()), "colsum");
}
int t2v_colsum_f32(const float* x, float* out, int32_t S, int32_t C, void* stream) {
    launch_pdl(colsum_f32_kernel, dim3(ew_grid(C)), dim3(256), size_t(0), ST, x, out, S, C);
    return launch_checked(int(cudaGetLastError()), "colsum_f32");
}
int t2v_softmax_fwd(const float* s, void* p, int64_t rows, int32_t n_valid, int32_t ld_in, int32_t ld_out, int32_t causal_period,
                    void* stream) {
    const int grid = int(std::min<int64_t>((rows + 7) / 8, int64_t(device_sm_count()) * 16));
    launch_pdl(softmax_fwd_kernel, dim3(grid), dim3(256), size_t(0), ST, s, BFW(p), rows, n_valid, ld_in, ld_out, causal_period);
    return launch_checked(int(cudaGetLastError()), "softmax_fwd");
}
int t2v_softmax_bwd(const void* p, const float* dp, void* ds, int64_t rows, int32_t n_valid, int32_t ld_p, int32_t ld_dp, float scale,
                    void* stream) {
    const int grid = int(std::min<int64_t>((rows + 7) / 8, int64_t(device_sm_count()) * 16));
    launch_pdl(softmax_bwd_kernel, dim3(grid), dim3(256), size_t(0), ST, BF(p), dp, BFW(ds), rows, n_valid, ld_p, ld_dp, scale);
    return launch_checked(int(cudaGetLastError()), "softmax_bwd");
}
int t2v_dropout_scale_add(const void* x, const void* base, void* out, int64_t n, float p, float scale, uint64_t seed, const int64_t* epoch,
                          void* stream) {
    if (n % 8) return fail(-2, "dropout_scale_add: n must be a multiple of 8");
    if (!(p >= 0.f && p < 1.f)) return fail(-2, "dropout_scale_add: p=%f out of range", p);
    launch_pdl(dropout_scale_add_kernel, dim3(ew_grid(n / 8)), dim3(256), size_t(0), ST, BF(x), BF(base), BFW(out), n / 8, p, scale, seed, epoch);
    return launch_checked(int(cudaGetLastError()), "dropout_scale_add");
}
int t2v_vae_sample(const void* moments, const float* eps, float* out, int32_t B, int32_t F, int32_t HW, float scale, void* stream) {
    launch_pdl(vae_sample_kernel, dim3(ew_grid(int64_t(B) * F * HW)), dim3(256), size_t(0), ST, BF(moments), eps, out, B, F, HW, scale);
    return launch_checked(int(cudaGetLastError()), "vae_sample");
}
int t2v_timestep_embedding(const int64_t* t, void* out, int32_t B, int32_t dim, void* stream) {
    launch_pdl(timestep_embed_kernel, dim3(ew_grid(int64_t(B) * dim / 2)), dim3(256), size_t(0), ST, t, BFW(out), B, dim);
    return launch_checked(int(cudaGetLastError()), "timestep_embedding");
}

}  // extern "C"
