// GroupNorm (+SiLU) and LayerNorm, forward and backward, for channels-last bf16 activations.
// HBM-bound kernels: 128-bit loads, fp32 statistics, warp-shuffle / shared-memory reductions.
//
// GroupNorm works on x [S][P][C]: S normalisation samples (frames for the per-frame norms of ResnetBlock2D /
// Transformer2DModel, clips for the per-clip norms of TemporalConvLayer / TransformerTemporalModel), P pixels per
// sample, C channels in G groups.  Statistics are reduced in two levels (pixel chunks -> sample) so the grid fills
// the GPU even when S == 1.
#include "common.h"
#include "gemm_tc.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cuda_bf16.h>
#include <mutex>

namespace t2v {

__device__ __forceinline__ void unpack8(const uint4& q, float* v) {
    v[0] = bf16_lo(q.x); v[1] = bf16_hi(q.x); v[2] = bf16_lo(q.y); v[3] = bf16_hi(q.y);
    v[4] = bf16_lo(q.z); v[5] = bf16_hi(q.z); v[6] = bf16_lo(q.w); v[7] = bf16_hi(q.w);
}
__device__ __forceinline__ uint4 pack8(const float* v) {
    uint4 q;
    q.x = pack_bf16(v[0], v[1]); q.y = pack_bf16(v[2], v[3]); q.z = pack_bf16(v[4], v[5]); q.w = pack_bf16(v[6], v[7]);
    return q;
}
// sigmoid with a small RELATIVE error for every z (ex2.approx + rcp.approx, a few ulps): SiLU(z) = z sigmoid(z) is small for
// z < 0, so an absolute error in sigmoid is a relative error in SiLU and its derivative.  (0.5 tanh.approx(z / 2) + 0.5, one
// MUFU op instead of two, put SiLU 1% off at z = -9.7, 5% off at z = -13.6 and at 0 instead of -1.8e-6 at z = -16 on an H100:
// tests/test_norm_step_gpu.py.)  For z < -88 the result is 0.
__device__ __forceinline__ float sigmoidf_(float z) {
    float e, r;   // ftz forms: the non-ftz ones add denormal scaling around each MUFU op (+13% instructions in the forward)
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * z));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return r;
}

// ------------------------------------------------------------------------------------------------ GroupNorm
// Streaming kernels with many small blocks (<= 256 threads, several resident per SM, so the per-block latency chain
// "sums -> group statistics -> coefficients -> pixels" of one block overlaps the streaming of its neighbours):
//   forward    [sums] -> apply      sums: per-(sample, channel) (sum x, sum x^2).  Usually NOT run: the GEMM that produced x
//                                   accumulated them in its epilogue (gemm_tc.cu, EPI_STATS), at the granularity this norm
//                                   needs (per frame or per clip), so forward is ONE kernel: one read + one write of x.
//   backward   sums   -> apply      sums: per-channel (sum dz, sum dz*xhat), red.add into zeroed scratch
//   apply      every block finalises ITS sample's group statistics from the per-channel sums (C values from L2, fp64 group
//              combine) and then streams its chunk of pixels; the sample's first block also writes stat / ab (forward) or
//              dgamma / dbeta (backward).
// Layout: V = C/8 channel vectors; a thread owns vector tid % V (its coefficients live in registers) and pixel lane
// tid / V; loads are 16 bytes, four pixels in flight per thread.
struct GnArgs {
    const __nv_bfloat16* x;
    const __nv_bfloat16* dy;
    const __nv_bfloat16* add;
    __nv_bfloat16* out;       // y (fwd) / dx (bwd)
    const float* gamma;
    const float* beta;
    float* stat;              // [S][G][2] (mean, rstd): written by fwd, read by bwd
    float* ab;                // [S][C][2] (a, b) with z = a x + b: written by fwd, read by bwd
    float* accum;             // [S][C][2] sums (bwd; fwd when the kernel computes them itself)
    const float* stats0;      // fwd input: per-frame sums of channels [0, C0), row pitch ld0 channels
    const float* stats1;      // ... of channels [C0, C), row pitch ld1 (NULL when C0 == C)
    int64_t ld0, ld1;
    float* dgamma;
    float* dbeta;
    int64_t P;
    int C, C0, G, fps, chunk_pixels, chunks, silu, lanes;
    float eps;
};

enum { GN_FWD_APPLY = 0, GN_BWD_SUMS = 1, GN_BWD_APPLY = 2, GN_FWD_SUMS = 3 };
constexpr int GN_CSLOTS = 8;   // channels per thread in the statistics prologue: C / blockDim.x <= 8 (gn_stream)

template <int MODE>
__global__ void __launch_bounds__(384, MODE == GN_BWD_SUMS ? 1 : 2) gn_stream_kernel(const GnArgs g) {
    pdl_sync();
    extern __shared__ float sh[];  // apply: [2][C] per-channel sums, [2][G] group terms (bwd: + [C] gamma, [G] float2 stat);
                                   // sums: [4][blockDim] float4
    constexpr bool kSums = MODE == GN_BWD_SUMS || MODE == GN_FWD_SUMS;
    constexpr bool kBwd = MODE == GN_BWD_SUMS || MODE == GN_BWD_APPLY;
    const int C = g.C, G = g.G, cpg = C / G;
    const int s = blockIdx.x / g.chunks, chunk = blockIdx.x % g.chunks;
    const int V = C >> 3;
    const int lanes = g.lanes;
    const int cv = threadIdx.x % V, pl = threadIdx.x / V;
    // block-local 32-bit addressing: the chunk starts at pixel p0 of sample s; this thread walks pixels pl, pl + lanes, ...
    const int64_t p0 = int64_t(chunk) * g.chunk_pixels;
    const int np = int(min(g.P, p0 + g.chunk_pixels) - p0);          // pixels of this chunk
    const int64_t base = (int64_t(s) * g.P + p0) * V + cv;            // in 16-byte vectors
    const uint4* xs = reinterpret_cast<const uint4*>(g.x) + base;
    const uint4* ds = kBwd ? reinterpret_cast<const uint4*>(g.dy) + base : nullptr;
    const int stepv = lanes * V;                                      // vector stride between a thread's consecutive pixels
    float* cs = sh;              // [2][C]
    float* t0 = sh + 2 * C;      // [G]  fwd: group mean   bwd: sum_c gamma * sum dz
    float* t1 = t0 + G;          // [G]  fwd: group rstd   bwd: sum_c gamma * sum dz*xhat
    float* gs = t1 + G;          // [C]  bwd: gamma
    float2* ss = reinterpret_cast<float2*>(gs + C);   // [G] bwd apply: (mean, rstd)
    float a[8], b[8], gam[8];

    // backward modes: saved per-channel coefficients.  The sums pass needs them first; the apply pass fetches (a, b) after
    // the statistics loads, so that they land during the group combine instead of holding registers across the prologue, and
    // reads (mean, rstd) from shared memory, where the prologue put them
    float mean[8], rstd[8];
    auto load_ab = [&]() {
        const float4* ab4 = reinterpret_cast<const float4*>(g.ab + (int64_t(s) * C + cv * 8) * 2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 q = __ldg(ab4 + j);
            a[2 * j] = q.x; b[2 * j] = q.y; a[2 * j + 1] = q.z; b[2 * j + 1] = q.w;
        }
    };
    if (MODE == GN_BWD_SUMS) {
        load_ab();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = cv * 8 + j;
            mean[j] = __ldg(g.stat + (int64_t(s) * G + c / cpg) * 2);
            rstd[j] = __ldg(g.stat + (int64_t(s) * G + c / cpg) * 2 + 1);
        }
    }
    // apply modes: this thread's first pixels do not depend on the statistics - their loads are issued now and land while the
    // block finalises its sample's statistics (one L2 round trip and two barriers)
    constexpr int UA = MODE == GN_FWD_APPLY ? 4 : 2;
    uint4 fx[UA], fd[UA];
    if (!kSums) {
#pragma unroll
        for (int u = 0; u < UA; ++u) {
            if (pl + u * lanes < np) {
                fx[u] = __ldg(xs + (pl + u * lanes) * V);
                if (MODE == GN_BWD_APPLY) {
                    fd[u] = __ldg(ds + (pl + u * lanes) * V);
                }
            }
        }
    }

    if (!kSums) {
        // ---- finalise this sample's statistics (redundantly per block: C values from L2, one round trip)
        // blockDim.x = V * lanes >= C / 8, so a thread owns at most GN_CSLOTS of the C channels: all its loads are issued
        // before the first use, one L2 round trip instead of one per channel slot
        if (MODE == GN_FWD_APPLY) {
            float2 sum[GN_CSLOTS];
#pragma unroll
            for (int i = 0; i < GN_CSLOTS; ++i) sum[i] = make_float2(0.f, 0.f);
            for (int f = 0; f < g.fps; ++f) {   // a few slots per sample (layers.clip_stats_rows)
#pragma unroll
                for (int i = 0; i < GN_CSLOTS; ++i) {
                    const int c = threadIdx.x + i * blockDim.x;
                    if (c < C) {
                        const bool first = c < g.C0;
                        const float2* src = reinterpret_cast<const float2*>(first ? g.stats0 : g.stats1) + (first ? c : c - g.C0);
                        const float2 v = __ldcg(src + (int64_t(s) * g.fps + f) * (first ? g.ld0 : g.ld1));
                        sum[i].x += v.x;
                        sum[i].y += v.y;
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < GN_CSLOTS; ++i) {
                const int c = threadIdx.x + i * blockDim.x;
                if (c < C) {
                    cs[c] = sum[i].x;
                    cs[C + c] = sum[i].y;
                }
            }
        } else {
            const float2* acc = reinterpret_cast<const float2*>(g.accum + int64_t(s) * C * 2);
            float2 v[GN_CSLOTS], ms[GN_CSLOTS];
            float w[GN_CSLOTS];
#pragma unroll
            for (int i = 0; i < GN_CSLOTS; ++i) {
                const int c = threadIdx.x + i * blockDim.x;
                if (c < C) {
                    v[i] = __ldcg(acc + c);
                    w[i] = __ldg(g.gamma + c);
                    if (c < G) ms[i] = __ldg(reinterpret_cast<const float2*>(g.stat) + int64_t(s) * G + c);
                }
            }
#pragma unroll
            for (int i = 0; i < GN_CSLOTS; ++i) {
                const int c = threadIdx.x + i * blockDim.x;
                if (c < C) {
                    cs[c] = v[i].x;
                    cs[C + c] = v[i].y;
                    gs[c] = w[i];
                    if (c < G) ss[c] = ms[i];
                    if (chunk == 0) {
                        if (g.dbeta) atomicAdd(g.dbeta + c, v[i].x);
                        if (g.dgamma) atomicAdd(g.dgamma + c, v[i].y);
                    }
                }
            }
        }
        __syncthreads();
        if (MODE == GN_FWD_APPLY) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                gam[j] = __ldg(g.gamma + cv * 8 + j);
                b[j] = __ldg(g.beta + cv * 8 + j);
            }
        } else {
            load_ab();
        }
        {   // full warps only: four lanes per group, eight groups per warp at a time, fp64 combine through shuffles
            const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
            if (warp < nw) {
                for (int g8 = warp * 8; g8 < G; g8 += nw * 8) {
                    const int gi = g8 + (lane >> 2);
                    double a0 = 0, a1 = 0;
                    if (gi < G) {
                        for (int j = lane & 3; j < cpg; j += 4) {
                            const int c = gi * cpg + j;
                            const double w = MODE == GN_FWD_APPLY ? 1.0 : double(gs[c]);
                            a0 += w * cs[c];
                            a1 += w * cs[C + c];
                        }
                    }
#pragma unroll
                    for (int o = 1; o < 4; o <<= 1) {
                        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
                        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
                    }
                    if (gi < G && (lane & 3) == 0) {
                        if (MODE == GN_FWD_APPLY) {
                            const double n = double(g.P) * cpg;
                            const double m = a0 / n;
                            double var = a1 / n - m * m;
                            if (var < 0) var = 0;
                            const float r = float(1.0 / sqrt(var + double(g.eps)));
                            t0[gi] = float(m);
                            t1[gi] = r;
                            if (chunk == 0) {
                                g.stat[(int64_t(s) * G + gi) * 2] = float(m);
                                g.stat[(int64_t(s) * G + gi) * 2 + 1] = r;
                            }
                        } else {
                            t0[gi] = float(a0);
                            t1[gi] = float(a1);
                        }
                    }
                }
            }
        }
        __syncthreads();
    }

    if (MODE == GN_FWD_APPLY) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = cv * 8 + j;
            a[j] = t1[c / cpg] * gam[j];
            b[j] = b[j] - t0[c / cpg] * a[j];
        }
        if (chunk == 0 && pl == 0) {
#pragma unroll
            for (int j = 0; j < 8; ++j) reinterpret_cast<float2*>(g.ab)[int64_t(s) * C + cv * 8 + j] = make_float2(a[j], b[j]);
        }
        uint4* os = reinterpret_cast<uint4*>(g.out) + base;
        auto apply = [&](const uint4& qx) {
            float v[8];
            unpack8(qx, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float z = a[j] * v[j] + b[j];
                if (g.silu) z *= sigmoidf_(z);
                v[j] = z;
            }
            return pack8(v);
        };
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (pl + u * lanes < np) os[(pl + u * lanes) * V] = apply(fx[u]);
        for (int p = pl + 4 * lanes, off = p * V; p < np; p += 4 * lanes, off += 4 * stepv) {   // four pixels in flight, predicated tail
            uint4 qx[4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (p + u * lanes < np) qx[u] = __ldg(xs + off + u * stepv);
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (p + u * lanes < np) os[off + u * stepv] = apply(qx[u]);
        }
        return;
    }

    if (kSums) {
        float acc0[8], acc1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc0[j] = acc1[j] = 0.f;
        auto accumulate = [&](const uint4& qx, const uint4& qd) {
            float v[8];
            unpack8(qx, v);
            if (MODE == GN_FWD_SUMS) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    acc0[j] += v[j];
                    acc1[j] += v[j] * v[j];
                }
            } else {
                float d[8];
                unpack8(qd, d);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float dz = d[j];
                    if (g.silu) {
                        const float z = a[j] * v[j] + b[j];
                        const float sg = sigmoidf_(z);
                        dz *= sg * (1.f + z * (1.f - sg));
                    }
                    acc0[j] += dz;
                    acc1[j] += dz * (v[j] - mean[j]) * rstd[j];
                }
            }
        };
        constexpr int U = MODE == GN_FWD_SUMS ? 4 : 2;
        for (int p = pl, off = pl * V; p < np; p += U * lanes, off += U * stepv) {
            uint4 qx[U], qd[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (p + u * lanes < np) {
                    qx[u] = __ldg(xs + off + u * stepv);
                    if (kBwd) qd[u] = __ldg(ds + off + u * stepv);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (p + u * lanes < np) accumulate(qx[u], qd[u]);
        }
        // Per-block reduction over the pixel lanes without shared-memory atomics (a float atomicAdd on shared memory is a CAS
        // loop on sm_90): every thread stages its 16 partials as [4][blockDim] float4, then one thread per channel sums
        // them over the lanes in lane order and issues one red.add.
        float4* st = reinterpret_cast<float4*>(sh) + threadIdx.x;
        st[0] = make_float4(acc0[0], acc0[1], acc0[2], acc0[3]);
        st[blockDim.x] = make_float4(acc0[4], acc0[5], acc0[6], acc0[7]);
        st[2 * blockDim.x] = make_float4(acc1[0], acc1[1], acc1[2], acc1[3]);
        st[3 * blockDim.x] = make_float4(acc1[4], acc1[5], acc1[6], acc1[7]);
        __syncthreads();
        float* acc = g.accum + int64_t(s) * C * 2;
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            const float* col = sh + ((c & 4) ? blockDim.x * 4 : 0) + (c >> 3) * 4 + (c & 3);   // float4 q = (c & 7) / 4, vector c / 8
            float s0 = 0.f, s1 = 0.f;
            for (int l = 0; l < lanes; ++l) {
                s0 += col[l * V * 4];
                s1 += col[l * V * 4 + blockDim.x * 8];
            }
            red_add_f32x2(acc + 2 * c, s0, s1);
        }
        return;
    }

    // GN_BWD_APPLY: dx = pc * dz + qc * x + rc (+ add)
    float pc[8], qc[8], rc[8];
    const float invn = 1.0f / (float(g.P) * cpg);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = cv * 8 + j;
        const float m = ss[c / cpg].x, r = ss[c / cpg].y;
        const float q = -r * r * t1[c / cpg] * invn;
        pc[j] = r * gs[c];
        qc[j] = q;
        rc[j] = -r * t0[c / cpg] * invn - q * m;
    }
    uint4* os = reinterpret_cast<uint4*>(g.out) + base;
    const uint4* as = g.add ? reinterpret_cast<const uint4*>(g.add) + base : nullptr;
    auto apply = [&](const uint4& qx, const uint4& qd, float* v) {
        float d[8];
        unpack8(qx, v);
        unpack8(qd, d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float dz = d[j];
            if (g.silu) {
                const float z = a[j] * v[j] + b[j];
                const float sg = sigmoidf_(z);
                dz *= sg * (1.f + z * (1.f - sg));
            }
            v[j] = pc[j] * dz + qc[j] * v[j] + rc[j];
        }
    };
    auto apply_add = [&](const uint4& qx, const uint4& qd, const uint4& qa) {
        float v[8], r[8];
        apply(qx, qd, v);
        unpack8(qa, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += r[j];
        return pack8(v);
    };
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        if (pl + u * lanes < np) {
            float v[8];
            if (as) {
                os[(pl + u * lanes) * V] = apply_add(fx[u], fd[u], __ldg(as + (pl + u * lanes) * V));
            } else {
                apply(fx[u], fd[u], v);
                os[(pl + u * lanes) * V] = pack8(v);
            }
        }
    }
    if (as) {   // residual gradient: one pixel (three vectors) in flight, which keeps the 80-register budget of the bound
        for (int p = pl + 2 * lanes, off = p * V; p < np; p += lanes, off += stepv)
            os[off] = apply_add(__ldg(xs + off), __ldg(ds + off), __ldg(as + off));
        return;
    }
    for (int p = pl + 2 * lanes, off = p * V; p < np; p += 2 * lanes, off += 2 * stepv) {
        uint4 qx[2], qd[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            if (p + u * lanes < np) {
                qx[u] = __ldg(xs + off + u * stepv);
                qd[u] = __ldg(ds + off + u * stepv);
            }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            if (p + u * lanes < np) {
                float v[8];
                apply(qx[u], qd[u], v);
                os[off + u * stepv] = pack8(v);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// One warp per row; the row lives in registers (VPL 16-byte vectors per lane), exact two-pass statistics.
template <int VPL>
__global__ void ln_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                              const float* __restrict__ beta, __nv_bfloat16* __restrict__ y, float* __restrict__ stat,
                              int64_t rows, int C, float eps) {
    pdl_sync();
    const int V = C >> 3;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
    // software pipeline over this warp's rows: the next row's vectors are in flight while the current row is reduced
    uint4 nx[VPL];
    auto fetch = [&](int64_t row) {
#pragma unroll
        for (int k = 0; k < VPL; ++k)
            if (lane + 32 * k < V) nx[k] = __ldg(reinterpret_cast<const uint4*>(x + row * C) + lane + 32 * k);
    };
    if (warp < rows) fetch(warp);
    for (int64_t row = warp; row < rows; row += nwarps) {
        float v[VPL][8];
        float sum = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = lane + 32 * k;
            if (cv < V) {
                unpack8(nx[k], v[k]);
#pragma unroll
                for (int j = 0; j < 8; ++j) sum += v[k][j];
            }
        }
        if (row + nwarps < rows) fetch(row + nwarps);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float mean = sum / C;
        float sq = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (lane + 32 * k < V) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float d = v[k][j] - mean;
                    sq += d * d;
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
        const float rstd = rsqrtf(sq / C + eps);
        if (lane == 0 && stat) {
            stat[row * 2] = mean;
            stat[row * 2 + 1] = rstd;
        }
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = lane + 32 * k;
            if (cv < V) {
                float o[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = (v[k][j] - mean) * rstd * __ldg(gamma + cv * 8 + j) + __ldg(beta + cv * 8 + j);
                reinterpret_cast<uint4*>(y + row * C)[cv] = pack8(o);
            }
        }
    }
}

// dx = rstd (dy g - mean_c(dy g) - xhat mean_c(dy g xhat)) (+ add); dgamma += sum_rows dy xhat; dbeta += sum_rows dy.
// Register budget: the per-lane parameter-gradient accumulators (16 VPL floats) are the only fp32 arrays that live across rows;
// the row itself stays packed (bf16, as loaded) and is unpacked twice - once for the row sums, once for dx - and gamma comes
// from L1 each time, so two 256-thread blocks stay resident per SM up to C = 640.
constexpr int LN_BWD_WARPS = 8;   // 256-thread blocks
constexpr size_t LN_BWD_SMEM = LN_BWD_WARPS * 4 * 32 * sizeof(float4);

template <int VPL>
__global__ void __launch_bounds__(LN_BWD_WARPS * 32, VPL <= 3 ? 2 : 1) ln_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                              const float* __restrict__ gamma, const float* __restrict__ stat,
                              const __nv_bfloat16* __restrict__ add, __nv_bfloat16* __restrict__ dx,
                              float* __restrict__ dgamma, float* __restrict__ dbeta, int64_t rows, int C) {
    pdl_sync();
    const int V = C >> 3;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * int64_t(blockDim.x) + threadIdx.x) >> 5;
    const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
    float gacc[VPL][8], bacc[VPL][8];
#pragma unroll
    for (int k = 0; k < VPL; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) gacc[k][j] = bacc[k][j] = 0.f;
    // software pipeline over this warp's rows: x, dy and the saved statistics of the next row are in flight while the
    // current row is reduced.  The dx pass takes the current row from a register copy where that copy fits the launch
    // bound's register budget next to the 16 VPL accumulators (128 registers for VPL <= 3, 255 above), and otherwise
    // re-reads it (L1 hits: the warp has just loaded it); ptxas -v shows no spills either way.
    constexpr bool kHold = VPL <= 2 || (VPL >= 4 && VPL <= 5);
    uint4 nx[VPL], nd[VPL];
    float2 nst = make_float2(0.f, 0.f);
    auto fetch = [&](int64_t row) {
        nst = __ldg(reinterpret_cast<const float2*>(stat) + row);
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            if (lane + 32 * k < V) {
                nx[k] = __ldg(reinterpret_cast<const uint4*>(x + row * C) + lane + 32 * k);
                nd[k] = __ldg(reinterpret_cast<const uint4*>(dy + row * C) + lane + 32 * k);
            }
        }
    };
    if (warp < rows) fetch(warp);
    for (int64_t row = warp; row < rows; row += nwarps) {
        const float mean = nst.x, rstd = nst.y;
        uint4 cx[kHold ? VPL : 1], cd[kHold ? VPL : 1];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = lane + 32 * k;
            if (cv < V) {
                if (kHold) {
                    cx[k] = nx[k];
                    cd[k] = nd[k];
                }
                float v[8], d[8];
                unpack8(nx[k], v);
                unpack8(nd[k], d);
                const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + cv * 2), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + cv * 2 + 1);
                const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float xh = (v[j] - mean) * rstd;
                    const float dg = d[j] * gm[j];
                    s1 += dg;
                    s2 += dg * xh;
                    gacc[k][j] += d[j] * xh;
                    bacc[k][j] += d[j];
                }
            }
        }
        if (row + nwarps < rows) fetch(row + nwarps);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
            s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        }
        s1 /= C;
        s2 /= C;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            const int cv = lane + 32 * k;
            if (cv < V) {
                float v[8], d[8], o[8], r[8];
                unpack8(kHold ? cx[k] : __ldg(reinterpret_cast<const uint4*>(x + row * C) + cv), v);
                unpack8(kHold ? cd[k] : __ldg(reinterpret_cast<const uint4*>(dy + row * C) + cv), d);
                if (add) unpack8(__ldg(reinterpret_cast<const uint4*>(add + row * C) + cv), r);
                const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + cv * 2), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + cv * 2 + 1);
                const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float xh = (v[j] - mean) * rstd;
                    o[j] = rstd * (d[j] * gm[j] - s1 - xh * s2);
                    if (add) o[j] += r[j];
                }
                reinterpret_cast<uint4*>(dx + row * C)[cv] = pack8(o);
            }
        }
    }
    // Block-level reduction of the parameter gradients, then one red.add per channel per block.  No shared-memory atomics:
    // a float atomicAdd on shared memory is a CAS loop on sm_90, and eight warps contending for the same 2C words cost more
    // than the rows themselves.  Per 32-channel-vector slice k, every warp stages its 16 partials per lane ([q][lane] float4,
    // conflict-free), then each thread sums one gamma and one beta partial over the eight warps in warp order.
    extern __shared__ float4 stage[];  // [LN_BWD_WARPS][4][32]
    const int wib = threadIdx.x >> 5;
    const int t = threadIdx.x, rl = (t >> 2) & 31, rc = (t >> 7) * 4 + (t & 3);   // reader: lane, channel within the vector
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        if (k) __syncthreads();
        float4* st = stage + wib * 128 + lane;
        st[0] = make_float4(gacc[k][0], gacc[k][1], gacc[k][2], gacc[k][3]);
        st[32] = make_float4(gacc[k][4], gacc[k][5], gacc[k][6], gacc[k][7]);
        st[64] = make_float4(bacc[k][0], bacc[k][1], bacc[k][2], bacc[k][3]);
        st[96] = make_float4(bacc[k][4], bacc[k][5], bacc[k][6], bacc[k][7]);
        __syncthreads();
        if (rl + 32 * k < V) {
            const float* sf = reinterpret_cast<const float*>(stage);
            float sg = 0.f, sb = 0.f;
#pragma unroll
            for (int w = 0; w < LN_BWD_WARPS; ++w) {
                sg += sf[w * 512 + t];
                sb += sf[w * 512 + 256 + t];
            }
            const int c = (rl + 32 * k) * 8 + rc;
            if (dgamma) atomicAdd(dgamma + c, sg);
            if (dbeta) atomicAdd(dbeta + c, sb);
        }
    }
}

// dynamic shared memory of gn_stream_kernel<MODE> (layout at its declaration of sh)
static size_t gn_smem(int mode, int C, int G, int threads) {
    if (mode == GN_BWD_SUMS || mode == GN_FWD_SUMS) return size_t(threads) * 4 * sizeof(float4);
    return size_t(2 * C + 2 * G + (mode == GN_BWD_APPLY ? C + 2 * G : 0)) * sizeof(float);
}

// Streaming geometry: threads = V * lanes (<= 256, or V itself up to 384 for the 2560- / 3072-channel concatenations), a
// block owns `chunk_pixels` pixels of one sample.  Apply modes: exactly ONE wave of blocks - as many as are resident at once
// (`resident` per SM, from the occupancy calculator) - so that every block's latency chain (statistics -> coefficients ->
// first pixels) overlaps its neighbours' streaming and no partial second wave pays that chain again (4 x SMs blocks with 3
// resident per SM ran as 1.33 waves = 2 block times).  Sums modes pay 2C atomics per block: fewer, longer blocks.
static void gn_plan(GnArgs& g, int S, bool sums, int resident) {
    const int V = g.C / 8;
    g.lanes = std::max(1, 256 / V);
    const int sms = device_sm_count();
    const int64_t blocks = sums ? 2 * int64_t(sms) : int64_t(std::max(1, resident)) * sms;
    const int64_t want = sums ? std::max<int64_t>(1, (blocks + S - 1) / S) : std::max<int64_t>(1, blocks / S);
    const int64_t min_px = int64_t(g.lanes) * (sums ? 8 : 4);
    const int64_t cp = std::max<int64_t>(min_px, (g.P + want - 1) / want);
    g.chunk_pixels = int(std::min<int64_t>(cp, g.P));
    g.chunks = int((g.P + g.chunk_pixels - 1) / g.chunk_pixels);
}

static int gn_check(const GnArgs& g) {
    if (g.C % 8 || g.C % g.G || g.C / 8 > 384 || gn_smem(GN_BWD_APPLY, g.C, g.G, 0) > 48 * 1024)
        return fail(-2, "groupnorm: C=%d G=%d unsupported", g.C, g.G);
    return 0;
}

// resident blocks per SM of gn_stream_kernel<MODE> for a block size (cached: the occupancy query is a driver call)
template <int MODE>
static int gn_resident(int threads, size_t smem) {
    static std::mutex mu;
    static int cache[13] = {};   // index: warps per block (threads <= 384)
    const int w = (threads + 31) / 32;
    std::lock_guard<std::mutex> lock(mu);
    if (cache[w] == 0) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gn_stream_kernel<MODE>, threads, smem) != cudaSuccess || n < 1) n = 2;
        cache[w] = n;
    }
    return cache[w];
}

template <int MODE>
static int gn_stream(GnArgs& g, int S, cudaStream_t st) {
    const bool sums = MODE == GN_BWD_SUMS || MODE == GN_FWD_SUMS;
    const int V = g.C / 8;
    const int threads = V * std::max(1, 256 / V);
    const size_t smem = gn_smem(MODE, g.C, g.G, threads);
    gn_plan(g, S, sums, sums ? 0 : gn_resident<MODE>(threads, smem));
    return int(launch_pdl(gn_stream_kernel<MODE>, dim3(S * g.chunks), dim3(V * g.lanes), smem, st, g));
}

// Standalone per-sample channel sums of x [S][P][C] into stats (+=), row pitch ld channels.  Used by t2v_channel_stats and
// by conv_fwd when a problem's tiling cannot produce the statistics in the GEMM epilogue.
int launch_channel_stats(const void* x, float* stats, int S, int64_t P, int C, int64_t ld, cudaStream_t st) {
    if (ld != C) return fail(-2, "channel_stats: row pitch %lld != C=%d is not supported by the standalone pass", (long long)ld, C);
    GnArgs g{};
    g.x = static_cast<const __nv_bfloat16*>(x);
    g.accum = stats;
    g.P = P; g.C = C; g.G = 1;
    if (int r = gn_check(g)) return r;
    return gn_stream<GN_FWD_SUMS>(g, S, st);
}

// Resident 256-thread blocks per SM of the LayerNorm kernels (occupancy calculator, cached per VPL): the grids are ONE wave of
// persistent blocks whose warps stride over the rows - a partial second wave would start only when first-wave blocks retire.
static int ln_resident(bool bwd, int vpl, size_t smem) {
    static std::mutex mu;
    static int cache[2][9] = {};
    vpl = std::min(std::max(vpl, 1), 8);
    std::lock_guard<std::mutex> lock(mu);
    int& c = cache[bwd ? 1 : 0][vpl];
    if (c == 0) {
        int n = 0;
        cudaError_t e = cudaErrorUnknown;
#define LN_OCC(K) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, K, 256, smem)
        switch (vpl) {
            case 1: if (bwd) LN_OCC(ln_bwd_kernel<1>); else LN_OCC(ln_fwd_kernel<1>); break;
            case 2: if (bwd) LN_OCC(ln_bwd_kernel<2>); else LN_OCC(ln_fwd_kernel<2>); break;
            case 3: if (bwd) LN_OCC(ln_bwd_kernel<3>); else LN_OCC(ln_fwd_kernel<3>); break;
            case 4: if (bwd) LN_OCC(ln_bwd_kernel<4>); else LN_OCC(ln_fwd_kernel<4>); break;
            case 5: if (bwd) LN_OCC(ln_bwd_kernel<5>); else LN_OCC(ln_fwd_kernel<5>); break;
            case 6: if (bwd) LN_OCC(ln_bwd_kernel<6>); else LN_OCC(ln_fwd_kernel<6>); break;
            case 7: if (bwd) LN_OCC(ln_bwd_kernel<7>); else LN_OCC(ln_fwd_kernel<7>); break;
            default: if (bwd) LN_OCC(ln_bwd_kernel<8>); else LN_OCC(ln_fwd_kernel<8>); break;
        }
#undef LN_OCC
        c = (e == cudaSuccess && n >= 1) ? n : (bwd ? 2 : 4);
    }
    return c;
}

}  // namespace t2v

using namespace t2v;

extern "C" {

int64_t t2v_groupnorm_workspace_bytes(int32_t S, int64_t P, int32_t C) {
    (void)P;
    return int64_t(S) * C * 2 * sizeof(float);
}

int t2v_channel_stats(const void* x, float* stats, int32_t S, int64_t P, int32_t C, int64_t ld, void* stream_) {
    return launch_checked(launch_channel_stats(x, stats, S, P, C, ld, static_cast<cudaStream_t>(stream_)), "channel_stats");
}

int t2v_groupnorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stat, float* ab, const float* stats0,
                      int32_t C0, int64_t ld0, const float* stats1, int64_t ld1, int32_t fps, void* workspace, int32_t S, int64_t P,
                      int32_t C, int32_t G, float eps, int32_t silu, void* stream_) {
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    GnArgs g{};
    g.x = static_cast<const __nv_bfloat16*>(x);
    g.out = static_cast<__nv_bfloat16*>(y);
    g.gamma = gamma; g.beta = beta; g.stat = stat; g.ab = ab;
    g.P = P; g.C = C; g.G = G; g.silu = silu; g.eps = eps;
    if (int r = gn_check(g)) return r;
    if (stats0) {
        if (fps < 1 || C0 <= 0 || C0 > C || (C0 < C && !stats1)) return fail(-2, "groupnorm_fwd: bad statistics arguments");
        g.stats0 = stats0; g.stats1 = stats1; g.C0 = C0; g.ld0 = ld0; g.ld1 = ld1; g.fps = fps;
    } else {
        if (!workspace) return fail(-3, "groupnorm_fwd: needs producer statistics or a zeroed workspace");
        g.accum = static_cast<float*>(workspace);
        if (int rc = gn_stream<GN_FWD_SUMS>(g, S, st)) return launch_checked(rc, "groupnorm_fwd(sums)");
        count_launch(1);
        g.stats0 = g.accum; g.stats1 = nullptr; g.C0 = C; g.ld0 = C; g.ld1 = 0; g.fps = 1;
    }
    return launch_checked(gn_stream<GN_FWD_APPLY>(g, S, st), "groupnorm_fwd");
}

int t2v_groupnorm_bwd(const void* dy, const void* x, const float* gamma, const float* stat, const float* ab, const void* add,
                      void* dx, float* dgamma, float* dbeta, void* workspace, int32_t S, int64_t P, int32_t C, int32_t G,
                      int32_t silu, void* stream_) {
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    GnArgs g{};
    g.x = static_cast<const __nv_bfloat16*>(x);
    g.dy = static_cast<const __nv_bfloat16*>(dy);
    g.add = static_cast<const __nv_bfloat16*>(add);
    g.out = static_cast<__nv_bfloat16*>(dx);
    g.gamma = gamma; g.stat = const_cast<float*>(stat); g.ab = const_cast<float*>(ab);
    g.dgamma = dgamma; g.dbeta = dbeta;
    g.P = P; g.C = C; g.G = G; g.silu = silu;
    if (int r = gn_check(g)) return r;
    if (!workspace) return fail(-3, "groupnorm_bwd: needs a zeroed workspace");
    g.accum = static_cast<float*>(workspace);
    if (int rc = gn_stream<GN_BWD_SUMS>(g, S, st)) return launch_checked(rc, "groupnorm_bwd(sums)");
    count_launch(1);
    return launch_checked(gn_stream<GN_BWD_APPLY>(g, S, st), "groupnorm_bwd");
}

#define LN_DISPATCH(KERNEL, GRID, SMEM, ST, ...)                                                       \
    switch (vpl) {                                                                                         \
        case 1: launch_pdl(KERNEL<1>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;       \
        case 2: launch_pdl(KERNEL<2>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;       \
        case 3: launch_pdl(KERNEL<3>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;       \
        case 4: launch_pdl(KERNEL<4>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;       \
        case 5: launch_pdl(KERNEL<5>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;       \
        case 6: launch_pdl(KERNEL<6>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;       \
        case 7: launch_pdl(KERNEL<7>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;       \
        default: launch_pdl(KERNEL<8>, dim3(GRID), dim3(256), size_t(SMEM), ST, __VA_ARGS__); break;      \
    }

int t2v_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stat, int64_t rows, int32_t C,
                      float eps, void* stream_) {
    if (C % 8 || C > 2048) return fail(-2, "layernorm: C=%d unsupported (multiple of 8, <= 2048)", C);
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const int vpl = (C / 8 + 31) / 32;
    const int grid = int(std::min<int64_t>((rows + 7) / 8, int64_t(device_sm_count()) * ln_resident(false, vpl, 0)));
    LN_DISPATCH(ln_fwd_kernel, grid, 0, st, static_cast<const __nv_bfloat16*>(x), gamma, beta, static_cast<__nv_bfloat16*>(y), stat,
                rows, C, eps);
    return launch_checked(int(cudaGetLastError()), "layernorm_fwd");
}

int t2v_layernorm_bwd(const void* dy, const void* x, const float* gamma, const float* stat, const void* add, void* dx,
                      float* dgamma, float* dbeta, int64_t rows, int32_t C, void* stream_) {
    if (C % 8 || C > 2048) return fail(-2, "layernorm: C=%d unsupported (multiple of 8, <= 2048)", C);
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const int vpl = (C / 8 + 31) / 32;
    const int grid = int(std::min<int64_t>((rows + 7) / 8, int64_t(device_sm_count()) * ln_resident(true, vpl, LN_BWD_SMEM)));
    LN_DISPATCH(ln_bwd_kernel, grid, LN_BWD_SMEM, st, static_cast<const __nv_bfloat16*>(x),
                static_cast<const __nv_bfloat16*>(dy), gamma, stat, static_cast<const __nv_bfloat16*>(add),
                static_cast<__nv_bfloat16*>(dx), dgamma, dbeta, rows, C);
    return launch_checked(int(cudaGetLastError()), "layernorm_bwd");
}

}  // extern "C"
