// Stable (loralib-style) LoRA on convolutions: the weight delta scaling * view(B @ A) is merged into the conv weight before
// the GEMM, and the gradient of the merged weight is projected back onto A and B.
//
// B @ A is [Cout*k][Cin*k] (A [r*k][Cin*k], B [Cout*k][r*k]); the module views it as the logical (Cout, Cin, k, k) weight
// (Conv2d) or averages triples of it into (Cout, Cin, 3, 1, 1) (Conv3d (3,1,1)).  Written as indices: with m = c*k + kh,
// j = m / Cin and q = m % Cin, the logical element (o, c, kh, kw) is BA[o*k + j][q*k + kw] (Conv3d: the mean over kw of
// BA[3o + j][3q + kw], j, q from m = 3c + t).  So a CTA that fixes j and takes a run of output channels o and a run of BA
// columns computes an ordinary GEMM tile  B[o*k + j, :] @ A[:, cols]  and scatters it into the channels-last weight
// [Cout][KH][KW][Cin] in runs of consecutive c.
//
// Arithmetic: at r = 16, k = 3 each BA element is a 48-term dot product (96 FLOP) against 6 B of weight traffic in the merge
// (fp32 base read, bf16 write) and 4 B in the gradient (fp32 dW read), so both kernels sit near the fp32 FFMA ridge.  They run
// fp32 FFMA on 32 x 96 register-blocked tiles out of shared memory: fp32 keeps the merged weight one bf16 rounding away from
// the exact value, and bf16 mma.sync would need a rounded copy of A and B for little gain at these K (12..192).
#include "common.h"
#include "ptx.cuh"

#include <cuda_bf16.h>

namespace t2v {
namespace {

constexpr int TO = 32;        // output channels (BA rows o*k + j) per CTA
constexpr int NC = 96;        // BA columns per CTA (a multiple of k = 1 and 3)
constexpr int KC = 32;        // chunk of the rank dimension r*k staged in shared memory
constexpr int THREADS = 256;  // 8 warps: warp ty owns rows ty*4 .. ty*4+3, lane tx owns columns tx, tx+32, tx+64

struct DeltaGeom {
    int cout, cin, k, rk, conv3d;
    float scaling;
};

// Range of m = c*k + kh covered by the tile (j, col0) and the c values that touch it.
struct TileRange {
    int q_lo, m_lo, m_hi, c_lo, cc;
};

__device__ __forceinline__ TileRange tile_range(const DeltaGeom& g, int j, int col0) {
    TileRange t;
    t.q_lo = col0 / g.k;
    const int q_hi = min(g.cin, t.q_lo + NC / g.k);
    t.m_lo = j * g.cin + t.q_lo;
    t.m_hi = j * g.cin + q_hi;
    t.c_lo = t.m_lo / g.k;
    t.cc = (t.m_hi - 1) / g.k - t.c_lo + 1;
    return t;
}

// Visits every weight element of the tile in channels-last order (c fastest): fn(i, n, dst) with tile row i, tile column n
// of the first BA column involved (Conv3d: the first of the three averaged columns) and the physical element index dst.
template <typename Fn>
__device__ __forceinline__ void for_each_weight(const DeltaGeom& g, int j, int o0, const TileRange& t, Fn fn) {
    const int k = g.k;
    const int taps = g.conv3d ? 3 : k * k;    // (kh, kw) pairs per output channel; Conv3d: 3 temporal taps
    const int total = TO * taps * t.cc;
    for (int e = threadIdx.x; e < total; e += THREADS) {
        const int cc = e % t.cc;
        const int rest = e / t.cc;
        const int tap = rest % taps;
        const int i = rest / taps;
        const int o = o0 + i;
        const int kh = g.conv3d ? tap : tap / k;
        const int kw = g.conv3d ? 0 : tap % k;
        const int c = t.c_lo + cc;
        const int m = c * k + kh;
        if (o >= g.cout || c >= g.cin || m < t.m_lo || m >= t.m_hi) continue;
        const int n = (m - t.m_lo) * k + kw;
        const int64_t dst = g.conv3d ? (int64_t(o) * 3 + kh) * g.cin + c : ((int64_t(o) * k + kh) * k + kw) * g.cin + c;
        fn(i, n, dst);
    }
}

__global__ void __launch_bounds__(THREADS) lora_delta_merge_kernel(const float* __restrict__ base, const float* __restrict__ A,
                                                                   const float* __restrict__ B, __nv_bfloat16* __restrict__ out,
                                                                   DeltaGeom g) {
    __shared__ float As[KC][NC];
    __shared__ float Bs[KC][TO + 1];
    __shared__ float Cs[TO][NC + 1];
    pdl_sync();
    const int col0 = blockIdx.x * NC, j = blockIdx.y, o0 = blockIdx.z * TO;
    const int ncol = g.cin * g.k;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    float acc[4][3] = {};
    for (int t0 = 0; t0 < g.rk; t0 += KC) {
        for (int idx = threadIdx.x; idx < KC * NC; idx += THREADS) {
            const int t = idx / NC, n = idx % NC;
            As[t][n] = (t0 + t < g.rk && col0 + n < ncol) ? A[int64_t(t0 + t) * ncol + col0 + n] : 0.f;
        }
        for (int idx = threadIdx.x; idx < KC * TO; idx += THREADS) {
            const int t = idx % KC, i = idx / KC;
            const int o = o0 + i;
            Bs[t][i] = (t0 + t < g.rk && o < g.cout) ? B[(int64_t(o) * g.k + j) * g.rk + t0 + t] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int t = 0; t < KC; ++t) {
            float bv[4], av[3];
#pragma unroll
            for (int a = 0; a < 4; ++a) bv[a] = Bs[t][ty * 4 + a];
#pragma unroll
            for (int b = 0; b < 3; ++b) av[b] = As[t][tx + 32 * b];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 3; ++b) acc[a][b] = fmaf(bv[a], av[b], acc[a][b]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) Cs[ty * 4 + a][tx + 32 * b] = acc[a][b];
    __syncthreads();
    const TileRange tr = tile_range(g, j, col0);
    for_each_weight(g, j, o0, tr, [&](int i, int n, int64_t dst) {
        const float d = g.conv3d ? (Cs[i][n] + Cs[i][n + 1] + Cs[i][n + 2]) / 3.f : Cs[i][n];
        out[dst] = __float2bfloat16_rn(base[dst] + g.scaling * d);
    });
}

// dBA = scaling * dW (Conv3d: scaling * dW / 3 on each averaged column), then per tile
//   dB[rows, :] += dBA_tile @ A[:, cols]^T        dA[:, cols] += B[rows, :]^T @ dBA_tile
// accumulated with red.global.add: a dB row receives Cin*k / 96 contributions and a dA column Cout / 32.  The order of those
// adds is not fixed, so the result is not bitwise reproducible - like the split-K weight-gradient GEMM that produces dW.
__global__ void __launch_bounds__(THREADS) lora_delta_grad_kernel(const float* __restrict__ dw, const float* __restrict__ A,
                                                                  const float* __restrict__ B, float* __restrict__ dA,
                                                                  float* __restrict__ dB, DeltaGeom g) {
    __shared__ float Gs[TO][NC + 1];
    __shared__ float As[KC][NC + 1];
    __shared__ float Bs[KC][TO + 1];
    pdl_sync();
    const int col0 = blockIdx.x * NC, j = blockIdx.y, o0 = blockIdx.z * TO;
    const int ncol = g.cin * g.k;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int idx = threadIdx.x; idx < TO * (NC + 1); idx += THREADS) (&Gs[0][0])[idx] = 0.f;
    __syncthreads();
    const TileRange tr = tile_range(g, j, col0);
    const float s = g.conv3d ? g.scaling / 3.f : g.scaling;
    for_each_weight(g, j, o0, tr, [&](int i, int n, int64_t src) {
        const float v = s * dw[src];
        Gs[i][n] = v;
        if (g.conv3d) {
            Gs[i][n + 1] = v;
            Gs[i][n + 2] = v;
        }
    });
    for (int t0 = 0; t0 < g.rk; t0 += KC) {
        __syncthreads();   // Gs complete (first chunk) / previous chunk's As, Bs consumed
        for (int idx = threadIdx.x; idx < KC * NC; idx += THREADS) {
            const int t = idx / NC, n = idx % NC;
            As[t][n] = (t0 + t < g.rk && col0 + n < ncol) ? A[int64_t(t0 + t) * ncol + col0 + n] : 0.f;
        }
        for (int idx = threadIdx.x; idx < KC * TO; idx += THREADS) {
            const int t = idx % KC, i = idx / KC;
            const int o = o0 + i;
            Bs[t][i] = (t0 + t < g.rk && o < g.cout) ? B[(int64_t(o) * g.k + j) * g.rk + t0 + t] : 0.f;
        }
        __syncthreads();
        {   // dB: lane tx = rank column t, warp ty = tile rows ty*4 .. +3, reduced over the 96 tile columns
            float acc[4] = {};
#pragma unroll 8
            for (int n = 0; n < NC; ++n) {
                const float av = As[tx][n];
#pragma unroll
                for (int a = 0; a < 4; ++a) acc[a] = fmaf(Gs[ty * 4 + a][n], av, acc[a]);
            }
            const int t = t0 + tx;
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                const int o = o0 + ty * 4 + a;
                if (o < g.cout && t < g.rk) atomicAdd(dB + (int64_t(o) * g.k + j) * g.rk + t, acc[a]);
            }
        }
        {   // dA: warp ty = rank rows ty*4 .. +3, lane tx = tile columns tx, tx+32, tx+64, reduced over the 32 tile rows
            float acc[4][3] = {};
#pragma unroll 8
            for (int i = 0; i < TO; ++i) {
                float bv[4], gv[3];
#pragma unroll
                for (int a = 0; a < 4; ++a) bv[a] = Bs[ty * 4 + a][i];
#pragma unroll
                for (int b = 0; b < 3; ++b) gv[b] = Gs[i][tx + 32 * b];
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b) acc[a][b] = fmaf(bv[a], gv[b], acc[a][b]);
            }
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                const int t = t0 + ty * 4 + a;
                if (t >= g.rk) continue;
#pragma unroll
                for (int b = 0; b < 3; ++b) {
                    const int col = col0 + tx + 32 * b;
                    if (col < ncol) atomicAdd(dA + int64_t(t) * ncol + col, acc[a][b]);
                }
            }
        }
    }
}

int check_geom(const char* what, int cout, int cin, int k, int r, int conv3d, DeltaGeom* g) {
    if (conv3d ? k != 3 : (k != 1 && k != 3)) return fail(-2, "%s: kernel size %d%s not supported (Conv2d k in {1, 3}, Conv3d (3,1,1))", what, k, conv3d ? " (Conv3d)" : "");
    if (cout <= 0 || cin <= 0 || r <= 0 || r > 256) return fail(-2, "%s: bad shape cout %d cin %d r %d", what, cout, cin, r);
    if ((cout + TO - 1) / TO > 65535) return fail(-2, "%s: cout %d too large", what, cout);
    *g = DeltaGeom{cout, cin, k, r * k, conv3d, 0.f};
    return 0;
}

dim3 delta_grid(const DeltaGeom& g) { return dim3((g.cin * g.k + NC - 1) / NC, g.k, (g.cout + TO - 1) / TO); }

}  // namespace
}  // namespace t2v

extern "C" {

int t2v_lora_delta_merge(const float* base, const float* A, const float* B, float scaling, int32_t k, int32_t conv3d, int32_t cout,
                         int32_t cin, int32_t r, void* out_bf16, void* stream) {
    using namespace t2v;
    DeltaGeom g;
    if (int rc = check_geom("t2v_lora_delta_merge", cout, cin, k, r, conv3d, &g)) return rc;
    g.scaling = scaling;
    return launch_checked(launch_pdl(lora_delta_merge_kernel, delta_grid(g), dim3(THREADS), 0, static_cast<cudaStream_t>(stream), base, A,
                                     B, static_cast<__nv_bfloat16*>(out_bf16), g),
                          "t2v_lora_delta_merge");
}

int t2v_lora_delta_grad(const float* dw, const float* A, const float* B, float scaling, int32_t k, int32_t conv3d, int32_t cout,
                        int32_t cin, int32_t r, float* dA, float* dB, void* stream) {
    using namespace t2v;
    DeltaGeom g;
    if (int rc = check_geom("t2v_lora_delta_grad", cout, cin, k, r, conv3d, &g)) return rc;
    g.scaling = scaling;
    return launch_checked(launch_pdl(lora_delta_grad_kernel, delta_grid(g), dim3(THREADS), 0, static_cast<cudaStream_t>(stream), dw, A, B,
                                     dA, dB, g),
                          "t2v_lora_delta_grad");
}

}  // extern "C"
