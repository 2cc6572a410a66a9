// "Affine TMA GEMM": one persistent, warp-specialised wgmma kernel that serves every contraction on the
// finetune hot path (linear, 3x3 / strided / temporal convolutions as implicit GEMM, their dgrad and wgrad,
// and the batched attention products).
//
//   D[tile] = sum over k-blocks  A_box(tile, kb) * B_box(tile, kb)^T       (bf16 in, fp32 accumulate in registers)
//
// Every operand tile is fetched by TMA from a rank<=5 tensor map.  The TMA coordinates are an *affine*
// function of six tile variables t[0..5] (decomposition of the linear tile id) and three k-loop variables
// k[0..2] (decomposition of the k-block id).  Zero padding of convolutions, ragged edges, channel tails and
// 4->8 channel padding all come from TMA out-of-bounds zero fill, so there is no im2col and no masking in the
// main loop.  The host-side planners in gemm_plan.cu only fill in the coefficient tables.
//
// Operand storage in shared memory is always the 128-byte-swizzle canonical wgmma layout:
//   K-major  operand: one box  {64 k-elems (128 B), rows}            -> [rows][128 B],      SBO = 1024
//   MN-major operand: n boxes  {64 mn-elems (128 B), 64 k-rows} each -> [n][64][128 B],     SBO = 1024, LBO = 8192
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace t2v {

constexpr int kBlockM = 128;      // two MMA warpgroups x wgmma M = 64
constexpr int kBlockK = 64;       // bf16 elements per k-block (= one 128-byte swizzle row)
constexpr int kMaxBlockN = 128;   // wgmma N; the fp32 accumulator is N / 2 registers per MMA thread
constexpr int kMaxStages = 8;
constexpr int kNumThreads = 512;  // warps 0-7: two MMA warpgroups, warps 8-11: TMA producer (one lane), warps 12-15: epilogue
constexpr int kEpilogueStagingBytes = 4 * 4096 + 4 * 128;  // per epilogue warp: a 32-row x 128-byte staging tile + 32 bias floats
// The finished accumulator goes through shared memory ([128 rows][N rounded up to 32] fp32, plus 128 row sums) so that the
// epilogue can own whole output rows.
constexpr int acc_smem_bytes(int block_n) { return kBlockM * ((block_n + 31) / 32 * 32) * 4 + kBlockM * 4; }
// Shared memory a launch may use besides the pipeline stages.
constexpr int gemm_fixed_smem_bytes(int block_n) { return 1024 /*align*/ + 256 /*barriers*/ + kEpilogueStagingBytes + acc_smem_bytes(block_n); }
constexpr int kMaxSmemBytes = 232448;  // 227 KB per block

struct alignas(64) TmaOperand {
    CUtensorMap map;
    int32_t base[5];
    int32_t tcoef[5][6];
    int32_t kcoef[5][3];
    int32_t rank;
    int32_t nbox;       // TMA boxes per pipeline stage
    int32_t box_dim;    // coordinate that advances between boxes
    int32_t box_step;   // ... by this many elements
    int32_t box_bytes;  // shared-memory bytes per box
    int32_t pad_[3];
};

enum OutMode : int32_t { OUT_BF16 = 0, OUT_F32 = 1, OUT_F32_RED = 2 };
enum EpiFlags : int32_t {
    EPI_BIAS = 1,       // + bias[col]                        (fp32)
    EPI_ROWBIAS = 2,    // + rowbias[gn * rb_ld + col]        (fp32; e.g. per-frame time-embedding projection)
    EPI_RESIDUAL = 4,   // + residual[same offset as out]     (bf16)
    EPI_VEC = 8,        // 16-byte vector access is legal for out/residual
    EPI_STATS = 16,     // accumulate per-(frame, channel) sum / sum of squares of the output into `stats` (GroupNorm input statistics)
    EPI_ROWSUM_A = 32,  // rowsum[row] += sum over K of operand A (weight gradient: A = dy^T, so this is the bias gradient)
};
constexpr int kOnesTileBytes = 2048;  // EPI_ROWSUM_A: a 16 x 64 K-major bf16 tile of ones in front of the pipeline stages

struct alignas(64) GemmParams {
    TmaOperand a, b;
    int32_t tdim[6];       // tile grid, t[0] fastest
    uint32_t tdiv_mul[6];  // magic numbers for division by tdim[i]
    uint32_t tdiv_shr[6];
    int32_t kdim[3];       // k-block grid, k[0] fastest
    int32_t num_tiles;
    int32_t kb_total;
    int32_t ksplit_var;    // tile variable that selects a k-range (split-K), or -1
    int32_t kb_per_split;
    int32_t block_n;       // wgmma N (multiple of 16, <= kMaxBlockN)
    int32_t num_stages;
    int32_t stage_bytes_a, stage_bytes_b;
    // epilogue: accumulator row r of a tile maps to the "pixel box" (w,h,n) = (r % bw, r / bw % bh, r / (bw*bh))
    // at global position (t[1]*bw + w, t[2]*bh + h, t[3]*bn + n); column c maps to t[0]*block_n + c.
    int32_t bw, bh, bn;
    int32_t W, H, N;       // row-space extents (rows beyond them are not stored)
    int32_t ncols;         // column extent
    int32_t out_mode;
    int32_t flags;
    float alpha;
    int64_t ldw, ldh, ldn; // element strides of the row-space coordinates in the output
    int64_t otc[6];        // extra element offset per tile variable
    int64_t rb_ld;
    int32_t rb_div;
    int32_t pad2_;
    void* out;
    const void* residual;
    const float* bias;
    const float* rowbias;
    // EPI_STATS: stats[(frame * st_ld + column) * 2 + {0, 1}] += {sum, sum of squares} over the rows of the tile, where
    // frame = (gw * st_cw + gh * st_ch + gn * st_cn) / st_div.  The planner guarantees that every aligned run of st_seg
    // (32 or 16) consecutive accumulator rows of a tile belongs to one frame.
    float* stats;
    int64_t st_ld;
    int32_t st_cw, st_ch, st_cn, st_div, st_seg;
    // EPI_ROWSUM_A: tiles with t[0] == t[2] == t[3] == 0 issue, next to every main MMA, an N = 16 MMA of the same A tile against
    // a constant tile of ones; the epilogue adds column 0 of that accumulator (16 identical columns) to rowsum[t[1] * bw + row]
    // (red.add: split-K partials sum up).
    float* rowsum;
};

// Launches the kernel (grid = min(num_tiles, #SMs) persistent CTAs).  Returns cudaError_t as int.
int launch_gemm(const GemmParams& p, bool a_mn_major, bool b_mn_major, cudaStream_t stream);

// Encodes a bf16 tiled tensor map with 128-byte swizzle and zero OOB fill.  dims/box in elements, strides in bytes
// (strides[i] is the byte stride of dimension i+1).  Returns 0 on success.
int encode_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                     const uint32_t* box, const uint32_t* elem_strides);

}  // namespace t2v
