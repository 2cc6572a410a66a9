// Persistent warp-specialised wgmma GEMM for sm_90a.  See gemm_tc.cuh for the operand model.
//
//   warps 0-7   : two MMA warpgroups.  Warpgroup g runs wgmma on rows 64g..64g+63 of the 128-row tile (fp32 accumulator in
//                 registers), then hands the finished accumulator to the epilogue through shared memory.
//   warp 8      : TMA producer (one elected lane of warpgroup 2) - fills the smem ring, one mbarrier pair per stage
//   warps 12-15 : the epilogue warpgroup.  Thread <-> output row (warp w owns rows 32w..32w+31 and every column chunk);
//                 smem-staged coalesced global stores / red.add.
//
// The accumulator tile in shared memory is handed over with two mbarriers: acc_full (MMA -> epilogue) and acc_empty
// (epilogue -> MMA, arrived once the epilogue has read the last accumulator chunk, before that chunk's global stores).  So
// the MMA warpgroups start the next tile's main loop while the epilogue of the previous one is still running.
#include "common.h"
#include "gemm_tc.cuh"
#include "ptx.cuh"

#include <cstdio>
#include <mutex>
#include <type_traits>

namespace t2v {

struct TileVars {
    int32_t t[6];
};

// tile id -> six mixed-radix digits, with host-precomputed magic numbers (q = umulhi(n, mul) >> shr; n < 2^31)
__device__ __forceinline__ void decompose_tile(const GemmParams& p, int32_t tile, TileVars& tv) {
    uint32_t n = static_cast<uint32_t>(tile);
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        const uint32_t d = static_cast<uint32_t>(p.tdim[i]);
        const uint32_t q = d == 1u ? n : (__umulhi(n, p.tdiv_mul[i]) >> p.tdiv_shr[i]);
        tv.t[i] = static_cast<int32_t>(n - q * d);
        n = q;
    }
}

__device__ __forceinline__ void k_range(const GemmParams& p, const TileVars& tv, int32_t& kb0, int32_t& kb1) {
    if (p.ksplit_var >= 0) {
        int32_t sv = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i) sv |= tv.t[i] & -static_cast<int32_t>(i == p.ksplit_var);   // (a select chain would be
                                                                                                 // lowered to an indexed local array)
        kb0 = sv * p.kb_per_split;
        kb1 = min(p.kb_total, kb0 + p.kb_per_split);
    } else {
        kb0 = 0;
        kb1 = p.kb_total;
    }
}

// TMA coordinates of one operand at (tile, k-loop digits kv)
__device__ __forceinline__ void operand_coords(const TmaOperand& op, const TileVars& tv, const int32_t* kv, int32_t* c) {
#pragma unroll
    for (int d = 0; d < 5; ++d) {
        int32_t v = op.base[d];
#pragma unroll
        for (int i = 0; i < 6; ++i) v += tv.t[i] * op.tcoef[d][i];
        v += kv[0] * op.kcoef[d][0] + kv[1] * op.kcoef[d][1] + kv[2] * op.kcoef[d][2];
        c[d] = v;
    }
}

__device__ __forceinline__ void issue_boxes(const TmaOperand& op, const int32_t* c_in, uint8_t* smem_dst, uint64_t* bar) {
    int32_t c[5] = {c_in[0], c_in[1], c_in[2], c_in[3], c_in[4]};
    for (int b = 0; b < op.nbox; ++b) {  // boxes of an MN-major operand always advance along dimension 0
        tma_load(op.rank, smem_dst + b * op.box_bytes, &op.map, bar, c);
        c[0] += op.box_step;
    }
}

// The accumulator tile in shared memory: row r at acc_s + r * pitch * 4 bytes, its 16-byte chunk c stored at chunk c ^ acc_swz(r).
// Conflict-free both for the wgmma fragment stores (8 bytes per lane, rows r..r+3 per half-warp) and for the row reads of the
// epilogue (16 bytes per lane, 8 consecutive rows per quarter-warp).
__device__ __forceinline__ uint32_t acc_swz(uint32_t r) { return ((r & 3u) << 1) | ((r >> 2) & 1u); }
// 32 fp32 columns (chunk ch) of one accumulator row
__device__ __forceinline__ void acc_ld32(uint32_t arow, uint32_t key, int ch, uint32_t* r) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 q = lds128(arow + ((static_cast<uint32_t>(ch * 8 + j) ^ key) << 4));
        r[4 * j] = q.x; r[4 * j + 1] = q.y; r[4 * j + 2] = q.z; r[4 * j + 3] = q.w;
    }
}

// flags of the epilogue's chunk body: known at compile time (folded away) or only at run time (the catch-all instantiation)
template <bool V>
struct ConstFlag {
    __device__ constexpr operator bool() const { return V; }
};
struct RuntimeFlag {
    bool v;
    __device__ constexpr operator bool() const { return v; }
};

// Epilogue of one tile (epilogue warp w = 0..3).  Warp w owns accumulator rows 32w..32w+31, i.e. thread <-> output row, and
// all of the tile's column chunks.  Output rows are strided in global memory, so every 32-column chunk goes through a per-warp
// swizzled staging tile and is moved with 16 bytes per lane covering whole rows (full 64/128-byte segments); the residual
// comes in the same way.  The per-column bias is fetched with one coalesced load per chunk and broadcast through shared
// memory.  Buffers that are not 16-byte aligned (EPI_VEC clear) take a per-thread scalar path.
// The accumulator tile is read after acc_full completes phase acc_phase; every thread arrives on acc_empty once it has read
// its last accumulator chunk (and row sum).  rowsum_tile: rs_s holds the row sums of operand A for this tile (EPI_ROWSUM_A).
template <int ESZ>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const TileVars& tv, bool rowsum_tile, uint32_t warp, uint32_t lane,
                                              uint32_t acc_s, uint32_t acc_pitch, uint32_t rs_s, uint8_t* stg_base,
                                              uint64_t* acc_full, uint64_t* acc_empty, uint32_t acc_phase) {
    constexpr int CPR = ESZ * 2;        // 16-byte chunks per 32-column row: 4 (bf16) or 8 (fp32)
    constexpr int EPC = 16 / ESZ;       // elements per 16-byte chunk
    constexpr int RPI = 32 / CPR;       // rows covered by one warp-wide 16-byte access
    const uint32_t row = warp * 32u + lane;
    const int32_t rw = static_cast<int32_t>(row) % p.bw;
    const int32_t rh = (static_cast<int32_t>(row) / p.bw) % p.bh;
    const int32_t rn = static_cast<int32_t>(row) / (p.bw * p.bh);
    const bool has_bias = p.flags & EPI_BIAS, has_rb = p.flags & EPI_ROWBIAS, has_res = p.flags & EPI_RESIDUAL;
    const bool vec = p.flags & EPI_VEC;
    const bool has_stats = ESZ == 2 && (p.flags & EPI_STATS) && vec;
    const int32_t col0 = tv.t[0] * p.block_n;
    // the tile's 32-column chunks, without the chunks past the output's last column
    const int c_end = min((p.block_n + 31) >> 5, (p.ncols - col0 + 31) >> 5);
    const uint32_t stg_s = smem_u32(stg_base + warp * 4096u);                   // 32 rows x <= 128 B
    float* sbias = reinterpret_cast<float*>(stg_base + 4 * 4096u) + warp * 32;  // 32 floats per warp
    // swizzled byte offset of logical 16-byte chunk j of row r in a dense [32][n] chunk array
    auto phys = [](int r, int j, int n) { return (r * n + (j ^ (((r * n) >> 3) & (n - 1)))) * 16; };
    const int sr = lane / CPR, sj = lane % CPR;  // (row-in-group, chunk) this lane moves in the coalesced phases
    // Tile-invariant shared-memory addresses of the staging tile.  stg_s is 256-byte aligned and a staged row is CPR (or 4)
    // chunks, so each family of addresses is one base register and a compile-time XOR or offset: rows 512 bytes apart share
    // the swizzle key (up to bit 2 with 8 chunks a row), and the chunk index sits in the bits a row base leaves clear.
    const uint32_t w_own0 = stg_s + phys(static_cast<int>(lane), 0, CPR);
    const uint32_t r_mov0 = stg_s + phys(sr, sj, CPR);
    const uint32_t w_res0 = stg_s + phys(static_cast<int>(lane >> 2), static_cast<int>(lane & 3), 4);
    const uint32_t r_res0 = stg_s + phys(static_cast<int>(lane), 0, 4);
    // this lane's own row, 16-byte chunk j (write after the math)
    auto w_own = [&](int j) { return w_own0 ^ (static_cast<uint32_t>(j) << 4); };
    // the (row sr + RPI j, chunk sj) this lane moves in the coalesced store (read); with 8 chunks a row, odd j flips key bit 2
    auto r_mov = [&](int j) { return (r_mov0 ^ (CPR == 8 ? static_cast<uint32_t>(j & 1) << 6 : 0u)) + 512u * j; };
    // residual staging (bf16 rows of 64 B): write row (lane / 4) + 8 j, chunk lane % 4; read own row, chunk j
    auto w_res = [&](int j) { return w_res0 + 512u * j; };
    auto r_res = [&](int j) { return r_res0 ^ (static_cast<uint32_t>(j) << 4); };
    const bool alpha_one = p.alpha == 1.0f;
    const int32_t gw = tv.t[1] * p.bw + rw, gh = tv.t[2] * p.bh + rh, gn = tv.t[3] * p.bn + rn;
    const bool row_ok = (rn < p.bn) && gw < p.W && gh < p.H && gn < p.N;
    int64_t off = gw * p.ldw + gh * p.ldh + gn * p.ldn;
#pragma unroll
    for (int i = 0; i < 6; ++i) off += tv.t[i] * p.otc[i];
    // rows this lane moves in the coalesced phases (constant over the tile's chunks)
    int64_t off_s[CPR];
    uint32_t ok_s = 0;
#pragma unroll
    for (int i = 0; i < CPR; ++i) {
        const int r = sr + RPI * i;
        off_s[i] = __shfl_sync(0xffffffffu, off, r);
        ok_s |= (__shfl_sync(0xffffffffu, row_ok ? 1u : 0u, r) & 1u) << i;
    }
    // every row of this warp inside the output: full chunks run without per-row predicates
    const bool all_rows = vec && __all_sync(0xffffffffu, row_ok);
    // GroupNorm statistics: frame of this lane's segment (taken from the segment's first row, which is in bounds
    // whenever any row of the segment is)
    int64_t st_off = 0;
    uint32_t okmask = 0;
    if (has_stats) {
        const int32_t fr = (gw * p.st_cw + gh * p.st_ch + gn * p.st_cn) / p.st_div;
        st_off = int64_t(__shfl_sync(0xffffffffu, fr, lane & ~uint32_t(p.st_seg - 1))) * p.st_ld;
        okmask = __ballot_sync(0xffffffffu, row_ok);
    }
    // ---- software pipeline of the epilogue's global loads.  Per-column additive terms (bias, and the time-embedding row
    // when every row of this warp takes the same one) are fetched two chunks ahead, the residual tile one chunk ahead;
    // the first of them are issued BEFORE the wait for the accumulator, so their latency hides behind the main loop.
    // (every lane takes part in the shuffle: it must not sit behind a short-circuit that depends on row_ok)
    // The row is taken from the warp's first IN-BOUNDS lane: an out-of-bounds lane (frames beyond N in the last tile) would
    // name a row past the end of the time-embedding matrix.  A warp without any valid row folds nothing.
    const int32_t rb_row = has_rb ? gn / p.rb_div : 0;
    const uint32_t ok_lanes = __ballot_sync(0xffffffffu, row_ok);
    const int32_t rb_first = __shfl_sync(0xffffffffu, rb_row, ok_lanes ? __ffs(ok_lanes) - 1 : 0);
    const bool rb_same = !row_ok || rb_row == rb_first;
    const bool rb_uniform = has_rb && vec && ok_lanes != 0u && __all_sync(0xffffffffu, rb_same);
    const float* rb_base = has_rb ? p.rowbias + static_cast<int64_t>(rb_first) * p.rb_ld : nullptr;
    const bool colterm = has_bias || rb_uniform;   // a per-column term, broadcast through sbias
    const bool row_rb = has_rb && !rb_uniform;     // a time-embedding row per output row
    auto load_colterm = [&](int ch) {
        const int32_t c = col0 + ch * 32 + static_cast<int32_t>(lane);
        float b = 0.f;
        if (static_cast<int32_t>(lane) < min(32, min(p.block_n - ch * 32, p.ncols - (col0 + ch * 32)))) {
            if (has_bias) b = __ldg(p.bias + c);
            if (rb_uniform) b += __ldg(rb_base + c);
        }
        return b;
    };
    // The residual is prefetched only when every row is in bounds, and only for a full-width chunk: only a full chunk uses it
    const bool res_pref = all_rows && has_res;
    const __nv_bfloat16* res_lane = static_cast<const __nv_bfloat16*>(p.residual) + (lane & 3) * 8;
    int64_t off_q[4];   // residual rows this lane fetches: (lane / 4) + 8 i - for bf16 output the rows of off_s
#pragma unroll
    for (int i = 0; i < 4; ++i) off_q[i] = ESZ == 2 ? off_s[i] : __shfl_sync(0xffffffffu, off, (lane >> 2) + 8 * i);
    auto load_res = [&](int ch, uint4 (&q)[4]) {
        const int32_t c = col0 + ch * 32;
        if (min(p.block_n - ch * 32, p.ncols - c) >= 32) {
#pragma unroll
            for (int i = 0; i < 4; ++i) q[i] = __ldg(reinterpret_cast<const uint4*>(res_lane + off_q[i] + c));
        }
    };
    float bq0 = 0.f, bq1 = 0.f;
    uint4 rq[4] = {};
    if (c_end > 0) bq0 = load_colterm(0);
    if (c_end > 1) bq1 = load_colterm(1);
    if (res_pref && c_end > 0) load_res(0, rq);
    mbar_wait(acc_full, acc_phase);
    const uint32_t arow = acc_s + row * acc_pitch * 4u, akey = acc_swz(row);
    uint32_t acc[32];
    if (c_end > 0) acc_ld32(arow, akey, 0, acc);  // chunk ch+1 is read while chunk ch goes out to global memory
    // row sums of operand A (weight gradient: the bias gradient)
    if (rowsum_tile && row_ok) atomicAdd(p.rowsum + gw, __uint_as_float(lds32(rs_s + row * 4u)));
    if (c_end <= 1) mbar_arrive(acc_empty);   // (with more chunks: once the last one has been read, in its predecessor's body)
    for (int ch = 0; ch < c_end; ++ch) {
        const int32_t col = col0 + ch * 32;
        const int32_t cvalid = min(32, min(p.block_n - ch * 32, p.ncols - col));  // valid columns of this chunk, >= 1
        __syncwarp();
        const float bcur = bq0;          // this chunk's per-column term; keep the pipeline two chunks deep
        bq0 = bq1;
        if (ch + 2 < c_end) bq1 = load_colterm(ch + 2);
        if (!vec) {
            // unaligned buffers: each thread writes its own row, element by element
            if (row_ok) {
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    if (j >= cvalid) break;
                    float x = __uint_as_float(acc[j]) * p.alpha;
                    if (has_bias) x += p.bias[col + j];
                    if (has_rb) x += p.rowbias[(gn / p.rb_div) * p.rb_ld + col + j];
                    if (has_res) x += __bfloat162float(static_cast<const __nv_bfloat16*>(p.residual)[off + col + j]);
                    if (ESZ == 2) static_cast<__nv_bfloat16*>(p.out)[off + col + j] = __float2bfloat16_rn(x);
                    else if (p.out_mode == OUT_F32) static_cast<float*>(p.out)[off + col + j] = x;
                    else atomicAdd(static_cast<float*>(p.out) + off + col + j, x);
                }
            }
            if (ch + 1 < c_end) acc_ld32(arow, akey, ch + 1, acc);
            if (ch + 2 == c_end) mbar_arrive(acc_empty);
            continue;
        }
        // ---- one chunk: alpha, column term, per-row time embedding, residual, packing, statistics, coalesced store.  The
        // body is instantiated per combination of (full chunk, column term, residual, statistics, alpha, per-row time
        // embedding) so that the common full chunks run straight-line code without flag tests (in a flag-driven version a
        // third of the instructions per chunk were predicate bookkeeping).  A full chunk is 32 x 32 with every row of the
        // warp in bounds; any other chunk applies the row and column predicates.
        auto body = [&](auto kFull, auto kCol, auto kRes, auto kStats, auto kAlpha, auto kRowRb) {
            // each flag is a ConstFlag (folded at compile time) or a RuntimeFlag (the catch-all instantiation)
            const bool FULL = kFull, COL = kCol, RES = kRes, STATS = kStats, ALPHA = kAlpha, ROWRB = kRowRb;
            if (COL) sbias[lane] = bcur;
            if (RES) {   // residual -> staging: a full chunk's was prefetched one chunk ago, any other is loaded here
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    uint4 q = rq[i];
                    if (!FULL) {
                        const bool ok_r = __shfl_sync(0xffffffffu, row_ok ? 1 : 0, (lane >> 2) + 8 * i);
                        q = make_uint4(0, 0, 0, 0);
                        if (ok_r && (lane & 3) * 8 + 8 <= cvalid) q = __ldg(reinterpret_cast<const uint4*>(res_lane + off_q[i] + col));
                    }
                    sts128(w_res(i), q);
                }
                if ((FULL || res_pref) && ch + 1 < c_end) load_res(ch + 1, rq);
            }
            float* v = reinterpret_cast<float*>(acc);   // in place: the accumulator registers are not reloaded until the
            if (ALPHA) {                                  // values have been packed into the staging tile
#pragma unroll
                for (int j = 0; j < 32; ++j) v[j] *= p.alpha;
            }
            if (COL || RES) __syncwarp();
            if (COL) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float4 b = *reinterpret_cast<const float4*>(sbias + 4 * j);  // shared-memory broadcast
                    v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
                }
            }
            if (ROWRB && (FULL || row_ok)) {
                const float4* b4 = reinterpret_cast<const float4*>(p.rowbias + (gn / p.rb_div) * p.rb_ld + col);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (FULL || j * 4 + 4 <= cvalid) {
                        const float4 b = __ldg(b4 + j);
                        v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
                    }
                }
            }
            if (RES) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint4 q = lds128(r_res(j));
                    v[8 * j + 0] += bf16_lo(q.x); v[8 * j + 1] += bf16_hi(q.x);
                    v[8 * j + 2] += bf16_lo(q.y); v[8 * j + 3] += bf16_hi(q.y);
                    v[8 * j + 4] += bf16_lo(q.z); v[8 * j + 5] += bf16_hi(q.z);
                    v[8 * j + 6] += bf16_lo(q.w); v[8 * j + 7] += bf16_hi(q.w);
                }
                __syncwarp();
            }
            // own row -> staging
            if constexpr (ESZ == 2) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    uint4 q;
                    q.x = pack_bf16(v[8 * j + 0], v[8 * j + 1]);
                    q.y = pack_bf16(v[8 * j + 2], v[8 * j + 3]);
                    q.z = pack_bf16(v[8 * j + 4], v[8 * j + 5]);
                    q.w = pack_bf16(v[8 * j + 6], v[8 * j + 7]);
                    sts128(w_own(j), q);
                }
            } else {
#pragma unroll
                for (int j = 0; j < CPR; ++j) sts128(w_own(j), make_uint4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]));
            }
            if (ch + 1 < c_end) acc_ld32(arow, akey, ch + 1, acc);   // next chunk
            if (ch + 2 == c_end) mbar_arrive(acc_empty);             // ... the last one: the MMA warps may overwrite the tile
            __syncwarp();
            if (ESZ == 2 && STATS) {
                // GroupNorm statistics of the tile just staged (the bf16 values the consumer will read): lanes 0-15 walk
                // rows 0-15, lanes 16-31 rows 16-31 (staggered by one row so the two halves hit different banks), each lane
                // owns the column pair (2c, 2c+1), c = lane % 16.  16-row segments: every half is one frame; 32-row
                // segments: the halves are combined with one shuffle.
                const uint32_t half = lane >> 4, cw = lane & 15u;
                float s0 = 0.f, q0 = 0.f, s1 = 0.f, q1 = 0.f;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int r = half ? 16 + ((i + 1) & 15) : i;
                    const uint32_t w = lds32(stg_s + phys(r, int(cw >> 2), 4) + (cw & 3u) * 4u);
                    if (FULL || ((okmask >> r) & 1u)) {
                        const float lo = bf16_lo(w), hi = bf16_hi(w);
                        s0 += lo; q0 += lo * lo;
                        s1 += hi; q1 += hi * hi;
                    }
                }
                if (p.st_seg == 32) {
                    s0 += __shfl_xor_sync(0xffffffffu, s0, 16); q0 += __shfl_xor_sync(0xffffffffu, q0, 16);
                    s1 += __shfl_xor_sync(0xffffffffu, s1, 16); q1 += __shfl_xor_sync(0xffffffffu, q1, 16);
                }
                // a segment without a valid row has no frame (its offset is meaningless): it contributes nothing
                const bool any_row = FULL || (p.st_seg == 16 ? ((okmask >> (half * 16u)) & 0xFFFFu) != 0u : okmask != 0u);
                if (any_row && (p.st_seg == 16 || half == 0) && (FULL || int(2 * cw) < cvalid))
                    red_add_f32x4(p.stats + (st_off + col + 2 * cw) * 2, s0, q0, s1, q1);
            }
            // staging -> global: 16 bytes per lane, whole row segments
            const int nval = cvalid - sj * EPC;  // valid elements in this lane's 16-byte chunk
            char* ob = static_cast<char*>(p.out) + (static_cast<int64_t>(col) + sj * EPC) * ESZ;
#pragma unroll
            for (int i = 0; i < CPR; ++i) {
                if (!FULL && (!((ok_s >> i) & 1u) || nval <= 0)) continue;
                const uint4 q = lds128(r_mov(i));
                char* o = ob + off_s[i] * ESZ;
                if (FULL || nval >= EPC) {
                    if (ESZ == 2 || p.out_mode == OUT_F32) {
                        *reinterpret_cast<uint4*>(o) = q;
                    } else {
                        red_add_f32x4(reinterpret_cast<float*>(o), __uint_as_float(q.x), __uint_as_float(q.y), __uint_as_float(q.z),
                                      __uint_as_float(q.w));
                    }
                } else {  // ragged last chunk: element-wise
                    // (static indexing only: a runtime-indexed register array would be demoted to local memory)
                    const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                    for (int e = 0; e < EPC; ++e) {
                        if (e >= nval) break;
                        if (ESZ == 2) reinterpret_cast<uint16_t*>(o)[e] = static_cast<uint16_t>((w4[e >> 1] >> ((e & 1) * 16)) & 0xFFFFu);
                        else if (p.out_mode == OUT_F32) reinterpret_cast<float*>(o)[e] = __uint_as_float(w4[e & 3]);
                        else atomicAdd(reinterpret_cast<float*>(o) + e, __uint_as_float(w4[e & 3]));
                    }
                }
            }
        };
        using T = ConstFlag<true>;
        using F = ConstFlag<false>;
        const bool full = all_rows && cvalid == 32;
        const int key = full && alpha_one && !row_rb ? (colterm ? 1 : 0) | (has_res ? 2 : 0) | (has_stats ? 4 : 0) : 8;
        switch (key) {
            case 0: body(T{}, F{}, F{}, F{}, F{}, F{}); break;     // plain (dgrad, attention products)
            case 1: body(T{}, T{}, F{}, F{}, F{}, F{}); break;     // bias (+ folded time embedding)
            case 2: body(T{}, F{}, T{}, F{}, F{}, F{}); break;     // residual
            case 3: body(T{}, T{}, T{}, F{}, F{}, F{}); break;     // bias + residual
            case 4: body(T{}, F{}, F{}, T{}, F{}, F{}); break;     // ... the same with GroupNorm statistics
            case 5: body(T{}, T{}, F{}, T{}, F{}, F{}); break;
            case 6: body(T{}, F{}, T{}, T{}, F{}, F{}); break;
            case 7: body(T{}, T{}, T{}, T{}, F{}, F{}); break;
            default: {                                              // alpha != 1 / per-row time embedding / ragged chunk
                using R = RuntimeFlag;
                body(R{full}, R{colterm}, R{has_res}, R{has_stats}, R{!alpha_one}, R{row_rb});
                break;
            }
        }
    }
}

// One 64 x BN x 16 step of a consumer warpgroup.
template <int BN, int TA, int TB>
__device__ __forceinline__ void mma_step(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    if constexpr (BN == 16) wgmma_n16<TA, TB>(d, da, db, acc);
    else if constexpr (BN == 32) wgmma_n32<TA, TB>(d, da, db, acc);
    else if constexpr (BN == 48) wgmma_n48<TA, TB>(d, da, db, acc);
    else if constexpr (BN == 64) wgmma_n64<TA, TB>(d, da, db, acc);
    else if constexpr (BN == 80) wgmma_n80<TA, TB>(d, da, db, acc);
    else if constexpr (BN == 96) wgmma_n96<TA, TB>(d, da, db, acc);
    else if constexpr (BN == 112) wgmma_n112<TA, TB>(d, da, db, acc);
    else wgmma_n128<TA, TB>(d, da, db, acc);
}

// Ring position of the consumer warpgroups
struct Ring {
    uint32_t stage, phase;
};

// Main loop of one tile for one consumer warpgroup: k-blocks kb0..kb1 into d (and, ROWSUM, the row sums of A into drs).
// Compiled per wgmma N so that the MMAs of a k-block issue back to back.
template <bool A_MN, bool B_MN, int BN, bool ROWSUM>
__device__ __forceinline__ void mainloop(const GemmParams& p, int32_t kb0, int32_t kb1, Ring& ring, uint64_t* full_bar,
                                         uint64_t* empty_bar, uint32_t a_base, uint32_t b_base, uint64_t d_ones, bool release,
                                         float* d, float* drs) {
    constexpr int TA = A_MN ? 1 : 0, TB = B_MN ? 1 : 0;
    // descriptor advance per k = 16 step, in 16-byte units
    constexpr uint32_t a_kstep = A_MN ? (16u * 128u) >> 4 : 32u >> 4;
    constexpr uint32_t b_kstep = B_MN ? (16u * 128u) >> 4 : 32u >> 4;
    constexpr uint32_t a_lbo = A_MN ? 64u * 128u : 0u;
    constexpr uint32_t b_lbo = B_MN ? 64u * 128u : 0u;
    uint32_t prev_stage = 0;
    bool has_prev = false;
    for (int32_t kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[ring.stage], ring.phase);
        const uint64_t da = make_sw128_desc(a_base + ring.stage * static_cast<uint32_t>(p.stage_bytes_a), a_lbo, 1024);
        const uint64_t db = make_sw128_desc(b_base + ring.stage * static_cast<uint32_t>(p.stage_bytes_b), b_lbo, 1024);
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < kBlockK / 16; ++k) {
            const uint32_t accumulate = (kb > kb0 || k > 0) ? 1u : 0u;
            mma_step<BN, TA, TB>(d, da + k * a_kstep, db + k * b_kstep, accumulate);
            if constexpr (ROWSUM) wgmma_n16<TA, 0>(drs, da + k * a_kstep, d_ones, accumulate);
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have completed: its stage may be refilled
        if (has_prev && release) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = ring.stage;
        has_prev = true;
        if (++ring.stage == static_cast<uint32_t>(p.num_stages)) {
            ring.stage = 0;
            ring.phase ^= 1;
        }
    }
    wgmma_wait<0>();
    if (has_prev && release) mbar_arrive(&empty_bar[prev_stage]);
    wgmma_fence_regs(d, BN / 2);
    if constexpr (ROWSUM) wgmma_fence_regs(drs, 8);
}

template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kNumThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment is required by the 128-byte swizzle atoms.
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int S = p.num_stages;
    const bool rowsum_a = p.flags & EPI_ROWSUM_A;
    const uint8_t* ones_tile = smem;              // EPI_ROWSUM_A: 16 rows x 128 bytes of bf16 1.0 (any layout: all elements equal)
    if (rowsum_a) smem += kOnesTileBytes;
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + static_cast<size_t>(S) * p.stage_bytes_a;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + static_cast<size_t>(S) * p.stage_bytes_b);
    uint64_t* full_bar = bars;                       // [S]   TMA -> MMA
    uint64_t* empty_bar = bars + kMaxStages;         // [S]   MMA -> TMA
    uint64_t* acc_full = bars + 2 * kMaxStages;      // accumulator tile written (MMA -> epilogue)
    uint64_t* acc_empty = acc_full + 1;              // accumulator tile read (epilogue -> MMA)
    uint8_t* stg_base = reinterpret_cast<uint8_t*>(bars) + 256;               // epilogue staging tiles
    float* acc_f = reinterpret_cast<float*>(stg_base + kEpilogueStagingBytes);  // accumulator tile (acc_smem_bytes)
    const uint32_t acc_pitch = static_cast<uint32_t>((p.block_n + 31) / 32 * 32);
    const uint32_t acc_s = smem_u32(acc_f);
    float* rs_s = acc_f + kBlockM * acc_pitch;   // EPI_ROWSUM_A: row sums of the tile

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t lane = lane_id();
    const uint32_t wg = warp >> 2;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&p.a.map);
        tma_prefetch_desc(&p.b.map);
        for (int s = 0; s < S; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);   // one arrival per MMA warp
        }
        mbar_init(acc_full, 256);          // every MMA thread, after its fragment stores
        mbar_init(acc_empty, 128);         // every epilogue thread, after its last accumulator read
        fence_mbar_init();
    }
    if (rowsum_a && warp == 0) {   // the constant B operand of the row-sum MMAs; made visible to the tensor core (async proxy)
        const uint32_t one2 = 0x3F803F80u;         // two bf16 1.0
        uint4* o = reinterpret_cast<uint4*>(const_cast<uint8_t*>(ones_tile));
        for (uint32_t i = lane; i < kOnesTileBytes / 16; i += 32) o[i] = make_uint4(one2, one2, one2, one2);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    pdl_sync();  // the prologue above (barriers, descriptor prefetch) overlaps the tail of the previous kernel

    // Registers: 40 (producer) + 2 x 168 (MMA) + 136 (epilogue) per thread of each warpgroup = the whole 64 K register file
    if (wg == 2) {
        // ------------------------------------------------------------------ TMA producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && elect_one()) {
            uint32_t stage = 0, phase = 0;
            const uint32_t tx_bytes = p.stage_bytes_a + p.stage_bytes_b;
            for (int32_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                TileVars tv;
                decompose_tile(p, tile, tv);
                int32_t kb0, kb1;
                k_range(p, tv, kb0, kb1);
                // k-loop digits advance as a mixed-radix counter; coordinates are updated incrementally (adds only) and
                // recomputed from scratch only when the fastest digit wraps
                int32_t kv[3];
                kv[0] = kb0 % p.kdim[0];
                kv[1] = (kb0 / p.kdim[0]) % p.kdim[1];
                kv[2] = kb0 / (p.kdim[0] * p.kdim[1]);
                int32_t ca[5], cb[5];
                operand_coords(p.a, tv, kv, ca);
                operand_coords(p.b, tv, kv, cb);
                for (int32_t kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], tx_bytes);
                    issue_boxes(p.a, ca, smem_a + static_cast<size_t>(stage) * p.stage_bytes_a, &full_bar[stage]);
                    issue_boxes(p.b, cb, smem_b + static_cast<size_t>(stage) * p.stage_bytes_b, &full_bar[stage]);
                    if (++kv[0] < p.kdim[0]) {
#pragma unroll
                        for (int d = 0; d < 5; ++d) {
                            ca[d] += p.a.kcoef[d][0];
                            cb[d] += p.b.kcoef[d][0];
                        }
                    } else {
                        kv[0] = 0;
                        if (++kv[1] == p.kdim[1]) {
                            kv[1] = 0;
                            ++kv[2];
                        }
                        operand_coords(p.a, tv, kv, ca);
                        operand_coords(p.b, tv, kv, cb);
                    }
                    if (++stage == static_cast<uint32_t>(S)) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
    } else if (wg == 3) {
        // ------------------------------------------------------------------ epilogue warpgroup
        asm volatile("setmaxnreg.inc.sync.aligned.u32 136;");
        uint32_t acc_phase = 0;
        for (int32_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            TileVars tv;
            decompose_tile(p, tile, tv);
            const bool rowsum_tile = rowsum_a && tv.t[0] == 0 && tv.t[2] == 0 && tv.t[3] == 0;
            if (p.out_mode == OUT_BF16) epilogue_tile<2>(p, tv, rowsum_tile, warp & 3u, lane, acc_s, acc_pitch, smem_u32(rs_s), stg_base, acc_full, acc_empty, acc_phase);
            else epilogue_tile<4>(p, tv, rowsum_tile, warp & 3u, lane, acc_s, acc_pitch, smem_u32(rs_s), stg_base, acc_full, acc_empty, acc_phase);
            acc_phase ^= 1;
        }
    } else {
        // ------------------------------------------------------------------ MMA warpgroups
        asm volatile("setmaxnreg.inc.sync.aligned.u32 168;");
        // this warpgroup's 64 rows of A: K-major, rows 64g.. (64 x 128 B further); MN-major, the g-th 64-wide box (8 KB)
        const uint32_t a_wg_off = wg * 8192u;
        // EPI_ROWSUM_A: D[64 x 16] += A_tile * ones: the same A descriptor against a K-major tile of ones (never advanced
        // along K - every element is 1.0)
        const uint64_t d_ones = make_sw128_desc(smem_u32(ones_tile), 0u, 1024);
        const bool release = lane == 0;
        const uint32_t a_base = smem_u32(smem_a) + a_wg_off, b_base = smem_u32(smem_b);
        Ring ring{0, 0};
        uint32_t acc_phase = 0;
        for (int32_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            float d[kMaxBlockN / 2];
            float drs[8];
            TileVars tv;
            decompose_tile(p, tile, tv);
            int32_t kb0, kb1;
            k_range(p, tv, kb0, kb1);
            const bool rowsum_tile = rowsum_a && tv.t[0] == 0 && tv.t[2] == 0 && tv.t[3] == 0;
            auto run = [&](auto bn) {
                constexpr int BN = decltype(bn)::value;
                if (rowsum_tile) mainloop<A_MN, B_MN, BN, true>(p, kb0, kb1, ring, full_bar, empty_bar, a_base, b_base, d_ones, release, d, drs);
                else mainloop<A_MN, B_MN, BN, false>(p, kb0, kb1, ring, full_bar, empty_bar, a_base, b_base, d_ones, release, d, drs);
            };
            switch (p.block_n) {   // the launch checked: a multiple of 16, at most kMaxBlockN
                case 16: run(std::integral_constant<int, 16>{}); break;
                case 32: run(std::integral_constant<int, 32>{}); break;
                case 48: run(std::integral_constant<int, 48>{}); break;
                case 64: run(std::integral_constant<int, 64>{}); break;
                case 80: run(std::integral_constant<int, 80>{}); break;
                case 96: run(std::integral_constant<int, 96>{}); break;
                case 112: run(std::integral_constant<int, 112>{}); break;
                default: run(std::integral_constant<int, 128>{}); break;
            }
            // accumulator -> shared memory.  Fragment of m64nNk16: d[4j + 2h + e] is row 16 * (warp % 4) + lane / 4 + 8h,
            // column 8j + 2 * (lane % 4) + e.
            mbar_wait(acc_empty, acc_phase ^ 1);   // the epilogue has read the previous tile (the first wait passes at once)
            {
                const uint32_t r0 = wg * 64u + (warp & 3u) * 16u + (lane >> 2);
                const uint32_t key = acc_swz(r0);   // == acc_swz(r0 + 8)
#pragma unroll
                for (int j = 0; j < kMaxBlockN / 8; ++j) {
                    if (8 * j >= p.block_n) break;
                    const uint32_t c = 8u * j + 2u * (lane & 3u);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t r = r0 + 8u * h;
                        const uint32_t addr = acc_s + (r * acc_pitch + (((c >> 2) ^ key) << 2) + (c & 3u)) * 4u;
                        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(d[4 * j + 2 * h]), "f"(d[4 * j + 2 * h + 1]) : "memory");
                    }
                }
                if (rowsum_tile && (lane & 3u) == 0) {
                    rs_s[r0] = drs[0];
                    rs_s[r0 + 8] = drs[2];
                }
            }
            mbar_arrive(acc_full);
            acc_phase ^= 1;
        }
    }
}

// ---------------------------------------------------------------------------------------------- host side

static int g_sm_count = 0;
int device_sm_count() {
    if (g_sm_count == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
        if (g_sm_count <= 0) g_sm_count = 132;
    }
    return g_sm_count;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    });
    return fn;
}

int encode_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                     const uint32_t* box, const uint32_t* elem_strides) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return -1;
    // cuTensorMapEncodeTiled is a driver-API call: it needs a context bound to the calling thread.  Autograd worker
    // threads may reach this point before any runtime-API call has bound the primary context, so bind it once.
    static thread_local bool ctx_bound = false;
    if (!ctx_bound) {
        cudaFree(nullptr);
        ctx_bound = true;
    }
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bdim[i] = box[i];
        estr[i] = elem_strides ? elem_strides[i] : 1;
    }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides[i];
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                    gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 1000;
}

template <bool A_MN, bool B_MN>
static int launch_impl(const GemmParams& p, cudaStream_t stream) {
    static std::once_flag attr_once;   // forward runs on the Python thread, backward on autograd worker threads
    static cudaError_t attr_err = cudaSuccess;
    const size_t smem = static_cast<size_t>(p.num_stages) * (p.stage_bytes_a + p.stage_bytes_b) + gemm_fixed_smem_bytes(p.block_n) +
                        ((p.flags & EPI_ROWSUM_A) ? kOnesTileBytes : 0);
    auto kern = gemm_tc_kernel<A_MN, B_MN>;
    std::call_once(attr_once, [&] { attr_err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmemBytes); });
    if (attr_err != cudaSuccess) return static_cast<int>(attr_err);
    if (p.block_n < 16 || p.block_n > kMaxBlockN || p.block_n % 16 || smem > static_cast<size_t>(kMaxSmemBytes))
        return static_cast<int>(cudaErrorInvalidValue);
    int grid = p.num_tiles < device_sm_count() ? p.num_tiles : device_sm_count();
    if (grid < 1) return 0;
    return static_cast<int>(launch_pdl(kern, dim3(grid), dim3(kNumThreads), smem, stream, p));
}

int launch_gemm(const GemmParams& p, bool a_mn, bool b_mn, cudaStream_t stream) {
    if (!a_mn && !b_mn) return launch_impl<false, false>(p, stream);
    if (!a_mn && b_mn) return launch_impl<false, true>(p, stream);
    if (a_mn && b_mn) return launch_impl<true, true>(p, stream);
    return launch_impl<true, false>(p, stream);
}

}  // namespace t2v
