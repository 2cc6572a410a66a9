// Host side of the affine TMA GEMM (gemm_tc.cuh) behind the C ABI of include/t2v_b200.h.  plan() turns a problem shape, the
// requested options, the SM count and the overrides into the shape-only GemmParams of each launch, without pointers or CUDA
// calls (t2v_gemm_plan exports it; tests/golden/gemm_plans.json pins it).  t2v_conv_* / t2v_bgemm plan, encode the tensor
// maps and epilogue pointers, and launch.
#include "common.h"
#include "gemm_tc.cuh"

#include "ptx.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <cuda_bf16.h>

using namespace t2v;

namespace t2v {
int launch_channel_stats(const void* x, float* stats, int S, int64_t P, int C, int64_t ld, cudaStream_t st);  // norms.cu
}

namespace {

struct Box3 {
    int w, h, n;
};

// Factor `prod` (a power of two) into (w,h,n) box extents over a (W,H,N) pixel space, maximising useful coverage.
Box3 choose_pixel_box(int prod, int W, int H, int N) {
    Box3 best{prod, 1, 1};
    double best_eff = -1.0;
    for (int bw = prod; bw >= 1; bw >>= 1) {
        for (int bh = prod / bw; bh >= 1; bh >>= 1) {
            const int bn = prod / (bw * bh);
            if (bw > 256 || bh > 256 || bn > 256) continue;
            const double cover = double((W + bw - 1) / bw) * bw * double((H + bh - 1) / bh) * bh * double((N + bn - 1) / bn) * bn;
            const double eff = double(W) * H * N / cover;
            if (eff > best_eff + 1e-9) {
                best_eff = eff;
                best = Box3{bw, bh, bn};
            }
        }
    }
    return best;
}

// Planner overrides: sweep hooks, test cases, A/B switches.  Read on every plan (the sweeps change them between calls).
struct Overrides {
    int bn;          // T2V_FORCE_BN: only this wgmma N
    int splits;      // T2V_FORCE_SPLITS: split factor of wgrad and of accumulating bgemm
    int fwd_splits;  // T2V_FORCE_FWD_SPLITS: split factor of fwd / dgrad problems that may split
    int stages;      // T2V_FORCE_STAGES: at most this many pipeline stages
    int no_split;    // T2V_NO_SPLIT: fwd / dgrad never split
    int no_rowsum;   // T2V_NO_ROWSUM_FUSE: the bias gradient of wgrad comes from a column-sum pass
};

Overrides read_overrides() {
    auto get = [](const char* name) { const char* v = std::getenv(name); return v ? std::atoi(v) : 0; };
    return Overrides{get("T2V_FORCE_BN"), get("T2V_FORCE_SPLITS"), get("T2V_FORCE_FWD_SPLITS"), get("T2V_FORCE_STAGES"),
                     get("T2V_NO_SPLIT"), get("T2V_NO_ROWSUM_FUSE")};
}

int b_stage_bytes(int bn, bool b_mn) { return b_mn ? ((bn + 63) / 64) * 8192 : bn * 128; }

// Shared memory the pipeline stages of an N = bn launch may use.  It still holds back the 16.5 KB of staging the epilogue
// needed before it moved into its own warpgroup of four warps: handing that space to the stages would change the stage
// count of most launches, a planner decision that tests/golden/gemm_plans.json pins and that a sweep of its own
// (tools/plan_sweep.py) has to justify.
constexpr int kStageBudgetHoldback = 4 * 4096 + 4 * 128;
int stage_budget(int bn, int smem_reserve) { return kMaxSmemBytes - gemm_fixed_smem_bytes(bn) - kStageBudgetHoldback - smem_reserve; }

// A (wgmma N, split-K factor) candidate as the cost models see it.
struct Cand {
    int bn, s, kper;       // N, split factor, k-blocks per split
    int stage_bytes;       // A + B bytes of one pipeline stage
    int64_t tiles, waves;  // work tiles (splits included) and waves of them over the SMs
    double active;         // CTAs busy in a full wave
};

// The one search over (N descending, split ascending); the first strictly cheaper candidate wins.  Skips an N that pads by a
// whole 16-column step or leaves fewer than 3 pipeline stages besides `smem_reserve`, and splits that repeat a smaller one's
// schedule; forced_s != 0 admits only that split.  row_tiles: tiles per N tile.  No candidate: N = 16, no split.
template <class MaxSplit, class Cost>
Cand search(int64_t row_tiles, int ncols, bool b_mn, int kblocks, int smem_reserve, int forced_bn, int forced_s, int sms,
            MaxSplit max_split, Cost cost) {
    Cand best{16, 1, kblocks, 0, 0, 0, 0.0};
    double best_cost = 1e30;
    for (int bn = kMaxBlockN; bn >= 16; bn -= 16) {
        if (forced_bn && bn != forced_bn) continue;
        if (bn > 16 && bn - 16 >= ncols) continue;
        const int stage_bytes = kBlockM * 128 + b_stage_bytes(bn, b_mn);
        if (stage_budget(bn, smem_reserve) / stage_bytes < 3) continue;
        const int64_t base = row_tiles * ((ncols + bn - 1) / bn);
        const int max_s = max_split(base);
        for (int s = 1; s <= max_s; ++s) {
            const int kper = (kblocks + s - 1) / s;
            if (forced_s ? s != forced_s : (kblocks + kper - 1) / kper != s) continue;
            const int64_t tiles = base * s;
            const Cand c{bn, s, kper, stage_bytes, tiles, (tiles + sms - 1) / sms, double(std::min<int64_t>(tiles, sms))};
            const double v = cost(c);
            if (v < best_cost - 1e-9) { best_cost = v; best = c; }
        }
    }
    return best;
}

// Cost models (clk) of one launch.  The bandwidth constants are estimates, not fitted on H100 (tools/plan_sweep.py and
// tools/gemm_sweep.py time the alternatives); split partials are red.added at ~2500 B/clk chip-wide.
constexpr double kRedBytesPerClk = 2500.0;
// fwd / dgrad, and the N of bgemm: per k-block the slowest of the tensor cores (128 x bn x 64 MACs at 2048 bf16 MACs/clk per
// SM: 4*bn clk), the chip-wide L2->SM bandwidth shared by the active CTAs and the per-SM shared-memory fill rate; per tile an
// epilogue that does not overlap the next tile's MMAs and a fixed overhead; a split adds red.add traffic, memset and finishing.
constexpr double kFwdL2BytesPerClk = 5200.0, kFwdFillBytesPerClk = 48.0, kFwdMinKBlockClk = 260.0, kFwdEpiClk = 450.0,
                 kFwdTileClk = 1800.0, kFwdSplitClk = 10000.0;
double fwd_cost(const Cand& c) {
    const double t_kb = std::max({4.0 * c.bn, c.stage_bytes * c.active / kFwdL2BytesPerClk, c.stage_bytes / kFwdFillBytesPerClk,
                                  kFwdMinKBlockClk});
    const double t_epi = (c.bn / 32.0 + 1.0) * kFwdEpiClk * 0.5;
    double cost = double(c.waves) * (c.kper * t_kb + t_epi + kFwdTileClk);
    if (c.s > 1) cost += double(c.tiles) * kBlockM * c.bn * 4.0 / kRedBytesPerClk + kFwdSplitClk;
    return cost;
}

// wgrad: MN-major operand boxes fill shared memory at ~40 B/clk per SM, the L2->SM ceiling is ~6000 B/clk, and every tile
// (no split included) is red.added into the fp32 gradient.
constexpr double kWgradL2BytesPerClk = 6000.0, kWgradFillBytesPerClk = 40.0, kWgradMinKBlockClk = 260.0, kWgradEpiClk = 500.0;
double wgrad_cost(const Cand& c) {
    const double t_kb = std::max({4.0 * c.bn, c.stage_bytes / kWgradFillBytesPerClk, c.stage_bytes * c.active / kWgradL2BytesPerClk,
                                  kWgradMinKBlockClk});
    const double t_epi = kWgradEpiClk + 4.0 * c.bn;
    const double red = double(c.tiles) * kBlockM * c.bn * 4.0 / kRedBytesPerClk;
    return double(c.waves) * (c.kper * t_kb + t_epi) + red;
}

// Split factor of an accumulating bgemm at its chosen N: waves * (k-blocks per split * T_kblock + T_epilogue).
constexpr double kAccKBlockClk = 320.0, kAccEpiClk = 2500.0;
double acc_split_cost(const Cand& c) { return double(c.waves) * (c.kper * kAccKBlockClk + kAccEpiClk); }

void finish_common(GemmParams& p, bool b_mn, int forced_stages, int smem_reserve) {
    p.stage_bytes_a = kBlockM * 128;
    p.stage_bytes_b = b_stage_bytes(p.block_n, b_mn);
    const int budget = stage_budget(p.block_n, smem_reserve);
    p.num_stages = std::min<int>(kMaxStages, budget / (p.stage_bytes_a + p.stage_bytes_b));
    if (forced_stages) p.num_stages = std::min(p.num_stages, forced_stages);
    int64_t tiles = 1;
    for (int i = 0; i < 6; ++i) tiles *= p.tdim[i];
    p.num_tiles = static_cast<int32_t>(tiles);
    for (int i = 0; i < 6; ++i) {  // q = umulhi(n, mul) >> shr for 0 <= n < 2^31 (CUTLASS FastDivmod construction)
        const uint32_t d = static_cast<uint32_t>(p.tdim[i]);
        if (d <= 1) {
            p.tdiv_mul[i] = 0;
            p.tdiv_shr[i] = 0;
            continue;
        }
        uint32_t lg = 0;
        while ((1ull << lg) < d) ++lg;
        const uint32_t pw = 31 + lg;
        p.tdiv_mul[i] = static_cast<uint32_t>(((1ull << pw) + d - 1) / d);
        p.tdiv_shr[i] = pw - 32;
    }
    p.kb_total = p.kdim[0] * p.kdim[1] * p.kdim[2];
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Epilogue pointers and options of the caller; keeps the epilogue work the planner chose in p.flags.
void fill_epilogue(GemmParams& p, const T2VEpilogue* e, void* out, int out_mode_default) {
    p.out = out;
    p.alpha = e ? e->alpha : 1.0f;
    p.bias = e ? e->bias : nullptr;
    p.rowbias = e ? e->rowbias : nullptr;
    p.residual = e ? e->residual : nullptr;
    p.out_mode = e ? (e->out_fp32 ? OUT_F32 : OUT_BF16) : out_mode_default;
    p.rb_div = (e && e->rowbias_div > 0) ? e->rowbias_div : 1;
    if (p.bias) p.flags |= EPI_BIAS;
    if (p.rowbias) p.flags |= EPI_ROWBIAS;
    if (p.residual) p.flags |= EPI_RESIDUAL;
}

// The shape half of EPI_VEC: every output stride is a whole number of 16-byte vectors.
bool vec_strides(const GemmParams& p) {
    const int64_t strides[] = {p.ldw, p.ldh, p.ldn, p.otc[0], p.otc[1], p.otc[2], p.otc[3], p.otc[4], p.otc[5], p.rb_ld};
    for (int64_t s : strides)
        if (s % 8) return false;
    return true;
}

void set_vec_flag(GemmParams& p) {
    const bool ok = aligned16(p.out) && (!p.residual || aligned16(p.residual)) && (!p.bias || aligned16(p.bias)) &&
                    (!p.rowbias || aligned16(p.rowbias)) && vec_strides(p);
    if (ok) p.flags |= EPI_VEC;
}

int check_channels(int c, const char* what) {
    if (c <= 0 || c % 8 != 0) return fail(-2, "%s=%d must be a positive multiple of 8 (16-byte TMA rows)", what, c);
    return 0;
}

// GroupNorm statistics in the epilogue (T2VEpilogue.stats): express "frame of an output row" in the tile's row coordinates
// and check that aligned runs of 32 (or 16) accumulator rows never straddle two frames.  Returns false when this tiling
// cannot do it (the caller then runs the standalone statistics pass over the finished output).
bool plan_epilogue_stats(GemmParams& p, int stats_rows, int Wo, int Ho, int N) {
    if (stats_rows <= 0) return false;
    const int64_t pf = stats_rows;        // output rows (flattened [N][Ho][Wo]) per statistics sample
    const int64_t frame = int64_t(Wo) * Ho;
    int cw = 0, ch = 0, cn = 0, div = 1;
    // does every aligned run of `seg` accumulator rows (tile row order: w fastest, then h, then n) share a sample?
    auto pick_seg = [&](auto&& ok) { return ok(32) ? 32 : (ok(16) ? 16 : 0); };
    int seg = 0;
    if (pf % frame == 0) {                // a sample is k whole images n (k = 1: per frame; k = F: per clip)
        const int64_t k = pf / frame, fp = int64_t(p.bw) * p.bh;
        cn = 1; div = int(k);
        seg = pick_seg([&](int sg) {
            if (fp % sg == 0) return true;                       // the run stays inside one image
            if (sg % fp) return false;
            const int64_t m = sg / fp;                           // the run covers m consecutive images of the tile
            return k % m == 0 && p.bn % m == 0;
        });
    } else if (pf % Wo == 0 && Ho % (pf / Wo) == 0) {   // a sample is k h-lines (temporal layout [B][F][HW]: h = frame index)
        const int64_t k = pf / Wo;
        ch = 1; cn = Ho; div = int(k);
        seg = pick_seg([&](int sg) {
            if (p.bw % sg == 0) return true;                     // the run stays inside one h-line
            if (sg % p.bw) return false;
            const int64_t m = sg / p.bw;                         // the run covers m consecutive h-lines of the tile
            return k % m == 0 && p.bh % m == 0;
        });
    } else if (Ho == 1 && N == 1 && Wo % pf == 0) {   // token matrix: sample = row / pf
        cw = 1; div = int(pf);
        seg = (p.bh == 1 && p.bn == 1) ? pick_seg([&](int sg) { return pf % sg == 0; }) : 0;
    }
    if (!seg) return false;
    p.st_cw = cw; p.st_ch = ch; p.st_cn = cn; p.st_div = div; p.st_seg = seg;
    p.flags |= EPI_STATS;
    return true;
}

struct Launch {             // one planned GEMM launch
    GemmParams p;           // shape-only fields; the entry point adds tensor maps and epilogue pointers
    int follow;             // T2V_FOLLOW_*: the pass that completes it
    int ph, pw, th0, tw0;   // dgrad: output parity class and its first contributing tap
    Box3 kbox;              // wgrad: the output pixels of one k-block
};

// Tile grid, N and split of a fwd / dgrad launch: (W, H, N) output pixels, `ncols` channels, (k0, k1, k2) k-blocks.
// Split-K serves few-tile problems (the 4x4 .. 16x16 UNet levels: 16-40 tiles of up to 180 k-blocks would idle most SMs): the
// k-range is split over tile variable 4, partials are red.added into an fp32 scratch image of the output, and launch_split's
// elementwise kernel applies alpha / bias / row bias / residual and writes the bf16 (or fp32) result.
void plan_pixels(Launch& l, int W, int H, int N, int ncols, bool b_mn, int k0, int k1, int k2, bool may_split, int sms,
                 const Overrides& ov) {
    GemmParams& p = l.p;
    const Box3 bx = choose_pixel_box(kBlockM, W, H, N);
    p.tdim[1] = (W + bx.w - 1) / bx.w;
    p.tdim[2] = (H + bx.h - 1) / bx.h;
    p.tdim[3] = (N + bx.n - 1) / bx.n;
    p.tdim[4] = p.tdim[5] = 1;
    p.kdim[0] = k0; p.kdim[1] = k1; p.kdim[2] = k2;
    p.ksplit_var = -1;
    const int kb = k0 * k1 * k2;
    const int forced_s = (may_split && ov.fwd_splits) ? std::min(ov.fwd_splits, kb) : 0;
    const Cand c = search(int64_t(p.tdim[1]) * p.tdim[2] * p.tdim[3], ncols, b_mn, kb, 0, ov.bn, forced_s, sms, [&](int64_t base) {
        return forced_s ? forced_s : ((may_split && base * 2 <= sms && kb >= 8) ? std::min(kb / 4, 64) : 1);
    }, fwd_cost);
    p.block_n = c.bn;
    p.tdim[0] = (ncols + p.block_n - 1) / p.block_n;
    if (c.s > 1) {
        p.kb_per_split = (kb + c.s - 1) / c.s;
        p.tdim[4] = (kb + p.kb_per_split - 1) / p.kb_per_split;
        p.ksplit_var = 4;
        l.follow = T2V_FOLLOW_SPLITK_FINISH;
    }
    finish_common(p, b_mn, ov.stages, 0);
    p.bw = bx.w; p.bh = bx.h; p.bn = bx.n;
    p.W = W; p.H = H; p.N = N; p.ncols = ncols;
}

int plan_conv_fwd(const T2VGemmProblem& q, int sms, const Overrides& ov, Launch* l) {
    const int N = q.N, H = q.H, W = q.W, Cin = q.Cin, Cout = q.Cout, KH = q.KH, KW = q.KW, stride = q.stride;
    if (int r = check_channels(Cin, "Cin")) return r;
    if (Cout <= 0 || N <= 0 || H <= 0 || W <= 0) return fail(-2, "conv_fwd: bad shape");
    if (stride != 1 && stride != 2) return fail(-2, "conv_fwd: stride %d unsupported", stride);
    const int Ho = (H + q.pad_h0 + q.pad_h1 - KH) / stride + 1, Wo = (W + q.pad_w0 + q.pad_w1 - KW) / stride + 1;
    if (Ho <= 0 || Wo <= 0) return fail(-2, "conv_fwd: empty output");
    std::memset(l, 0, sizeof(*l));
    plan_pixels(*l, Wo, Ho, N, Cout, false, (Cin + kBlockK - 1) / kBlockK, KW, KH, q.workspace && Cout % 8 == 0 && !ov.no_split, sms, ov);
    GemmParams& p = l->p;
    p.ldw = Cout; p.ldh = int64_t(Wo) * Cout; p.ldn = int64_t(Ho) * Wo * Cout;
    p.rb_ld = Cout;
    // statistics of a split problem come out of its finishing pass
    if (l->follow != T2V_FOLLOW_SPLITK_FINISH && q.stats_rows > 0 && !(vec_strides(p) && plan_epilogue_stats(p, q.stats_rows, Wo, Ho, N)))
        l->follow = T2V_FOLLOW_CHANNEL_STATS;   // this tiling cannot produce them in the epilogue
    return 1;
}

// One launch per output parity class (a single class when stride == 1).
int plan_conv_dgrad(const T2VGemmProblem& q, int sms, const Overrides& ov, Launch* l) {
    const int N = q.N, H = q.H, W = q.W, Cin = q.Cin, Cout = q.Cout, KH = q.KH, KW = q.KW, s = q.stride;
    if (int r = check_channels(Cin, "Cin")) return r;
    if (int r = check_channels(Cout, "Cout")) return r;
    if (s != 1 && s != 2) return fail(-2, "conv_dgrad: stride %d unsupported", s);
    int n = 0;
    for (int ph = 0; ph < s; ++ph) {
        for (int pw = 0; pw < s; ++pw) {
            const int Hc = (H - ph + s - 1) / s, Wc = (W - pw + s - 1) / s;  // outputs in this class
            if (Hc <= 0 || Wc <= 0) continue;
            const int th0 = (ph + q.pad_h0) % s, tw0 = (pw + q.pad_w0) % s;  // first contributing tap
            const int nth = th0 < KH ? (KH - th0 + s - 1) / s : 0, ntw = tw0 < KW ? (KW - tw0 + s - 1) / s : 0;
            if (nth == 0 || ntw == 0) return fail(-2, "conv_dgrad: parity class without taps is unsupported");
            Launch& L = l[n++];
            std::memset(&L, 0, sizeof(L));
            L.ph = ph; L.pw = pw; L.th0 = th0; L.tw0 = tw0;
            // split-K only for the single-class (stride 1) problem: the scratch image is the whole dx
            plan_pixels(L, Wc, Hc, N, Cin, true, (Cout + kBlockK - 1) / kBlockK, ntw, nth, s == 1 && q.workspace && !ov.no_split, sms, ov);
            L.p.ldw = int64_t(s) * Cin; L.p.ldh = int64_t(s) * W * Cin; L.p.ldn = int64_t(H) * W * Cin;
            L.p.rb_ld = Cin;
        }
    }
    return n;
}

// dbias: the bias gradient rides in the same launch (EPI_ROWSUM_A, gemm_tc.cuh); with T2V_NO_ROWSUM_FUSE a column-sum
// pass follows instead.
int plan_conv_wgrad(const T2VGemmProblem& q, int sms, const Overrides& ov, Launch* l) {
    const int N = q.N, H = q.H, W = q.W, Cin = q.Cin, Cout = q.Cout, KH = q.KH, KW = q.KW, stride = q.stride;
    if (int r = check_channels(Cin, "Cin")) return r;
    if (int r = check_channels(Cout, "Cout")) return r;
    if (stride != 1 && stride != 2) return fail(-2, "conv_wgrad: stride %d unsupported", stride);
    const int Ho = (H + q.pad_h0 + q.pad_h1 - KH) / stride + 1, Wo = (W + q.pad_w0 + q.pad_w1 - KW) / stride + 1;
    if (N <= 0 || Ho <= 0 || Wo <= 0) return fail(-2, "conv_wgrad: empty output");   // no k-blocks to split
    std::memset(l, 0, sizeof(*l));
    GemmParams& p = l->p;
    const Box3 kx = l->kbox = choose_pixel_box(kBlockK, Wo, Ho, N);  // 64 output pixels per k-block
    p.kdim[0] = (Wo + kx.w - 1) / kx.w;
    p.kdim[1] = (Ho + kx.h - 1) / kx.h;
    p.kdim[2] = (N + kx.n - 1) / kx.n;
    const int kb_total = p.kdim[0] * p.kdim[1] * p.kdim[2];
    p.tdim[1] = (Cout + kBlockM - 1) / kBlockM;
    p.tdim[2] = KW; p.tdim[3] = KH;
    // the fused bias gradient's 2 KB tile of ones is reserved for every candidate: the choice must not depend on dbias
    const int forced_s = ov.splits ? std::min(ov.splits, kb_total) : 0;
    const Cand c = search(int64_t(p.tdim[1]) * KH * KW, Cin, true, kb_total, kOnesTileBytes, ov.bn, forced_s, sms,
                          [&](int64_t) { return std::min(kb_total, 128); }, wgrad_cost);
    const bool fuse_rowsum = q.dbias && !ov.no_rowsum;
    p.block_n = c.bn;
    p.tdim[0] = (Cin + p.block_n - 1) / p.block_n;
    p.kb_per_split = (kb_total + c.s - 1) / c.s;
    p.tdim[4] = (kb_total + p.kb_per_split - 1) / p.kb_per_split;
    p.tdim[5] = 1;
    p.ksplit_var = 4;
    finish_common(p, true, ov.stages, fuse_rowsum ? kOnesTileBytes : 0);
    p.bw = kBlockM; p.bh = 1; p.bn = 1;
    p.W = Cout; p.H = KW; p.N = KH; p.ncols = Cin;
    p.ldw = int64_t(KH) * KW * Cin; p.ldh = Cin; p.ldn = int64_t(KW) * Cin;
    if (fuse_rowsum) p.flags |= EPI_ROWSUM_A;
    else if (q.dbias) l->follow = T2V_FOLLOW_COLSUM;
    return 1;
}

// Accumulating problems (out_mode OUT_F32_RED) choose N against max(2, k-blocks / 4), then their split factor.
int plan_bgemm(const T2VGemmProblem& q, int sms, const Overrides& ov, Launch* l) {
    const int M = q.gemm_m, N = q.gemm_n, K = q.gemm_k, Z1 = q.z1, Z2 = q.z2;
    if (M <= 0 || N <= 0 || K <= 0 || Z1 <= 0 || Z2 <= 0) return fail(-2, "bgemm: bad shape");
    const bool b_mn = !q.b_kmajor, acc = q.out_mode == OUT_F32_RED;
    std::memset(l, 0, sizeof(*l));
    GemmParams& p = l->p;
    p.kdim[0] = (K + kBlockK - 1) / kBlockK;
    p.kdim[1] = p.kdim[2] = 1;
    p.tdim[1] = (M + kBlockM - 1) / kBlockM;
    p.tdim[2] = p.tdim[3] = 1;
    p.tdim[4] = Z2; p.tdim[5] = Z1;
    const int kb = p.kdim[0];
    const int64_t row_tiles = int64_t(p.tdim[1]) * Z1 * Z2;
    const Cand c = search(row_tiles, N, b_mn, acc ? std::max(2, kb / 4) : kb, 0, ov.bn, 0, sms, [](int64_t) { return 1; }, fwd_cost);
    p.block_n = c.bn;
    p.tdim[0] = (N + p.block_n - 1) / p.block_n;
    p.ksplit_var = -1;
    int splits = 1;
    if (acc) {
        const int forced_s = ov.splits ? std::max(1, std::min(ov.splits, kb)) : 0;
        splits = search(row_tiles, N, b_mn, kb, 0, c.bn, forced_s, sms,
                        [&](int64_t) { return forced_s ? forced_s : std::min(kb, 128); }, acc_split_cost).s;
        p.kb_per_split = (kb + splits - 1) / splits;
        splits = (kb + p.kb_per_split - 1) / p.kb_per_split;
        p.tdim[2] = splits;
        p.ksplit_var = 2;
    }
    finish_common(p, b_mn, ov.stages, 0);
    p.bw = kBlockM; p.bh = 1; p.bn = 1;
    p.W = M; p.H = splits; p.N = 1; p.ncols = N;
    return 1;
}

// The launches of problem `q` on `sms` SMs (at most 4), or a negative error.
int plan(const T2VGemmProblem& q, int sms, const Overrides& ov, Launch* l) {
    static int (*const planners[])(const T2VGemmProblem&, int, const Overrides&, Launch*) = {plan_conv_fwd, plan_conv_dgrad,
                                                                                           plan_conv_wgrad, plan_bgemm};
    if (q.kind < 0 || q.kind > T2V_GEMM_BGEMM) return fail(-2, "gemm_plan: unknown problem kind %d", q.kind);
    return planners[q.kind](q, sms, ov, l);
}

// Finishing pass of a split-K problem: out = alpha * acc + bias + rowbias + residual and, when `stats` is set, the GroupNorm
// statistics of out.  A block owns RPB consecutive rows (with statistics: of ONE sample) and 256 column quads; a thread loads
// its quad of all RPB rows up front (independent loads: one memory round trip), finishes them, and adds the column sums with
// two red.add.v4.
template <int RPB>
__global__ void __launch_bounds__(256) splitk_finish_kernel(const float* __restrict__ acc, const float* __restrict__ bias,
                                                            const float* __restrict__ rowbias, const __nv_bfloat16* __restrict__ residual,
                                                            void* __restrict__ out, int64_t rows, int C, int64_t rows_per_sample, int rb_div,
                                                            int64_t rb_ld, float alpha, int out_fp32, float* __restrict__ stats,
                                                            int64_t st_ld, int st_rows) {
    pdl_sync();
    const int64_t r0 = int64_t(blockIdx.x) * RPB;
    const int c = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
    if (c >= C) return;
    float4 v[RPB];
    uint2 w[RPB];
#pragma unroll
    for (int i = 0; i < RPB; ++i) {
        const int64_t r = r0 + i;
        if (r < rows) {
            v[i] = __ldcg(reinterpret_cast<const float4*>(acc + r * C + c));
            if (residual) w[i] = __ldg(reinterpret_cast<const uint2*>(residual + r * C + c));
        }
    }
    float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias) b4 = __ldg(reinterpret_cast<const float4*>(bias + c));
    float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < RPB; ++i) {
        const int64_t r = r0 + i;
        if (r >= rows) break;
        float4 y = v[i];
        y.x *= alpha; y.y *= alpha; y.z *= alpha; y.w *= alpha;
        if (bias) {
            y.x += b4.x; y.y += b4.y; y.z += b4.z; y.w += b4.w;
        }
        if (rowbias) {
            const float4 b = __ldg(reinterpret_cast<const float4*>(rowbias + (r / rows_per_sample / rb_div) * rb_ld + c));
            y.x += b.x; y.y += b.y; y.z += b.z; y.w += b.w;
        }
        if (residual) {
            y.x += bf16_lo(w[i].x); y.y += bf16_hi(w[i].x); y.z += bf16_lo(w[i].y); y.w += bf16_hi(w[i].y);
        }
        if (out_fp32) {
            reinterpret_cast<float4*>(static_cast<float*>(out) + r * C)[c >> 2] = y;
        } else {
            uint2 o;
            o.x = pack_bf16(y.x, y.y);
            o.y = pack_bf16(y.z, y.w);
            reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(out) + r * C)[c >> 2] = o;
            // the statistics describe what the consumer reads: the rounded values
            y.x = bf16_lo(o.x); y.y = bf16_hi(o.x); y.z = bf16_lo(o.y); y.w = bf16_hi(o.y);
        }
        s[0] += y.x; s[1] += y.y; s[2] += y.z; s[3] += y.w;
        q[0] += y.x * y.x; q[1] += y.y * y.y; q[2] += y.z * y.z; q[3] += y.w * y.w;
    }
    if (stats) {
        float* sp = stats + ((r0 / st_rows) * st_ld + c) * 2;
        red_add_f32x4(sp, s[0], q[0], s[1], q[1]);
        red_add_f32x4(sp + 4, s[2], q[2], s[3], q[3]);
    }
}

// Runs the planned problem split over k into `ws` and finishes into the real output.  `e` is the caller's epilogue.
int launch_split(GemmParams& p, bool a_mn, bool b_mn, const T2VEpilogue& e, void* out, int64_t rows, int C, int64_t rows_per_sample,
                 cudaStream_t st, const char* what) {
    const size_t bytes = size_t(rows) * C * sizeof(float);
    if (!e.workspace || size_t(e.workspace_bytes) < bytes) return fail(-3, "%s: split-K needs %zu bytes of workspace", what, bytes);
    cudaMemsetAsync(e.workspace, 0, bytes, st);
    p.out = e.workspace;
    p.out_mode = OUT_F32_RED;
    p.alpha = 1.0f;
    p.bias = nullptr; p.rowbias = nullptr; p.residual = nullptr;
    p.flags = 0;
    set_vec_flag(p);
    if (int r = launch_checked(launch_gemm(p, a_mn, b_mn, st), what)) return r;
    const bool stats = e.stats && e.stats_rows > 0 && e.stats_ld % 2 == 0 && (reinterpret_cast<uintptr_t>(e.stats) & 15u) == 0;
    // rows per block: with statistics a divisor of the sample's rows, so that a block never straddles two samples
    const int rpb = !stats || e.stats_rows % 4 == 0 ? 4 : (e.stats_rows % 2 == 0 ? 2 : 1);
    const dim3 grid(unsigned((rows + rpb - 1) / rpb), unsigned((C / 4 + 255) / 256));
    const dim3 block(unsigned(std::min(256, (C / 4 + 31) / 32 * 32)));
    auto go = [&](auto kern) {
        return int(launch_pdl(kern, grid, block, 0, st, static_cast<const float*>(e.workspace), e.bias, e.rowbias,
                              static_cast<const __nv_bfloat16*>(e.residual), out, rows, C, rows_per_sample,
                              e.rowbias_div > 0 ? e.rowbias_div : 1, int64_t(C), e.alpha, e.out_fp32, stats ? e.stats : nullptr,
                              e.stats_ld, e.stats_rows));
    };
    return launch_checked(rpb == 4 ? go(splitk_finish_kernel<4>) : (rpb == 2 ? go(splitk_finish_kernel<2>) : go(splitk_finish_kernel<1>)), what);
}

}  // namespace

extern "C" {

int t2v_gemm_plan(const T2VGemmProblem* problem, int32_t sm_count, T2VGemmPlan* out, int32_t max_out) {
    Launch l[4];
    const int n = plan(*problem, sm_count, read_overrides(), l);
    for (int i = 0; i < n && i < max_out; ++i) {
        const GemmParams& p = l[i].p;
        T2VGemmPlan& o = out[i];
        o.block_n = p.block_n; o.num_stages = p.num_stages;
        o.splits = p.ksplit_var >= 0 ? p.tdim[p.ksplit_var] : 1; o.kb_per_split = p.kb_per_split; o.ksplit_var = p.ksplit_var;
        o.num_tiles = p.num_tiles; o.grid = std::min(p.num_tiles, sm_count);
        o.box[0] = p.bw; o.box[1] = p.bh; o.box[2] = p.bn;
        std::copy(p.tdim, p.tdim + 6, o.tdim); std::copy(p.kdim, p.kdim + 3, o.kdim);
        o.flags = p.flags; o.follow = l[i].follow;
        o.st[0] = p.st_cw; o.st[1] = p.st_ch; o.st[2] = p.st_cn; o.st[3] = p.st_div; o.st[4] = p.st_seg;
    }
    return n;
}

int t2v_conv_fwd(const void* x, const void* w, void* y, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                 int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0, int32_t pad_w1,
                 const T2VEpilogue* epi, void* stream) {
    const T2VGemmProblem q{T2V_GEMM_CONV_FWD, N, H, W, Cin, Cout, KH, KW, stride, pad_h0, pad_h1, pad_w0, pad_w1,
                           epi && epi->workspace, epi && epi->stats ? epi->stats_rows : 0};
    Launch l;
    if (int r = plan_conv_fwd(q, device_sm_count(), read_overrides(), &l); r < 0) return r;
    GemmParams& p = l.p;
    const int Ho = p.H, Wo = p.W;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    // A: activations, K-major pixel box with tap shifts
    {
        TmaOperand& a = p.a;
        const uint64_t dims[4] = {uint64_t(Cin), uint64_t(W), uint64_t(H), uint64_t(N)};
        const uint64_t str[3] = {uint64_t(Cin) * 2, uint64_t(W) * Cin * 2, uint64_t(H) * W * Cin * 2};
        const uint32_t box[4] = {64, uint32_t(p.bw * stride), uint32_t(p.bh * stride), uint32_t(p.bn)};
        const uint32_t est[4] = {1, uint32_t(stride), uint32_t(stride), 1};
        if (int r = encode_tmap_bf16(&a.map, x, 4, dims, str, box, est)) return fail(r, "conv_fwd: A tensor map (%d)", r);
        a.rank = 4; a.nbox = 1; a.box_dim = 0; a.box_step = 0; a.box_bytes = p.bw * p.bh * p.bn * 128;
        a.base[1] = -pad_w0; a.base[2] = -pad_h0;
        a.tcoef[1][1] = p.bw * stride; a.tcoef[2][2] = p.bh * stride; a.tcoef[3][3] = p.bn;
        a.kcoef[0][0] = kBlockK; a.kcoef[1][1] = 1; a.kcoef[2][2] = 1;
    }
    // B: weights [Cout][KH*KW*Cin], K-major rows
    {
        TmaOperand& b = p.b;
        const uint64_t kt = uint64_t(KH) * KW * Cin;
        const uint64_t dims[2] = {kt, uint64_t(Cout)};
        const uint64_t str[1] = {kt * 2};
        const uint32_t box[2] = {64, uint32_t(p.block_n)};
        if (int r = encode_tmap_bf16(&b.map, w, 2, dims, str, box, nullptr)) return fail(r, "conv_fwd: B tensor map (%d)", r);
        b.rank = 2; b.nbox = 1; b.box_bytes = p.block_n * 128;
        b.tcoef[1][0] = p.block_n;
        b.kcoef[0][0] = kBlockK; b.kcoef[0][1] = Cin; b.kcoef[0][2] = KW * Cin;
    }
    fill_epilogue(p, epi, y, OUT_BF16);
    if (l.follow == T2V_FOLLOW_SPLITK_FINISH)
        return launch_split(p, false, false, *epi, y, int64_t(N) * Ho * Wo, Cout, int64_t(Ho) * Wo, st, "conv_fwd");
    set_vec_flag(p);
    // (pointers that are not 16-byte aligned, or an fp32 output, also leave the statistics to the standalone pass)
    const bool stats_pass = epi && epi->stats && (!(p.flags & EPI_STATS) || !(p.flags & EPI_VEC) || epi->out_fp32);
    if (stats_pass) p.flags &= ~EPI_STATS;
    if (p.flags & EPI_STATS) { p.stats = epi->stats; p.st_ld = epi->stats_ld; }
    if (int r = launch_checked(launch_gemm(p, false, false, st), "conv_fwd")) return r;
    if (stats_pass) {   // the epilogue cannot produce the statistics: one extra read of the (L2-hot) output
        if (epi->out_fp32 || epi->stats_rows <= 0 || (int64_t(N) * Ho * Wo) % epi->stats_rows)
            return fail(-2, "conv_fwd: statistics requested for an unsupported output (fp32 or ragged frames)");
        const int frames = int(int64_t(N) * Ho * Wo / epi->stats_rows);
        return launch_checked(launch_channel_stats(y, epi->stats, frames, epi->stats_rows, Cout, epi->stats_ld, st), "conv_fwd(stats)");
    }
    return 0;
}

int t2v_conv_dgrad(const void* dy, const void* w, void* dx, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                   int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0,
                   int32_t pad_w1, const T2VEpilogue* epi, void* stream) {
    const T2VGemmProblem q{T2V_GEMM_CONV_DGRAD, N, H, W, Cin, Cout, KH, KW, stride, pad_h0, pad_h1, pad_w0, pad_w1, epi && epi->workspace};
    Launch ls[4];
    const int n = plan_conv_dgrad(q, device_sm_count(), read_overrides(), ls);
    if (n < 0) return n;
    const int s = stride, Ho = (H + pad_h0 + pad_h1 - KH) / s + 1, Wo = (W + pad_w0 + pad_w1 - KW) / s + 1;
    const T2VEpilogue e = epi ? *epi : T2VEpilogue{nullptr, nullptr, nullptr, 1.0f, 0, 1, nullptr, 0};
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i = 0; i < n; ++i) {
        GemmParams& p = ls[i].p;
        const int ph = ls[i].ph, pw = ls[i].pw, th0 = ls[i].th0, tw0 = ls[i].tw0;
        {
            TmaOperand& a = p.a;  // dy, K-major (K = Cout), pixel box shifted against the tap
            const uint64_t dims[4] = {uint64_t(Cout), uint64_t(Wo), uint64_t(Ho), uint64_t(N)};
            const uint64_t str[3] = {uint64_t(Cout) * 2, uint64_t(Wo) * Cout * 2, uint64_t(Ho) * Wo * Cout * 2};
            const uint32_t box[4] = {64, uint32_t(p.bw), uint32_t(p.bh), uint32_t(p.bn)};
            if (int r = encode_tmap_bf16(&a.map, dy, 4, dims, str, box, nullptr)) return fail(r, "conv_dgrad: A tensor map (%d)", r);
            a.rank = 4; a.nbox = 1; a.box_bytes = p.bw * p.bh * p.bn * 128;
            a.base[1] = (pw + pad_w0 - tw0) / s; a.base[2] = (ph + pad_h0 - th0) / s;
            a.tcoef[1][1] = p.bw; a.tcoef[2][2] = p.bh; a.tcoef[3][3] = p.bn;
            a.kcoef[0][0] = kBlockK; a.kcoef[1][1] = -1; a.kcoef[2][2] = -1;
        }
        {
            TmaOperand& b = p.b;  // w viewed as [Cout (k)][tap][Cin (n, contiguous)] -> MN-major
            const uint64_t dims[3] = {uint64_t(Cin), uint64_t(KH) * KW, uint64_t(Cout)};
            const uint64_t str[2] = {uint64_t(Cin) * 2, uint64_t(KH) * KW * Cin * 2};
            const uint32_t box[3] = {64, 1, 64};
            if (int r = encode_tmap_bf16(&b.map, w, 3, dims, str, box, nullptr)) return fail(r, "conv_dgrad: B tensor map (%d)", r);
            b.rank = 3; b.nbox = (p.block_n + 63) / 64; b.box_dim = 0; b.box_step = 64; b.box_bytes = 8192;
            b.base[1] = th0 * KW + tw0;
            b.tcoef[0][0] = p.block_n;
            b.kcoef[1][1] = s; b.kcoef[1][2] = s * KW; b.kcoef[2][0] = kBlockK;
        }
        const int64_t base_off = (int64_t(ph) * W + pw) * Cin;
        fill_epilogue(p, &e, static_cast<char*>(dx) + base_off * (e.out_fp32 ? 4 : 2), OUT_BF16);
        if (p.residual) p.residual = static_cast<const char*>(p.residual) + base_off * 2;
        if (ls[i].follow == T2V_FOLLOW_SPLITK_FINISH)
            return launch_split(p, false, true, e, dx, int64_t(N) * H * W, Cin, int64_t(H) * W, st, "conv_dgrad");
        set_vec_flag(p);
        if (int r = launch_checked(launch_gemm(p, false, true, st), "conv_dgrad")) return r;
    }
    return 0;
}

int64_t t2v_conv_workspace_bytes(int32_t dgrad, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout, int32_t KH, int32_t KW,
                                 int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0, int32_t pad_w1) {
    const T2VGemmProblem q{dgrad ? T2V_GEMM_CONV_DGRAD : T2V_GEMM_CONV_FWD, N, H, W, Cin, Cout, KH, KW, stride, pad_h0, pad_h1,
                           pad_w0, pad_w1, 1};
    Launch l[4];
    if (plan(q, device_sm_count(), read_overrides(), l) < 1 || l[0].follow != T2V_FOLLOW_SPLITK_FINISH) return 0;
    return int64_t(l[0].p.N) * l[0].p.H * l[0].p.W * l[0].p.ncols * 4;   // an fp32 image of the output
}

int t2v_conv_wgrad_bias(const void* x, const void* dy, float* dw, float* dbias, int32_t N, int32_t H, int32_t W, int32_t Cin,
                        int32_t Cout, int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0,
                        int32_t pad_w1, void* stream) {
    const T2VGemmProblem q{T2V_GEMM_CONV_WGRAD, N, H, W, Cin, Cout, KH, KW, stride, pad_h0, pad_h1, pad_w0, pad_w1, 0, 0, dbias != nullptr};
    Launch l;
    if (int r = plan_conv_wgrad(q, device_sm_count(), read_overrides(), &l); r < 0) return r;
    GemmParams& p = l.p;
    const Box3 kx = l.kbox;
    const int Ho = (H + pad_h0 + pad_h1 - KH) / stride + 1, Wo = (W + pad_w0 + pad_w1 - KW) / stride + 1;
    {
        TmaOperand& a = p.a;  // dy^T: M = Cout (contiguous), K = pixels -> MN-major, two 64-wide boxes
        const uint64_t dims[4] = {uint64_t(Cout), uint64_t(Wo), uint64_t(Ho), uint64_t(N)};
        const uint64_t str[3] = {uint64_t(Cout) * 2, uint64_t(Wo) * Cout * 2, uint64_t(Ho) * Wo * Cout * 2};
        const uint32_t box[4] = {64, uint32_t(kx.w), uint32_t(kx.h), uint32_t(kx.n)};
        if (int r = encode_tmap_bf16(&a.map, dy, 4, dims, str, box, nullptr)) return fail(r, "conv_wgrad: A tensor map (%d)", r);
        a.rank = 4; a.nbox = 2; a.box_dim = 0; a.box_step = 64; a.box_bytes = 8192;
        a.tcoef[0][1] = kBlockM;
        a.kcoef[1][0] = kx.w; a.kcoef[2][1] = kx.h; a.kcoef[3][2] = kx.n;
    }
    {
        TmaOperand& b = p.b;  // x shifted by the tap: N = Cin (contiguous), K = pixels -> MN-major
        const uint64_t dims[4] = {uint64_t(Cin), uint64_t(W), uint64_t(H), uint64_t(N)};
        const uint64_t str[3] = {uint64_t(Cin) * 2, uint64_t(W) * Cin * 2, uint64_t(H) * W * Cin * 2};
        const uint32_t box[4] = {64, uint32_t(kx.w * stride), uint32_t(kx.h * stride), uint32_t(kx.n)};
        const uint32_t est[4] = {1, uint32_t(stride), uint32_t(stride), 1};
        if (int r = encode_tmap_bf16(&b.map, x, 4, dims, str, box, est)) return fail(r, "conv_wgrad: B tensor map (%d)", r);
        b.rank = 4; b.nbox = (p.block_n + 63) / 64; b.box_dim = 0; b.box_step = 64; b.box_bytes = 8192;
        b.base[1] = -pad_w0; b.base[2] = -pad_h0;
        b.tcoef[0][0] = p.block_n; b.tcoef[1][2] = 1; b.tcoef[2][3] = 1;
        b.kcoef[1][0] = kx.w * stride; b.kcoef[2][1] = kx.h * stride; b.kcoef[3][2] = kx.n;
    }
    fill_epilogue(p, nullptr, dw, OUT_F32_RED);
    set_vec_flag(p);
    if (p.flags & EPI_ROWSUM_A) p.rowsum = dbias;
    if (int r = launch_checked(launch_gemm(p, true, true, static_cast<cudaStream_t>(stream)), "conv_wgrad")) return r;
    if (l.follow == T2V_FOLLOW_COLSUM) return t2v_colsum(dy, dbias, 1, int64_t(N) * Ho * Wo, Cout, stream);
    return 0;
}

int t2v_conv_wgrad(const void* x, const void* dy, float* dw, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                   int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0,
                   int32_t pad_w1, void* stream) {
    return t2v_conv_wgrad_bias(x, dy, dw, nullptr, N, H, W, Cin, Cout, KH, KW, stride, pad_h0, pad_h1, pad_w0, pad_w1, stream);
}

int t2v_bgemm(const T2VMat* A, const T2VMat* B, void* C, int64_t ldc, int64_t c_stride_z1, int64_t c_stride_z2,
              int32_t M, int32_t N, int32_t K, int32_t Z1, int32_t Z2, float alpha, int32_t out_mode, void* stream) {
    T2VGemmProblem q{T2V_GEMM_BGEMM};
    q.gemm_m = M; q.gemm_n = N; q.gemm_k = K; q.z1 = Z1; q.z2 = Z2; q.b_kmajor = B->kmajor; q.out_mode = out_mode;
    Launch l;
    if (int r = plan_bgemm(q, device_sm_count(), read_overrides(), &l); r < 0) return r;
    if (A->ld % 8 || B->ld % 8) return fail(-2, "bgemm: leading dimensions must be multiples of 8 elements");
    if ((Z1 > 1 && (A->stride_z1 % 8 || B->stride_z1 % 8)) || (Z2 > 1 && (A->stride_z2 % 8 || B->stride_z2 % 8)))
        return fail(-2, "bgemm: batch strides must be multiples of 8 elements");
    const bool a_mn = !A->kmajor, b_mn = !B->kmajor;
    GemmParams& p = l.p;
    auto stride_or = [](int64_t s, int64_t fallback) { return uint64_t((s > 0 ? s : fallback) * 2); };
    auto plan_operand = [&](TmaOperand& op, const T2VMat* m, bool mn, int rows_mn, int block_mn, int tile_var) -> int {
        // stored matrix: K-major [rows_mn][K]; MN-major [K][rows_mn]
        const uint64_t inner = mn ? uint64_t(rows_mn) : uint64_t(K), outer = mn ? uint64_t(K) : uint64_t(rows_mn);
        const uint64_t dims[4] = {inner, outer, uint64_t(Z2), uint64_t(Z1)};
        const uint64_t str[3] = {uint64_t(m->ld) * 2, stride_or(m->stride_z2, m->ld * int64_t(outer)),
                                 stride_or(m->stride_z1, m->ld * int64_t(outer) * Z2)};
        const uint32_t box[4] = {64, uint32_t(mn ? 64 : block_mn), 1, 1};
        if (int r = encode_tmap_bf16(&op.map, m->ptr, 4, dims, str, box, nullptr)) return r;
        op.rank = 4;
        op.tcoef[2][4] = 1;
        op.tcoef[3][5] = 1;
        if (mn) {
            op.nbox = (block_mn + 63) / 64; op.box_dim = 0; op.box_step = 64; op.box_bytes = 8192;
            op.tcoef[0][tile_var] = block_mn;
            op.kcoef[1][0] = kBlockK;
        } else {
            op.nbox = 1; op.box_bytes = block_mn * 128;
            op.tcoef[1][tile_var] = block_mn;
            op.kcoef[0][0] = kBlockK;
        }
        return 0;
    };
    if (int r = plan_operand(p.a, A, a_mn, M, kBlockM, 1)) return fail(r, "bgemm: A tensor map (%d)", r);
    if (int r = plan_operand(p.b, B, b_mn, N, p.block_n, 0)) return fail(r, "bgemm: B tensor map (%d)", r);
    p.ldw = ldc; p.ldh = 0; p.ldn = 0;
    p.otc[4] = c_stride_z2; p.otc[5] = c_stride_z1;
    T2VEpilogue e{nullptr, nullptr, nullptr, alpha, out_mode != OUT_BF16, 1};
    fill_epilogue(p, &e, C, OUT_BF16);
    p.out_mode = out_mode;
    set_vec_flag(p);
    return launch_checked(launch_gemm(p, a_mn, b_mn, static_cast<cudaStream_t>(stream)), "bgemm");
}

}  // extern "C"
