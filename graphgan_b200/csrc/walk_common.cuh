// walk_common.cuh -- building blocks shared by the walk sampler (walk.cu) and the per-pass
// precompute kernels (hub.cu): canonical scoring of a candidate list and the canonical
// softmax / CDF passes.  All of it is the arithmetic of DESIGN.md section 3.
#pragma once
#include "gg_common.cuh"

namespace gg {

// Tuning knobs (compile-time; tools/variants.py builds A/B libraries with -DGG_...): the walk kernels are latency
// bound, so the trade is occupancy (registers, shared memory per warp) against loads in flight per warp (unrolling)
// and against instruction footprint (the hot path must stay near the 32 KB L1.5 instruction cache).  The defaults are
// the H100's A/B winner (DESIGN.md section 8.1): 3 CTAs/SM at 80 registers, 2048 scores per warp in shared memory
// (3 x 74 KB of the SM's 228 KB), 4 tiles in flight.
#ifndef GG_SC_CAP
#define GG_SC_CAP 2048
#endif
#ifndef GG_UNR
#define GG_UNR 4
#endif
#ifndef GG_UNR_S1
#define GG_UNR_S1 8
#endif
#ifndef GG_WALK_MIN_CTAS
#define GG_WALK_MIN_CTAS 3
#endif
constexpr int WARPS_PER_CTA = 8;
constexpr int WALK_MIN_CTAS = GG_WALK_MIN_CTAS;   // CTAs per SM the walk kernels are compiled and launched for
constexpr int ID_CAP = 320;    // candidate ids per warp kept in shared memory (longer lists: global scratch)
constexpr int SC_CAP = GG_SC_CAP;   // candidate scores per warp kept in shared memory
constexpr int SMEM_CAP = ID_CAP;
constexpr int WALK_SMEM_PER_WARP = SC_CAP * 4 + ID_CAP * 4 + 16;   // + the warp's mbarrier (TMA staging of hub lists)
constexpr int STAGE_ENTRIES = 512;  // adjacency entries per bulk-copy block: 2 KB of ids + 2 KB of cached scores
static_assert(2 * STAGE_ENTRIES * 4 <= SC_CAP * 4, "the staging area is the warp's (idle) score buffer");

// Per-warp TMA staging state: `buf` = the warp's shared score buffer (free whenever a list is too long for it), `bar` =
// the warp's mbarrier, `phase` = its parity.  on = false: plain loads (stream-replay kernel, or desc.no_tma).
struct Stage {
    float *buf;
    unsigned long long *bar;
    unsigned phase;
    bool on;
};
constexpr int UNR = GG_UNR;    // tiles of 32 candidates in flight per pass iteration (walk kernel: short lists, many warps)
constexpr int UNR_S1 = GG_UNR_S1;   // same, for the per-pass list builders (step1_cdf_kernel: long lists)

// cur row in registers: lane (grp, g) holds float4 chunks g, g+8, ... (replicated over the 4 groups)
template <int CPL>
__device__ __forceinline__ void load_row(const float *__restrict__ emb, int ld, int node, int g, float4 (&c4)[CPL]) {
    const float *crow = emb + (size_t)node * (size_t)ld + 4 * g;
#pragma unroll
    for (int c = 0; c < CPL; ++c) c4[c] = ldg4(crow + 32 * c);
}

// sc[i] = dot(cur, emb[ids[i]]) + bias[ids[i]] for i in [0, n): all_score[cur, cand] (generator.py:21).
// Four 8-lane groups, two candidate rows in flight per group.
template <int CPL>
__device__ __forceinline__ void score_list(const float *__restrict__ emb, const float *__restrict__ bias, int ld,
                                           const float4 (&c4)[CPL], const int *ids, float *sc, int n, int fallback,
                                           int lane) {
    const int grp = lane >> 3, g = lane & 7;
    // (the ids of the NEXT eight candidates are fetched while this iteration's rows are in flight: the id -> row
    // dependency costs one exposed round trip per list instead of one per iteration)
    int ca_n = (grp < n) ? ids[grp] : fallback, cb_n = (4 + grp < n) ? ids[4 + grp] : fallback;
    for (int i0 = 0; i0 < n; i0 += 8) {
        const int ia = i0 + grp, ib = i0 + 4 + grp;
        const bool va = ia < n, vb = ib < n;
        const int ca = ca_n, cb = cb_n;
        ca_n = (ia + 8 < n) ? ids[ia + 8] : fallback;
        cb_n = (ib + 8 < n) ? ids[ib + 8] : fallback;
        const float *ra = emb + (size_t)ca * (size_t)ld + 4 * g;
        const float *rb = emb + (size_t)cb * (size_t)ld + 4 * g;
        float4 xa[CPL], xb[CPL];
#pragma unroll
        for (int c = 0; c < CPL; ++c) xa[c] = ldg4(ra + 32 * c);
#pragma unroll
        for (int c = 0; c < CPL; ++c) xb[c] = ldg4(rb + 32 * c);
        const float ba = __ldg(bias + ca), bb = __ldg(bias + cb);
        float sa = 0.0f, sb = 0.0f;
#pragma unroll
        for (int c = 0; c < CPL; ++c) sa = fma4(c4[c], xa[c], sa);
#pragma unroll
        for (int c = 0; c < CPL; ++c) sb = fma4(c4[c], xb[c], sb);
        sa = group8_sum(sa);
        sb = group8_sum(sb);
        if (g == 0) {
            if (va) sc[ia] = __fadd_rn(sa, ba);
            if (vb) sc[ib] = __fadd_rn(sb, bb);
        }
    }
    __syncwarp();
}

// The canonical dots of the register row c4 with rows ca and cb of emb: lane g's fma chain over its chunks g, g + 8, ...,
// then the group's butterfly.  fma(a, b, s) rounds a * b + s once whichever operand is the register row, so the dot of
// u and v is the same bits with either of them in c4 (score_edges holds the source, score_pairs the target).
template <int CPL>
__device__ __forceinline__ void dot2(const float *__restrict__ emb, int ld, const float4 (&c4)[CPL], int ca, int cb, int g,
                                     float &sa, float &sb) {
    const float *ra = emb + (size_t)ca * (size_t)ld + 4 * g;
    const float *rb = emb + (size_t)cb * (size_t)ld + 4 * g;
    float4 xa[CPL], xb[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) xa[c] = ldg4(ra + 32 * c);
#pragma unroll
    for (int c = 0; c < CPL; ++c) xb[c] = ldg4(rb + 32 * c);
    sa = 0.0f;
    sb = 0.0f;
#pragma unroll
    for (int c = 0; c < CPL; ++c) sa = fma4(c4[c], xa[c], sa);
#pragma unroll
    for (int c = 0; c < CPL; ++c) sb = fma4(c4[c], xb[c], sb);
    sa = group8_sum(sa);
    sb = group8_sum(sb);
}

// Same, for a contiguous run of adjacency entries (ids read straight from the CSR).
template <int CPL>
__device__ __forceinline__ void score_edges(const float *__restrict__ emb, const float *__restrict__ bias, int ld,
                                            const float4 (&c4)[CPL], const int *__restrict__ adj, long long e0,
                                            int n, float *out, int fallback, int lane) {
    const int grp = lane >> 3, g = lane & 7;
    int ca_n = (grp < n) ? __ldg(adj + e0 + grp) : fallback, cb_n = (4 + grp < n) ? __ldg(adj + e0 + 4 + grp) : fallback;
    for (int i0 = 0; i0 < n; i0 += 8) {
        const int ia = i0 + grp, ib = i0 + 4 + grp;
        const bool va = ia < n, vb = ib < n;
        const int ca = ca_n, cb = cb_n;          // (next iteration's ids in flight behind this iteration's rows, see score_list)
        ca_n = (ia + 8 < n) ? __ldg(adj + e0 + ia + 8) : fallback;
        cb_n = (ib + 8 < n) ? __ldg(adj + e0 + ib + 8) : fallback;
        float sa, sb;
        dot2<CPL>(emb, ld, c4, ca, cb, g, sa, sb);
        const float ba = __ldg(bias + ca), bb = __ldg(bias + cb);
        if (g == 0) {
            if (va) out[ia] = __fadd_rn(sa, ba);
            if (vb) out[ib] = __fadd_rn(sb, bb);
        }
    }
    __syncwarp();
}

// score_edges the other way round (hub_score_tm_kernel): c4 holds the row of ONE target v, and the group scores the n hub
// entries e_i = (u_i -> v) listed as pairs (u_i, e_i): out[e_i] = dot(E[u_i], E[v]) + b[v] = all_score[u_i, v].  Each
// group has its own list (n differs between the groups), two rows in flight, the next pairs fetched behind them;
// n_warp = the largest n of the warp keeps the group butterflies warp-uniform.
template <int CPL>
__device__ __forceinline__ void score_pairs(const float *__restrict__ emb, int ld, const float4 (&c4)[CPL], float bv,
                                            const int2 *__restrict__ pairs, int n, int n_warp, float *__restrict__ out,
                                            int fallback, int lane) {
    const int g = lane & 7;
    const int2 fb = make_int2(fallback, 0);
    int2 pa_n = (0 < n) ? __ldg(pairs) : fb, pb_n = (1 < n) ? __ldg(pairs + 1) : fb;
    for (int i0 = 0; i0 < n_warp; i0 += 2) {
        const int2 pa = pa_n, pb = pb_n;
        pa_n = (i0 + 2 < n) ? __ldg(pairs + i0 + 2) : fb;
        pb_n = (i0 + 3 < n) ? __ldg(pairs + i0 + 3) : fb;
        float sa, sb;
        dot2<CPL>(emb, ld, c4, pa.x, pb.x, g, sa, sb);
        if (g == 0) {
            if (i0 < n) out[pa.y] = __fadd_rn(sa, bv);
            if (i0 + 1 < n) out[pb.y] = __fadd_rn(sb, bv);
        }
    }
    __syncwarp();
}

// ---- ld = 512 (CPL = 16).  The current row (16 float4 per lane) and two candidate rows (32 more) do not fit in registers,
// so the warp keeps the current row in shared memory (WIDE_ROW_BYTES, one copy for the four groups) and each group streams
// ONE candidate row per iteration: 16 float4 per lane in flight, as many bytes per round trip as the two half-as-wide rows
// of CPL = 8.  Lane g still owns chunks g, g + 8, ..., g + 120 and runs one fma chain over them in that order, so a score
// is the same bits as the register path's.  The walk kernels append the rows after their per-warp blocks and run at
// WIDE_MIN_CTAS CTAs per SM (3 x (8 x 9 488 + 16 KB) does not fit in the SM's 228 KB; 2 x 92 KB does).
constexpr int WIDE_CPL = 16;
constexpr int WIDE_ROW_BYTES = WIDE_CPL * 32 * 4;
constexpr int WIDE_MIN_CTAS = 2;
__host__ __device__ constexpr int walk_min_ctas(int cpl) { return cpl == WIDE_CPL ? WIDE_MIN_CTAS : WALK_MIN_CTAS; }
// dynamic shared memory of a walk kernel of `nwarps` warps
__host__ __device__ constexpr int walk_smem_bytes(int cpl, int nwarps) {
    return nwarps * (WALK_SMEM_PER_WARP + (cpl == WIDE_CPL ? WIDE_ROW_BYTES : 0));
}
static_assert(WALK_SMEM_PER_WARP % 16 == 0 && WIDE_ROW_BYTES % 16 == 0, "the row buffers are read as float4");
static_assert(WIDE_MIN_CTAS * walk_smem_bytes(WIDE_CPL, WARPS_PER_CTA) <= 227 * 1024, "ld = 512 walk CTAs must fit on an SM");

// the warp's row buffer of a walk kernel: s_sc is the warp's block of the per-warp layout (blockDim.x / 32 blocks)
__device__ __forceinline__ float *walk_wide_row(float *s_sc) {
    const int nw = blockDim.x >> 5, wid = threadIdx.x >> 5;
    return reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(s_sc) + (size_t)(nw - wid) * WALK_SMEM_PER_WARP +
                                     (size_t)wid * WIDE_ROW_BYTES);
}

// the row of `node` into the warp's row buffer (the previous list's scoring has finished: score_* end with __syncwarp)
__device__ __forceinline__ void load_row_wide(const float *__restrict__ emb, int ld, int node, float *s_row, int lane) {
    const float *crow = emb + (size_t)node * (size_t)ld;
#pragma unroll
    for (int k = 0; k < WIDE_CPL / 4; ++k)
        *reinterpret_cast<float4 *>(s_row + 4 * (lane + 32 * k)) = ldg4(crow + 4 * (lane + 32 * k));
    __syncwarp();
}

// score of the candidate row `r` (this lane's chunks) against the row in s_row: the canonical dot, group-reduced
__device__ __forceinline__ float wide_dot(const float *s_row, const float *r, int g) {
    float4 x[WIDE_CPL];
#pragma unroll
    for (int c = 0; c < WIDE_CPL; ++c) x[c] = ldg4(r + 32 * c);
    float s = 0.0f;
#pragma unroll
    for (int c = 0; c < WIDE_CPL; ++c) s = fma4(*reinterpret_cast<const float4 *>(s_row + 4 * g + 32 * c), x[c], s);
    return group8_sum(s);
}

// score_list for ld = 512: one candidate per group per iteration
__device__ __forceinline__ void score_list_wide(const float *__restrict__ emb, const float *__restrict__ bias, int ld,
                                                const float *s_row, const int *ids, float *sc, int n, int fallback, int lane) {
    const int grp = lane >> 3, g = lane & 7;
    int c_n = (grp < n) ? ids[grp] : fallback;
    for (int i0 = 0; i0 < n; i0 += 4) {
        const int i = i0 + grp;
        const int c = c_n;
        c_n = (i + 4 < n) ? ids[i + 4] : fallback;   // (the next id in flight behind this row, see score_list)
        const float b = __ldg(bias + c);
        const float s = wide_dot(s_row, emb + (size_t)c * (size_t)ld + 4 * g, g);
        if (g == 0 && i < n) sc[i] = __fadd_rn(s, b);
    }
    __syncwarp();
}

// score_edges for ld = 512
__device__ __forceinline__ void score_edges_wide(const float *__restrict__ emb, const float *__restrict__ bias, int ld,
                                                 const float *s_row, const int *__restrict__ adj, long long e0, int n,
                                                 float *out, int fallback, int lane) {
    const int grp = lane >> 3, g = lane & 7;
    int c_n = (grp < n) ? __ldg(adj + e0 + grp) : fallback;
    for (int i0 = 0; i0 < n; i0 += 4) {
        const int i = i0 + grp;
        const int c = c_n;
        c_n = (i + 4 < n) ? __ldg(adj + e0 + i + 4) : fallback;
        const float b = __ldg(bias + c);
        const float s = wide_dot(s_row, emb + (size_t)c * (size_t)ld + 4 * g, g);
        if (g == 0 && i < n) out[i] = __fadd_rn(s, b);
    }
    __syncwarp();
}

// score_pairs for ld = 512: s_row = the GROUP's copy of the target row (load_row_group_wide), one hub row per iteration
__device__ __forceinline__ void score_pairs_wide(const float *__restrict__ emb, int ld, const float *s_row, float bv,
                                                 const int2 *__restrict__ pairs, int n, int n_warp, float *__restrict__ out,
                                                 int fallback, int lane) {
    const int g = lane & 7;
    const int2 fb = make_int2(fallback, 0);
    int2 p_n = (0 < n) ? __ldg(pairs) : fb;
    for (int i = 0; i < n_warp; ++i) {
        const int2 p = p_n;
        p_n = (i + 1 < n) ? __ldg(pairs + i + 1) : fb;
        const float s = wide_dot(s_row, emb + (size_t)p.x * (size_t)ld + 4 * g, g);
        if (g == 0 && i < n) out[p.y] = __fadd_rn(s, bv);
    }
    __syncwarp();
}

// the row of `node` into an 8-lane group's row buffer (WIDE_ROW_BYTES); the group's previous scoring has finished
__device__ __forceinline__ void load_row_group_wide(const float *__restrict__ emb, int ld, int node, float *s_row, int g) {
    const float *crow = emb + (size_t)node * (size_t)ld;
#pragma unroll
    for (int k = 0; k < WIDE_CPL; ++k)    // 128 float4 chunks, 16 per lane
        *reinterpret_cast<float4 *>(s_row + 4 * (g + 8 * k)) = ldg4(crow + 4 * (g + 8 * k));
    __syncwarp();
}

// max over sc[0..n)
__device__ __forceinline__ float list_max(const float *sc, int n, int lane) {
    float m = -INFINITY;
    for (int i = lane; i < n; i += 32) m = fmaxf(m, sc[i]);
    return warp_max(m);
}

// softmax numerators in place (sc[i] <- e_i = exp_c(s_i - m)) and their canonical sum
// S = T_0 + T_1 + ... (tile sums by butterfly; 0 + T_0 == T_0 and S + 0 == S exactly, so empty
// tiles of the unrolled tail are harmless).  UNR tiles are in flight per iteration.
template <int U = UNR>
__device__ __forceinline__ float softmax_exp_sum(float *sc, int n, float m, int lane) {
    float S = 0.0f;
    for (int t0 = 0; t0 < n; t0 += 32 * U) {
        float x[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int i = t0 + 32 * u + lane; x[u] = (i < n) ? sc[i] : 0.0f; }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (t0 + 32 * u >= n) break;            // warp-uniform: no work for the empty tiles of a short list
            const int i = t0 + 32 * u + lane;
            float e = 0.0f;
            if (i < n) { e = exp_c(__fsub_rn(x[u], m)); sc[i] = e; }
            S = __fadd_rn(S, warp_sum_butterfly(e));
        }
    }
    __syncwarp();
    return S;
}

// total of the float64 CDF over p_i = e_i / S.  Lane (t & 31) also keeps the running total after tile t
// in car[t >> 5] (tiles 0..63), so that the draw can jump straight to the tile that contains it.
template <int U = UNR>
__device__ __forceinline__ double cdf_total(const float *sc, int n, float S, int lane, double (&car)[2]) {
    double total = 0.0;
    car[0] = car[1] = 0.0;
    for (int t0 = 0; t0 < n; t0 += 32 * U) {
        float e[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int i = t0 + 32 * u + lane; e[u] = (i < n) ? sc[i] : 0.0f; }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (t0 + 32 * u >= n) break;            // warp-uniform
            double x = (double)__fdiv_rn(e[u], S);   // 0 / S == 0 for the padding lanes
            x = warp_scan_ks(x, lane);
            total = __dadd_rn(total, __shfl_sync(FULL, x, 31));
            const int t = (t0 >> 5) + u;
            if (t < 64 && lane == (t & 31)) car[t >> 5] = total;
        }
    }
    return total;
}

// first i with cdf_i / total > u, scanning tiles [t_begin, ...) with `carry` = CDF before tile t_begin
__device__ __forceinline__ int cdf_pick_from(const float *sc, int n, float S, double total, double u, int lane,
                                             int t_begin, double carry) {
    for (int t0 = 32 * t_begin; t0 < n; t0 += 32) {
        const int i = t0 + lane;
        double x = (double)__fdiv_rn((i < n) ? sc[i] : 0.0f, S);
        x = warp_scan_ks(x, lane);
        const double q = __ddiv_rn(__dadd_rn(carry, x), total);
        const unsigned hit = __ballot_sync(FULL, (i < n) && (q > u));
        if (hit) return t0 + __ffs(hit) - 1;
        carry = __dadd_rn(carry, __shfl_sync(FULL, x, 31));
    }
    return n - 1;
}

// The CDF is non-decreasing, so the first index with q > u lies in the first tile whose LAST q exceeds u,
// and that last q is exactly car[t] / total (same operations as the linear scan performs).  All lanes return idx.
__device__ __forceinline__ int cdf_pick(const float *sc, int n, float S, double total, double u, int lane,
                                        const double (&car)[2]) {
    const int ntiles = (n + 31) >> 5;
    int t_hit = -1;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int t = 32 * h + lane;
        const bool p = (t < ntiles) && (__ddiv_rn(car[h], total) > u);
        const unsigned mk = __ballot_sync(FULL, p);
        if (t_hit < 0 && mk) t_hit = 32 * h + __ffs(mk) - 1;
    }
    if (t_hit < 0) {   // beyond the 64 tracked tiles (n > 2048): linear scan from tile 64
        if (ntiles <= 64) return n - 1;
        const double c63 = __shfl_sync(FULL, car[1], 31);
        return cdf_pick_from(sc, n, S, total, u, lane, 64, c63);
    }
    double before = 0.0;
    if (t_hit > 0) {
        const int tp = t_hit - 1;
        const double lo = __shfl_sync(FULL, car[0], tp & 31), hi = __shfl_sync(FULL, car[1], tp & 31);
        before = (tp >> 5) ? hi : lo;
    }
    return cdf_pick_from(sc, n, S, total, u, lane, t_hit, before);
}

// Long lists (global scratch): running total after EVERY tile goes to `tiles` (the warp's idle shared score buffer
// viewed as doubles), so the draw can locate its tile among hundreds without a linear scan.
__device__ __forceinline__ double cdf_total_tiles(const float *sc, int n, float S, int lane, double *tiles) {
    constexpr int U = 8;
    double total = 0.0;
    for (int t0 = 0; t0 < n; t0 += 32 * U) {
        float e[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int i = t0 + 32 * u + lane; e[u] = (i < n) ? sc[i] : 0.0f; }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (t0 + 32 * u >= n) break;
            double x = (double)__fdiv_rn(e[u], S);
            x = warp_scan_ks(x, lane);
            total = __dadd_rn(total, __shfl_sync(FULL, x, 31));
            if (lane == 0) tiles[(t0 >> 5) + u] = total;
        }
    }
    __syncwarp();
    return total;
}
__device__ __forceinline__ int cdf_pick_tiles(const float *sc, int n, float S, double total, double u, int lane,
                                              const double *tiles) {
    const int ntiles = (n + 31) >> 5;
    for (int tb = 0; tb < ntiles; tb += 32) {
        const int t = tb + lane;
        const bool p = (t < ntiles) && (__ddiv_rn(tiles[t], total) > u);
        const unsigned mk = __ballot_sync(FULL, p);
        if (mk) {
            const int t_hit = tb + __ffs(mk) - 1;
            return cdf_pick_from(sc, n, S, total, u, lane, t_hit, t_hit > 0 ? tiles[t_hit - 1] : 0.0);
        }
    }
    return n - 1;
}

// One tile (n <= 32, the common case): S = 0 + T_0 = T_0, total = 0 + scan_31 = scan_31 and the carry of the draw is 0, so
// the canonical sequence collapses to ONE scan and ONE division per lane -- the same floats, bit for bit.  Returns the
// lane's inclusive scan x; the draw for u is the first lane with x / total > u.
__device__ __forceinline__ double tile1_cdf(const float *sc, int n, float m, int lane, double &total) {
    const float e = (lane < n) ? exp_c(__fsub_rn(sc[lane], m)) : 0.0f;
    const float S = warp_sum_butterfly(e);
    const double x = warp_scan_ks((double)__fdiv_rn(e, S), lane);
    total = __shfl_sync(FULL, x, 31);
    return x;
}
__device__ __forceinline__ int tile1_pick(double x, double total, int n, double u, int lane) {
    const unsigned hit = __ballot_sync(FULL, (lane < n) && (__ddiv_rn(x, total) > u));
    return hit ? __ffs(hit) - 1 : n - 1;
}

// A list's softmax + CDF, built once by cdf_prepare; cdf_draw then inverts it for as many uniforms as needed (it does
// not write sc).  Both run the passes choose_index runs, so a draw is the same bits whether or not other draws share
// the list.
struct ListCdf {
    float S;           // canonical softmax denominator
    double total;      // the CDF's total
    double car[2];     // n <= 32: car[0] = the lane's scan (tile1_cdf); else cdf_total's running totals
};

// lists longer than the shared score buffer (global scratch): rare, so kept out of line and modestly unrolled -- the
// walk kernel's instruction footprint is what its warps stall on otherwise (ncu: "no instruction").  With `tiles`, the
// running total after EVERY tile goes to the (idle) shared score buffer: the draw finds its tile among hundreds directly.
__device__ __forceinline__ bool long_uses_tiles(int n, const double *tiles) { return tiles && ((n + 31) >> 5) <= SC_CAP / 2; }
static __device__ __noinline__ void cdf_prepare_long(float *sc, int n, float m, int lane, double *tiles, ListCdf &c) {
    c.S = softmax_exp_sum<8>(sc, n, m, lane);
    if (long_uses_tiles(n, tiles)) c.total = cdf_total_tiles(sc, n, c.S, lane, tiles);
    else c.total = cdf_total<8>(sc, n, c.S, lane, c.car);
}
static __device__ __noinline__ int cdf_draw_long(const float *sc, int n, const ListCdf &c, double u, int lane,
                                                 const double *tiles) {
    if (long_uses_tiles(n, tiles)) return cdf_pick_tiles(sc, n, c.S, c.total, u, lane, tiles);
    return cdf_pick(sc, n, c.S, c.total, u, lane, c.car);
}
// (one draw: the same passes in one out-of-line call -- two calls here cost the per-walk kernels registers)
static __device__ __noinline__ int choose_index_long(float *sc, int n, float m, double u, int lane, double *tiles) {
    float S;
    double car[2], total;
    if (tiles && ((n + 31) >> 5) <= SC_CAP / 2) {
        S = softmax_exp_sum<8>(sc, n, m, lane);
        total = cdf_total_tiles(sc, n, S, lane, tiles);
        return cdf_pick_tiles(sc, n, S, total, u, lane, tiles);
    }
    S = softmax_exp_sum<8>(sc, n, m, lane);
    total = cdf_total<8>(sc, n, S, lane, car);
    return cdf_pick(sc, n, S, total, u, lane, car);
}

// softmax + CDF over sc[0..n) given its max m (n >= 2); `tiles`: see cdf_prepare_long (lists longer than SC_CAP)
__device__ __forceinline__ void cdf_prepare(float *sc, int n, float m, int lane, double *tiles, ListCdf &c) {
    if (n <= 32) {
        c.car[0] = tile1_cdf(sc, n, m, lane, c.total);
    } else if (n > SC_CAP) {
        cdf_prepare_long(sc, n, m, lane, tiles, c);
    } else {
        c.S = softmax_exp_sum(sc, n, m, lane);
        c.total = cdf_total(sc, n, c.S, lane, c.car);
    }
}

// the draw for uniform u from a prepared list.  All lanes return the index.
__device__ __forceinline__ int cdf_draw(const float *sc, int n, const ListCdf &c, double u, int lane, const double *tiles) {
    if (n <= 32) return tile1_pick(c.car[0], c.total, n, u, lane);
    if (n > SC_CAP) return cdf_draw_long(sc, n, c, u, lane, tiles);
    return cdf_pick(sc, n, c.S, c.total, u, lane, c.car);
}

// softmax + CDF + draw over sc[0..n) given its max m (== ggo_choose), n >= 2: a list drawn from once.  All lanes return
// the index.
__device__ __forceinline__ int choose_index(float *sc, int n, float m, double u, int lane, double *tiles = nullptr) {
    if (n <= 32) {
        double total;
        const double x = tile1_cdf(sc, n, m, lane, total);
        return tile1_pick(x, total, n, u, lane);
    }
    if (n > SC_CAP) return choose_index_long(sc, n, m, u, lane, tiles);
    double car[2];
    const float S = softmax_exp_sum(sc, n, m, lane);
    const double total = cdf_total(sc, n, S, lane, car);
    return cdf_pick(sc, n, S, total, u, lane, car);
}

// normalised CDF q_i = cdf_i / total written out (the array numpy's choice would searchsorted)
__device__ __forceinline__ void cdf_store(float *sc, int n, double *q_out, int lane) {
    const float m = list_max(sc, n, lane);
    const float S = softmax_exp_sum<UNR_S1>(sc, n, m, lane);
    double car[2];
    const double total = cdf_total<UNR_S1>(sc, n, S, lane, car);
    double carry = 0.0;
    for (int t0 = 0; t0 < n; t0 += 32) {
        const int i = t0 + lane;
        double x = (i < n) ? (double)__fdiv_rn(sc[i], S) : 0.0;
        x = warp_scan_ks(x, lane);
        if (i < n) q_out[i] = __ddiv_rn(__dadd_rn(carry, x), total);
        carry = __dadd_rn(carry, __shfl_sync(FULL, x, 31));
    }
}

// un-normalised CDF c_i = carry + scan(e/S)_i written out, the total after the n entries (c[n] = total).  One scan
// pass: the division by the total is left to the search, which performs it only on the entries it probes.
template <int U>
__device__ __forceinline__ void cdf_store_raw(float *sc, int n, float m, double *c_out, int lane) {
    const float S = softmax_exp_sum<U>(sc, n, m, lane);
    double carry = 0.0;
    for (int t0 = 0; t0 < n; t0 += 32 * U) {
        double x[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = t0 + 32 * u + lane;
            x[u] = (i < n) ? (double)__fdiv_rn(sc[i], S) : 0.0;   // 0 / S == 0 for the padding lanes
        }
#pragma unroll
        for (int u = 0; u < U; ++u) x[u] = warp_scan_ks(x[u], lane);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (t0 + 32 * u >= n) break;               // warp-uniform
            const int i = t0 + 32 * u + lane;
            if (i < n) c_out[i] = __dadd_rn(carry, x[u]);
            carry = __dadd_rn(carry, __shfl_sync(FULL, x[u], 31));
        }
    }
    if (lane == 0) c_out[n] = carry;
}

// first i in [0,n) with c[i] / c[n] > u: the same comparison as cdf_pick / cdf_search, on the raw array
__device__ __forceinline__ int cdf_search_raw(const double *__restrict__ c, int n, double u) {
    const double total = __ldg(c + n);
    int lo = 0, hi = n - 1;  // invariant: answer in [lo, hi]  (c[n-1] == total, so c[n-1] / total == 1 > u)
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ddiv_rn(__ldg(c + mid), total) > u) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// first i in [0,n) with q[i] > u (q non-decreasing, q[n-1] == 1 > u): what the linear scan finds
__device__ __forceinline__ int cdf_search(const double *__restrict__ q, int n, double u) {
    int lo = 0, hi = n - 1;  // invariant: answer in [lo, hi]
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(q + mid) > u) hi = mid; else lo = mid + 1;
    }
    return lo;
}

}  // namespace gg
