// value_gref.cu -- the exact expectation of the reference's generator step (DESIGN.md section 5.6).
//
// The reference's G pass (graph_gan.py:204-223, generator.py:22-31) takes every ordered pair within `window` of each
// walk's body and weights the pair's gradient by D's reward.  A G walk's body is the tree path root = a_0, ..., a_L = v
// (the path without the father it stops on), so it holds y exactly when the walk reaches y, with probability
//   reach(y) = fl(reach(father(y)) * pi_in(y)),  reach(root) = 1      (the section 5.1 chain, bit for bit)
// and for every reached y != root at depth delta(y) and d = 1 .. min(w, delta(y)), x = anc_d(y), the ordered pairs (x, y)
// and (y, x) each occur reach(y) times per walk.  Per pair (n1, n2), with the production bits:
//   r     = log(1 + exp(clip(s_D(n1, n2), +-10)))                         (gg_pair_reward)
//   kappa = -r (1 - p), p = sigmoid(s_G(n1, n2)); 0 when p < 1e-5f         (pair_delta mode 1, a_k = r, batch_total = 1)
// and the expected per-walk gradient adds rho kappa E_G[n2] to grad_E[n1], rho kappa E_G[n1] to grad_E[n2] and rho kappa to
// grad_b[n2] (rho = reach of the pair's deeper node).  kappa_up = kappa(x, y), kappa_dn = kappa(y, x) share one G dot and
// one D dot (the canonical fma chain is symmetric in its operands); each direction adds its own bias.
//
// Per chunk of roots: the recording section 5.1 kernel (gdist.cu); reach_kernel, top-down over the recorded levels;
// score_kernel, an 8-lane group per (item, d), writes kappa_up / kappa_dn into fp32 planes [w][R, N] indexed by the deeper
// node; npairs_kernel, a CTA per root; gather_kernel adds each root's contribution to each row.
//
// Order (the bits depend on the inputs only): a node's row takes the roots in the order given (WalkSampler sorts them by
// id), one fp64 chain per coordinate continued from the caller's accumulator.  A root's contribution to node a is
//   up + (((chain_0 + chain_1) + ...) + chain_7)
// where `up` runs over d = 1 .. min(w, delta(a)) (a as the deeper node) and chain_q, from +0, over the children of a at
// entries a0 + 256 (q + 8 m) + [0, 256) in entry order, each child followed by its reached descendants within w levels of
// a in depth-first pre-order, children in entry order (a as the ancestor).  A list of at most 256 entries has chain_0 only.
// Every term is one fma per coordinate with c = fl(rho * fl(kappa_up + kappa_dn)) (fp64), and one add of rho kappa for the
// bias.
//
// The second moment of one walk's step (DESIGN.md section 5.9, gg_expected_g_moments) runs the same stages and then:
// moment_kernel, an 8-lane group per item of depth >= 1, writes full(y) (the row depth(y) - w of y's path, complete
// whatever the walk does below y) and tail(y) (the rows depth(y) - w + 1 .. depth(y), truncated at y) in fp64 from the
// kappa planes and E_G rows of y's <= 2w ancestors; moment_prefix_kernel, top-down like reach_kernel, turns full into
// Pf(y) = Pf(father(y)) + full(y) and tail into |s(y)|^2 = Pf(y) + tail(y); root_sum_kernel gives sq_c = sum_y P(y)
// |s(y)|^2; gather_sq_kernel is gather_kernel that also stores each root's squared contribution to each row, and
// root_sum_kernel reduces that plane to mn_c = |m_c|^2.
//   row u (u levels above y): R = sum_v fl(kappa_up + kappa_dn) E_G[p_v] over the path nodes p_v within w of p_u, one
//   fp64 fma chain per coordinate from +0 in path order (v descending); B = the same chain of the kappas into p_u; a lane's
//   sum of R^2 over its coordinates gl, gl + 8, ... in order, then the group's xor butterfly 4, 2, 1; row = fl(R.R + B^2)
//   tail(y) = rows u = min(w - 1, depth(y)) .. 0 in that order from +0
#include <cooperative_groups.h>
#include <math.h>

#include "exact.cuh"
#include "update_dev.cuh"

namespace gg {
namespace {

namespace cg = cooperative_groups;

constexpr int GR_THREADS = 256;
constexpr int GR_CHAINS = GR_THREADS / 32;     // 8 chains, one per warp of a hub node's CTA
constexpr int GR_WMAX = 8;                     // the largest window

struct GrArgs {
    long long n_node, n_roots, tree_words, rn;
    int ld, window;
    const long long *indptr;
    const int *adj, *roots, *ok;
    const uint32_t *tree_bits;
    const float *emb, *bias, *d_emb, *d_bias;
    const double *pi_in;
    double *reach;
    const int *father;
    const int4 *items;
    const unsigned *lev_off, *n_lev;
    float *kup, *kdn;                          // [window][n_roots, n_node]: kappa(anc_d(y), y), kappa(y, anc_d(y))
    int *big;
    unsigned *big_cnt;
    double *n_pairs, *grad_emb, *grad_bias;
};

// top-down over the recorded levels, a thread per item, one grid barrier per level
__global__ void __launch_bounds__(GR_THREADS) reach_kernel(const GrArgs g) {
    cg::grid_group grid = cg::this_grid();
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
    const int n_lev = (int)*g.n_lev;
    for (int lev = 0; lev < n_lev; ++lev) {
        const long long i0 = g.lev_off[lev], i1 = g.lev_off[lev + 1];
        for (long long i = i0 + tid; i < i1; i += nt) {
            const int4 it = g.items[i];
            if (__ldg(g.ok + it.x) != 1) continue;
            const size_t o = (size_t)it.x * (size_t)g.n_node;
            g.reach[o + it.y] = it.z < 0 ? 1.0 : __dmul_rn(g.reach[o + it.z], g.pi_in[o + it.y]);
        }
        grid.sync();
    }
}

// the production reward and G coefficient of one pair from its dots (pairs.cu reward_kernel, update_dev.cuh pair_delta)
__device__ __forceinline__ float pair_kappa(float dot_g, float b_g, float dot_d, float b_d) {
    float sd = __fadd_rn(dot_d, b_d);
    sd = fminf(fmaxf(sd, -10.0f), 10.0f);
    const float r = logf(1.0f + expf(sd));
    const float s = __fadd_rn(dot_g, b_g);
    const float p = (float)(1.0 / (1.0 + exp(-(double)s)));
    return (p >= 1e-5f) ? __fmul_rn(-r, __fsub_rn(1.0f, p)) : 0.0f;
}

// an 8-lane group per (item of depth >= 1, d): the canonical group dots of (anc_d(y), y) under G and D
__global__ void __launch_bounds__(GR_THREADS) score_kernel(const GrArgs g) {
    const int lane = threadIdx.x & 31, grp = lane >> 3, gl = lane & 7;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((long long)gridDim.x * blockDim.x) >> 5;
    const long long i0 = g.lev_off[1 < *g.n_lev ? 1 : *g.n_lev], i1 = g.lev_off[*g.n_lev];
    const int per_item = (g.window + 3) / 4;                  // passes of 4 groups per item
    for (long long w0 = gw; w0 < (i1 - i0) * per_item; w0 += nw) {
        const int4 it = g.items[i0 + w0 / per_item];
        const int d = (int)(w0 % per_item) * 4 + grp + 1;
        const size_t o = (size_t)it.x * (size_t)g.n_node;
        const int y = it.y;
        int x = -1;
        if (__ldg(g.ok + it.x) == 1 && d <= g.window) {
            x = it.z;
            for (int k = 1; k < d && x >= 0; ++k) x = g.father[o + x];
        }
        const int xx = x >= 0 ? x : y;                         // x < 0: y is shallower than d (the dots are warp-wide)
        const float dg = group_dot_t<false>(g.emb + (size_t)xx * g.ld, g.emb + (size_t)y * g.ld, g.ld, gl);
        const float dd = group_dot_t<false>(g.d_emb + (size_t)xx * g.ld, g.d_emb + (size_t)y * g.ld, g.ld, gl);
        if (x < 0 || gl != 0) continue;
        const size_t at = (size_t)(d - 1) * (size_t)g.rn + o + y;
        g.kup[at] = pair_kappa(dg, __ldg(g.bias + y), dd, __ldg(g.d_bias + y));
        g.kdn[at] = pair_kappa(dg, __ldg(g.bias + x), dd, __ldg(g.d_bias + x));
    }
}

// min(w, depth of v) in root slot o (0 for the root and for nodes not reached)
__device__ __forceinline__ int window_depth(const GrArgs &g, size_t o, int v) {
    int x = g.father[o + v], m = 0;
    while (x >= 0 && m < g.window) {
        ++m;
        x = g.father[o + x];
    }
    return m;
}

// n_pairs[k] = sum_v reach(v) 2 min(w, depth(v)): thread t chains v = t, t + 256, ..., then the warps' butterflies in
// warp order
__global__ void __launch_bounds__(GR_THREADS) npairs_kernel(const GrArgs g) {
    __shared__ double s_w[GR_CHAINS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (long long k = blockIdx.x; k < g.n_roots; k += gridDim.x) {
        double s = 0.0;
        if (__ldg(g.ok + k) == 1) {
            const size_t o = (size_t)k * (size_t)g.n_node;
            for (long long v = threadIdx.x; v < g.n_node; v += GR_THREADS) {
                const int m = window_depth(g, o, (int)v);
                if (m) s = __dadd_rn(s, __dmul_rn(g.reach[o + v], (double)(2 * m)));
            }
        }
        s = warp_dsum(s);
        if (lane == 0) s_w[wid] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = s_w[0];
            for (int q = 1; q < GR_CHAINS; ++q) t = __dadd_rn(t, s_w[q]);
            g.n_pairs[k] = t;
        }
        __syncthreads();
    }
}

// the pair coefficient c = rho (kappa_up + kappa_dn) of (anc_d(y), y) and the bias term of its node side
__device__ __forceinline__ double pair_coef(const GrArgs &g, size_t o, int y, int d, double &rho) {
    const size_t at = (size_t)(d - 1) * (size_t)g.rn + o + y;
    rho = g.reach[o + y];
    return __dmul_rn(rho, __dadd_rn((double)g.kup[at], (double)g.kdn[at]));
}

// chain_q of node a in root slot o (see the top of the file): s[i] for coordinate lane + 32 i, sb for the bias.  A
// warp-uniform depth-first walk: frame t holds a node at distance t from a, the window of 32 of its entries being visited
// (mask: the reached children not yet taken) and the next window.
template <int CPL>
__device__ __forceinline__ void down_chain(const GrArgs &g, size_t o, const uint32_t *tb, int a, long long a0, long long a1,
                                           int q, int lane, double (&s)[CPL], double &sb) {
    constexpr int LD = 32 * CPL;
#pragma unroll
    for (int i = 0; i < CPL; ++i) s[i] = 0.0;
    sb = 0.0;
    int nd[GR_WMAX];
    long long nxt[GR_WMAX], end[GR_WMAX], base[GR_WMAX];
    unsigned msk[GR_WMAX];
    for (long long b0 = a0 + CHAIN_BLOCK * q; b0 < a1; b0 += CHAIN_BLOCK * GR_CHAINS) {
        int top = 0;
        nd[0] = a; nxt[0] = b0; end[0] = b0 + CHAIN_BLOCK < a1 ? b0 + CHAIN_BLOCK : a1; msk[0] = 0u; base[0] = b0;
        while (true) {
            if (msk[top] == 0u) {
                if (nxt[top] >= end[top]) {
                    if (top == 0) break;
                    --top;
                    continue;
                }
                const long long e = nxt[top] + lane;
                bool take = false;
                if (e < end[top] && tree_bit(tb, e)) take = g.father[o + __ldg(g.adj + e)] == nd[top];
                msk[top] = __ballot_sync(FULL, take);
                base[top] = nxt[top];
                nxt[top] += 32;
                continue;
            }
            const int bit = __ffs(msk[top]) - 1;
            msk[top] &= msk[top] - 1u;
            const int y = __ldg(g.adj + base[top] + bit);
            const int dist = top + 1;
            double rho;
            const double c = pair_coef(g, o, y, dist, rho);
            sb = __dadd_rn(sb, __dmul_rn(rho, (double)g.kdn[(size_t)(dist - 1) * (size_t)g.rn + o + y]));
#pragma unroll
            for (int i = 0; i < CPL; ++i) s[i] = __fma_rn(c, (double)__ldg(g.emb + (size_t)y * LD + lane + 32 * i), s[i]);
            if (dist < g.window) {
                ++top;
                nd[top] = y; nxt[top] = __ldg(g.indptr + y); end[top] = __ldg(g.indptr + y + 1); msk[top] = 0u;
                base[top] = nxt[top];
            }
        }
    }
}

// Work items: first one CTA per big node, then groups of 8 nodes, a warp per node (big nodes skipped).  Each item runs
// the roots in order and stores its rows once.  SQ: also mnp[k, a] = |root k's contribution to row a|^2 (coordinates,
// then the bias squared), with a fixed block reduction on the big-node path; the caller clears mnp.
template <int CPL, bool SQ>
__device__ __forceinline__ void gather_rows(const GrArgs &g, double *mnp) {
    constexpr int LD = 32 * CPL;
    extern __shared__ __align__(16) unsigned char gr_smem[];
    double *s_ch = reinterpret_cast<double *>(gr_smem);   // [GR_CHAINS, LD] chain sums, then [GR_CHAINS] bias chains
    double *s_chb = s_ch + GR_CHAINS * LD;
    double *s_sq = s_chb + GR_CHAINS;                      // SQ: [GR_CHAINS] warp partials of the squared contribution
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long n_big = *g.big_cnt, n_groups = (g.n_node + GR_CHAINS - 1) / GR_CHAINS;
    for (long long item = blockIdx.x; item < n_big + n_groups; item += gridDim.x) {
        if (item < n_big) {
            // ---- a big node: warp q runs chain_q; thread t owns coordinates t, t + 256
            const int a = g.big[item];
            const long long a0 = __ldg(g.indptr + a), a1 = __ldg(g.indptr + a + 1);
            double acc[2], accb = 0.0;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int j = threadIdx.x + GR_THREADS * r;
                acc[r] = j < LD ? g.grad_emb[(size_t)a * LD + j] : 0.0;
            }
            if (threadIdx.x == 0) accb = g.grad_bias[a];
            for (long long k = 0; k < g.n_roots; ++k) {
                if (__ldg(g.ok + k) != 1) continue;
                const size_t o = (size_t)k * (size_t)g.n_node;
                const bool is_root = __ldg(g.roots + k) == a;
                if (!is_root && g.father[o + a] < 0) continue;                 // not reached from this root
                double s[CPL], sb;
                down_chain<CPL>(g, o, g.tree_bits + (size_t)k * (size_t)g.tree_words, a, a0, a1, wid, lane, s, sb);
#pragma unroll
                for (int i = 0; i < CPL; ++i) s_ch[wid * LD + lane + 32 * i] = s[i];
                if (lane == 0) s_chb[wid] = sb;
                __syncthreads();
                double up[2] = {0.0, 0.0}, upb = 0.0;
                int x = is_root ? -1 : g.father[o + a];
                for (int d = 1; d <= g.window && x >= 0; ++d) {
                    double rho;
                    const double c = pair_coef(g, o, a, d, rho);
                    upb = __dadd_rn(upb, __dmul_rn(rho, (double)g.kup[(size_t)(d - 1) * (size_t)g.rn + o + a]));
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int j = threadIdx.x + GR_THREADS * r;
                        if (j < LD) up[r] = __fma_rn(c, (double)__ldg(g.emb + (size_t)x * LD + j), up[r]);
                    }
                    x = g.father[o + x];
                }
                double qs = 0.0, cb = 0.0;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int j = threadIdx.x + GR_THREADS * r;
                    if (j >= LD) continue;
                    double ch = s_ch[j];
                    for (int q = 1; q < GR_CHAINS; ++q) ch = __dadd_rn(ch, s_ch[q * LD + j]);
                    const double cr = __dadd_rn(up[r], ch);
                    acc[r] = __dadd_rn(acc[r], cr);
                    if (SQ) qs = __fma_rn(cr, cr, qs);
                }
                if (SQ) {
                    qs = warp_dsum(qs);
                    if (lane == 0) s_sq[wid] = qs;
                }
                if (threadIdx.x == 0) {
                    double chb = s_chb[0];
                    for (int q = 1; q < GR_CHAINS; ++q) chb = __dadd_rn(chb, s_chb[q]);
                    cb = __dadd_rn(upb, chb);
                    accb = __dadd_rn(accb, cb);
                }
                __syncthreads();
                if (SQ && threadIdx.x == 0) {       // s_sq is next written after the next root's first barrier
                    double t = s_sq[0];
                    for (int w = 1; w < GR_CHAINS; ++w) t = __dadd_rn(t, s_sq[w]);
                    mnp[o + a] = __dadd_rn(t, __dmul_rn(cb, cb));
                }
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int j = threadIdx.x + GR_THREADS * r;
                if (j < LD) g.grad_emb[(size_t)a * LD + j] = acc[r];
            }
            if (threadIdx.x == 0) g.grad_bias[a] = accb;
            continue;
        }
        // ---- a group of 8 nodes, a warp per node: chain_0 only
        const long long a = (item - n_big) * GR_CHAINS + wid;
        if (a >= g.n_node) continue;
        const long long a0 = __ldg(g.indptr + a), a1 = __ldg(g.indptr + a + 1);
        if (a1 - a0 > CHAIN_BLOCK) continue;
        double acc[CPL];
#pragma unroll
        for (int i = 0; i < CPL; ++i) acc[i] = g.grad_emb[(size_t)a * LD + lane + 32 * i];
        double accb = g.grad_bias[a];
        for (long long k = 0; k < g.n_roots; ++k) {
            if (__ldg(g.ok + k) != 1) continue;
            const size_t o = (size_t)k * (size_t)g.n_node;
            const bool is_root = __ldg(g.roots + k) == (int)a;
            if (!is_root && g.father[o + a] < 0) continue;
            double s[CPL], sb;
            down_chain<CPL>(g, o, g.tree_bits + (size_t)k * (size_t)g.tree_words, (int)a, a0, a1, 0, lane, s, sb);
            double up[CPL], upb = 0.0;
#pragma unroll
            for (int i = 0; i < CPL; ++i) up[i] = 0.0;
            int x = is_root ? -1 : g.father[o + a];
            for (int d = 1; d <= g.window && x >= 0; ++d) {
                double rho;
                const double c = pair_coef(g, o, (int)a, d, rho);
                upb = __dadd_rn(upb, __dmul_rn(rho, (double)g.kup[(size_t)(d - 1) * (size_t)g.rn + o + a]));
#pragma unroll
                for (int i = 0; i < CPL; ++i) up[i] = __fma_rn(c, (double)__ldg(g.emb + (size_t)x * LD + lane + 32 * i), up[i]);
                x = g.father[o + x];
            }
            double qs = 0.0;
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
                const double ci = __dadd_rn(up[i], s[i]);
                acc[i] = __dadd_rn(acc[i], ci);
                if (SQ) qs = __fma_rn(ci, ci, qs);
            }
            const double cb = __dadd_rn(upb, sb);
            accb = __dadd_rn(accb, cb);
            if (SQ) {
                qs = warp_dsum(qs);
                if (lane == 0) mnp[o + a] = __dadd_rn(qs, __dmul_rn(cb, cb));
            }
        }
#pragma unroll
        for (int i = 0; i < CPL; ++i) g.grad_emb[(size_t)a * LD + lane + 32 * i] = acc[i];
        if (lane == 0) g.grad_bias[a] = accb;
    }
}

template <int CPL>
__global__ void __launch_bounds__(GR_THREADS) gather_kernel(const GrArgs g) { gather_rows<CPL, false>(g, nullptr); }

template <int CPL>
__global__ void __launch_bounds__(GR_THREADS) gather_sq_kernel(const GrArgs g, double *mnp) { gather_rows<CPL, true>(g, mnp); }

// gather_kernel, or gather_sq_kernel when mnp is given
int gather(const GrArgs &g, double *mnp, cudaStream_t st) {
    return with_cpl(g.ld, [&](auto c) {
        const size_t smem = (size_t)GR_CHAINS * (32 * c + (mnp ? 2 : 1)) * sizeof(double);
        const void *fn = mnp ? (const void *)gather_sq_kernel<c> : (const void *)gather_kernel<c>;
        GG_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const long long n_groups = (g.n_node + GR_CHAINS - 1) / GR_CHAINS;
        unsigned grid = 0;
        int rc = fill_grid(fn, GR_THREADS, smem, n_groups + g.n_node, "expected G step gather", &grid);
        if (rc) return rc;
        if (mnp)
            gather_sq_kernel<c><<<grid, GR_THREADS, smem, st>>>(g, mnp);
        else
            gather_kernel<c><<<grid, GR_THREADS, smem, st>>>(g);
        return check_cuda(cudaGetLastError(), "expected G step gather launch");
    });
}

// ---- section 5.9: the second moment of one walk's step
struct GmArgs {
    GrArgs g;
    const double *dist;                        // the stop law P(y)
    double *pf;                                // [n_roots, n_node]: full(y), then Pf(y); later gather_sq_kernel's plane
    double *sqn;                               // [n_roots, n_node]: tail(y), then |s(y)|^2 (0 at the root and unreached)
};

constexpr int GM_PATH = 2 * GR_WMAX + 1;       // y and its ancestors up to 2w levels above it

// fl(R.R + B^2) of row u of y's path (p[v]: the node v levels above y, v <= lc = min(depth(y), 2w)); see the top of the
// file.  The pair (p_v, p_u) has its kappa planes at its deeper node, distance |u - v|.
__device__ __forceinline__ double path_row(const GrArgs &g, size_t o, const int (&p)[GM_PATH], int u, int lc, int gl,
                                           unsigned gmask) {
    const int lo = u > g.window ? u - g.window : 0, hi = u + g.window < lc ? u + g.window : lc;
    int pu = p[0];
#pragma unroll
    for (int v = 1; v < GM_PATH; ++v)
        if (v == u) pu = p[v];
    double cf[GM_PATH], b = 0.0;
    unsigned live = 0u;
#pragma unroll
    for (int v = GM_PATH - 1; v >= 0; --v) {
        cf[v] = 0.0;
        if (v < lo || v > hi || v == u) continue;
        live |= 1u << v;
        const int deep = v < u ? p[v] : pu;
        const size_t at = (size_t)((v < u ? u - v : v - u) - 1) * (size_t)g.rn + o + deep;
        const float ku = g.kup[at], kd = g.kdn[at];
        cf[v] = __dadd_rn((double)ku, (double)kd);
        b = __dadd_rn(b, (double)(v < u ? kd : ku));      // kappa(p_v, p_u)
    }
    double q = 0.0;
    for (int c = gl; c < g.ld; c += 8) {
        double r = 0.0;
#pragma unroll
        for (int v = GM_PATH - 1; v >= 0; --v)
            if (live >> v & 1u) r = __fma_rn(cf[v], (double)__ldg(g.emb + (size_t)p[v] * g.ld + c), r);
        q = __fma_rn(r, r, q);
    }
#pragma unroll
    for (int off = 4; off >= 1; off >>= 1) q = __dadd_rn(q, __shfl_xor_sync(gmask, q, off));
    return __dadd_rn(q, __dmul_rn(b, b));
}

// an 8-lane group per item of depth >= 1: pf = full(y), sqn = tail(y)
__global__ void __launch_bounds__(GR_THREADS) moment_kernel(const GmArgs m) {
    const GrArgs &g = m.g;
    const int lane = threadIdx.x & 31, gl = lane & 7;
    const unsigned gmask = 0xffu << (lane & 24);
    const long long gid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3, ng = ((long long)gridDim.x * blockDim.x) >> 3;
    const long long i0 = g.lev_off[1 < *g.n_lev ? 1 : *g.n_lev], i1 = g.lev_off[*g.n_lev];
    for (long long i = i0 + gid; i < i1; i += ng) {
        const int4 it = g.items[i];
        if (__ldg(g.ok + it.x) != 1) continue;
        const size_t o = (size_t)it.x * (size_t)g.n_node;
        int p[GM_PATH], lc = 0;
        p[0] = it.y;
#pragma unroll
        for (int v = 1; v < GM_PATH; ++v) {
            p[v] = (v <= 2 * g.window && p[v - 1] >= 0) ? (v == 1 ? it.z : g.father[o + p[v - 1]]) : -1;
            if (p[v] >= 0) lc = v;
        }
        const double full = lc >= g.window ? path_row(g, o, p, g.window, lc, gl, gmask) : 0.0;
        double tail = 0.0;
        for (int u = g.window - 1 < lc ? g.window - 1 : lc; u >= 0; --u) tail = __dadd_rn(tail, path_row(g, o, p, u, lc, gl, gmask));
        if (gl == 0) {
            m.pf[o + it.y] = full;
            m.sqn[o + it.y] = tail;
        }
    }
}

// top-down over the recorded levels (reach_kernel's shape): Pf(y) = Pf(father) + full(y), |s(y)|^2 = Pf(y) + tail(y)
__global__ void __launch_bounds__(GR_THREADS) moment_prefix_kernel(const GmArgs m) {
    cg::grid_group grid = cg::this_grid();
    const GrArgs &g = m.g;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
    const int n_lev = (int)*g.n_lev;
    for (int lev = 1; lev < n_lev; ++lev) {
        const long long i0 = g.lev_off[lev], i1 = g.lev_off[lev + 1];
        for (long long i = i0 + tid; i < i1; i += nt) {
            const int4 it = g.items[i];
            if (__ldg(g.ok + it.x) != 1) continue;
            const size_t o = (size_t)it.x * (size_t)g.n_node;
            const double pf = __dadd_rn(m.pf[o + it.z], m.pf[o + it.y]);
            m.pf[o + it.y] = pf;
            m.sqn[o + it.y] = __dadd_rn(pf, m.sqn[o + it.y]);
        }
        grid.sync();
    }
}

// out[k] = sum_v fl(w[k, v] x[k, v]) (w null: sum_v x[k, v]) over an ok root's nodes in npairs_kernel's order; 0 else
__global__ void __launch_bounds__(GR_THREADS) root_sum_kernel(const GrArgs g, const double *w, const double *x, double *out) {
    __shared__ double s_w[GR_CHAINS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (long long k = blockIdx.x; k < g.n_roots; k += gridDim.x) {
        double s = 0.0;
        if (__ldg(g.ok + k) == 1) {
            const size_t o = (size_t)k * (size_t)g.n_node;
            for (long long v = threadIdx.x; v < g.n_node; v += GR_THREADS)
                s = __dadd_rn(s, w ? __dmul_rn(w[o + v], x[o + v]) : x[o + v]);
        }
        s = warp_dsum(s);
        if (lane == 0) s_w[wid] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = s_w[0];
            for (int q = 1; q < GR_CHAINS; ++q) t = __dadd_rn(t, s_w[q]);
            out[k] = t;
        }
        __syncthreads();
    }
}

struct GrLayout {
    void *rec;                                 // gdist_rec_layout's part
    double *dist, *reach, *pi_in, *pi_stop;
    float *kup, *kdn;
    int *father, *root_ok, *big;
    unsigned *big_cnt;
    double *pf, *sqn;                          // moments only
};

size_t gr_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, int window, bool moments, GrLayout *v) {
    const size_t rn = (size_t)n_roots * (size_t)n_node;
    Slab s(buf);
    GrLayout t;
    t.rec = s.take<unsigned char>(gdist_rec_layout(nullptr, n_node, nnz_words, n_roots, nullptr));
    t.dist = s.take<double>(rn);
    t.reach = s.take<double>(rn);
    t.pi_in = s.take<double>(rn);
    t.pi_stop = s.take<double>(rn);
    t.kup = s.take<float>((size_t)window * rn);
    t.kdn = s.take<float>((size_t)window * rn);
    t.father = s.take<int>(rn);
    t.root_ok = s.take<int>((size_t)n_roots);
    t.big = s.take<int>((size_t)n_node);
    t.big_cnt = s.take<unsigned>(1);
    t.pf = moments ? s.take<double>(rn) : nullptr;
    t.sqn = moments ? s.take<double>(rn) : nullptr;
    if (buf && v) *v = t;
    return s.off;
}

struct GmOut {
    double *sq, *mn, *sq_node;
};

// gg_expected_g_grad's launch sequence; with mo, also gg_expected_g_moments' stages
int expected_g_run(const gg_walk_desc *gp, const float *d_emb, const float *d_bias, int32_t window, double *n_pairs,
                   int32_t *root_ok, double *grad_emb, double *grad_bias, void *scratch, int64_t scratch_bytes, void *stream,
                   const GmOut *mo) {
    GG_REQUIRE(window >= 1 && window <= GR_WMAX, "window must be 1 .. 8");
    int rc = check_law_desc(gp);
    if (rc || gp->n_roots == 0) return rc;
    const gg_walk_desc &d = *gp;
    GG_REQUIRE(d_emb && d_bias, "null discriminator pointer");
    GG_REQUIRE(n_pairs && root_ok && grad_emb && grad_bias && scratch, "null output or scratch pointer");
    GG_REQUIRE(!mo || (mo->sq && mo->mn), "null sq / mn pointer");
    GrLayout v;
    const size_t need = gr_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, window, mo != nullptr, &v);
    GG_REQUIRE(scratch_bytes >= (int64_t)need, mo ? "scratch too small (gg_expected_g_moments_scratch_bytes)"
                                                  : "scratch too small (gg_expected_g_grad_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t rn = (size_t)d.n_roots * (size_t)d.n_node;
    GG_CHECK(cudaMemsetAsync(v.dist, 0, rn * sizeof(double), st));
    GG_CHECK(cudaMemsetAsync(root_ok, 0, (size_t)d.n_roots * sizeof(int32_t), st));
    GG_CHECK(cudaMemsetAsync(v.father, 0xff, rn * sizeof(int), st));
    GG_CHECK(cudaMemsetAsync(v.big_cnt, 0, sizeof(unsigned), st));
    GdRec rec;
    rec.pi_in = v.pi_in; rec.pi_stop = v.pi_stop; rec.father = v.father;
    gdist_rec_layout(v.rec, d.n_node, d.tree_words - 1, d.n_roots, &rec);
    rc = gdist_rec_launch(d, v.dist, root_ok, rec, v.rec, st);
    if (rc) return rc;
    GrArgs g;
    g.n_node = d.n_node; g.n_roots = d.n_roots; g.tree_words = d.tree_words; g.rn = (long long)rn;
    g.ld = d.ld; g.window = window;
    g.indptr = (const long long *)d.indptr; g.adj = d.adj; g.roots = d.roots; g.ok = root_ok; g.tree_bits = d.tree_bits;
    g.emb = d.emb; g.bias = d.bias; g.d_emb = d_emb; g.d_bias = d_bias;
    g.pi_in = v.pi_in; g.reach = v.reach; g.father = v.father;
    g.items = rec.items; g.lev_off = rec.lev_off; g.n_lev = rec.n_lev;
    g.kup = v.kup; g.kdn = v.kdn; g.big = v.big; g.big_cnt = v.big_cnt;
    g.n_pairs = n_pairs; g.grad_emb = grad_emb; g.grad_bias = grad_bias;
    void *args[] = {(void *)&g};
    rc = coop_launch((const void *)reach_kernel, GR_THREADS, 0, 0, args, st, "expected G step reach");
    if (rc) return rc;
    score_kernel<<<(unsigned)(sm_count() * 8), GR_THREADS, 0, st>>>(g);
    GG_CHECK(cudaGetLastError());
    const unsigned root_grid = (unsigned)(d.n_roots < sm_count() * 4 ? d.n_roots : sm_count() * 4);
    npairs_kernel<<<root_grid, GR_THREADS, 0, st>>>(g);
    GG_CHECK(cudaGetLastError());
    rc = big_nodes_launch(d.n_node, g.indptr, v.big, v.big_cnt, st);
    if (rc) return rc;
    if (!mo) return gather(g, nullptr, st);
    GmArgs m;
    m.g = g; m.dist = v.dist; m.pf = v.pf; m.sqn = mo->sq_node ? mo->sq_node : v.sqn;
    GG_CHECK(cudaMemsetAsync(m.pf, 0, rn * sizeof(double), st));
    GG_CHECK(cudaMemsetAsync(m.sqn, 0, rn * sizeof(double), st));
    moment_kernel<<<(unsigned)(sm_count() * 8), GR_THREADS, 0, st>>>(m);
    GG_CHECK(cudaGetLastError());
    void *margs[] = {(void *)&m};
    rc = coop_launch((const void *)moment_prefix_kernel, GR_THREADS, 0, 0, margs, st, "expected G moments prefix");
    if (rc) return rc;
    root_sum_kernel<<<root_grid, GR_THREADS, 0, st>>>(g, m.dist, m.sqn, mo->sq);
    GG_CHECK(cudaGetLastError());
    GG_CHECK(cudaMemsetAsync(m.pf, 0, rn * sizeof(double), st));             // Pf is spent: the plane of mn's terms
    rc = gather(g, m.pf, st);
    if (rc) return rc;
    root_sum_kernel<<<root_grid, GR_THREADS, 0, st>>>(g, nullptr, m.pf, mo->mn);
    return check_cuda(cudaGetLastError(), "expected G moments mn launch");
}

}  // namespace
}  // namespace gg

extern "C" int gg_expected_g_grad_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int32_t window,
                                                int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0 && n_roots >= 0, "bad arguments");
    GG_REQUIRE(window >= 1 && window <= gg::GR_WMAX, "window must be 1 .. 8");
    *bytes = (int64_t)gg::gr_layout(nullptr, n_node, (nnz + 31) / 32, n_roots, window, false, nullptr);
    return 0;
}

extern "C" int gg_expected_g_grad(const gg_walk_desc *gp, const float *d_emb, const float *d_bias, int32_t window,
                                  double *n_pairs, int32_t *root_ok, double *grad_emb, double *grad_bias, void *scratch,
                                  int64_t scratch_bytes, void *stream) {
    return gg::expected_g_run(gp, d_emb, d_bias, window, n_pairs, root_ok, grad_emb, grad_bias, scratch, scratch_bytes,
                              stream, nullptr);
}

extern "C" int gg_expected_g_moments_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int32_t window,
                                                   int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0 && n_roots >= 0, "bad arguments");
    GG_REQUIRE(window >= 1 && window <= gg::GR_WMAX, "window must be 1 .. 8");
    *bytes = (int64_t)gg::gr_layout(nullptr, n_node, (nnz + 31) / 32, n_roots, window, true, nullptr);
    return 0;
}

extern "C" int gg_expected_g_moments(const gg_walk_desc *gp, const float *d_emb, const float *d_bias, int32_t window,
                                     double *n_pairs, int32_t *root_ok, double *sq, double *mn, double *sq_node,
                                     double *grad_emb, double *grad_bias, void *scratch, int64_t scratch_bytes, void *stream) {
    const gg::GmOut mo{sq, mn, sq_node};
    return gg::expected_g_run(gp, d_emb, d_bias, window, n_pairs, root_ok, grad_emb, grad_bias, scratch, scratch_bytes,
                              stream, &mo);
}
