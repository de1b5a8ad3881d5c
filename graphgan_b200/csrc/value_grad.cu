// value_grad.cu -- the exact generator gradient of the game value, grad_G sum_c V_c(G, D) (DESIGN.md section 5.3).
//
// Per root c with ok_c = 1, G the section 5.1 law (pi the exact step law of each list) and
//   h(v)    = G(v | c) * bce(s_D(c, v), 0)                 (the products value_kernel adds into neg_c = -sum_v h(v))
//   T(a)    = h(a) + sum_{children x} T(x)                 (sum of h over the subtree of a)
//   w_a(x)  = F_a(x) - pi_a(x) T(a),  F_a(x) = T(x) for a child x, F_a(father(a)) = h(a)
// the score s(a, x) = E_G[a] . E_G[x] + b_G[x] of candidate x in a's list has d neg_c / d s(a, x) = -w_a(x), so for every
// tree edge e = (a, child x), c_e = w_a(x) + w_x(a) (w_x(a) = 0 when x's father entry is removed):
//   grad_E[a] -= c_e E_G[x],  grad_E[x] -= c_e E_G[a],  grad_b[x] -= w_a(x),  grad_b[a] -= w_x(a)
// and grad_G V_c = grad_G neg_c (pos_c does not depend on G).
//
// Per chunk of roots: the recording section 5.1 kernel (gdist.cu: dist, and per (root, node) pi_in = pi_father(node),
// pi_stop = pi_node(father), father, every level's items); gg_game_value on that dist (pos / neg / ok); h (value.cu);
// tsum_kernel, bottom-up over the recorded levels, turns (pi_in, pi_stop) of every reached node x into
// (w_in, w_stop) = (w_father(x)(x), w_x(father(x))); gather_kernel adds each root's contribution to each row.
//
// Order (the bits depend on the inputs only): a node's row takes the roots in the order given (WalkSampler sorts them by
// id), one fp64 chain per coordinate continued from the caller's accumulator.  A root's contribution to node a is
//   (father term) + (((chain_0 + chain_1) + ...) + chain_7)
// where chain_q runs, in entry order from +0, over the children at entries a0 + 256 (q + 8 m) + [0, 256): a list of at most
// 256 entries has chain_0 only, a hub's 13 828 entries are eight chains (one warp each) instead of one warp's serial tail.
#include <cooperative_groups.h>
#include <math.h>

#include "exact.cuh"

namespace gg {
namespace {

namespace cg = cooperative_groups;

constexpr int VG_THREADS = 256;
constexpr int VG_CHAINS = VG_THREADS / 32;     // 8 chains, one per warp of a hub node's CTA

struct VgArgs {
    long long n_node, n_roots, tree_words;
    int ld;
    const long long *indptr;
    const int *adj, *roots, *ok;
    const uint32_t *tree_bits;
    const float *emb;
    const double *h;
    double *T, *w_in, *w_stop;                 // w_in / w_stop: pi_in / pi_stop until tsum_kernel rewrites them
    const int *father;
    const int4 *items;
    const unsigned *lev_off, *n_lev;
    int *big;                                  // [n_node]: nodes with more than CHAIN_BLOCK entries; big_cnt: their number
    unsigned *big_cnt;
    double *grad_emb, *grad_bias;
};

// one item (slot, a) of the bottom-up pass: T(a), then (w_in, w_stop) of a's reached children
__device__ void tsum_item(const VgArgs &g, const int4 it, int lane) {
    const int slot = it.x, a = it.y;
    if (__ldg(g.ok + slot) != 1) return;
    const size_t o = (size_t)slot * (size_t)g.n_node;
    const uint32_t *tb = g.tree_bits + (size_t)slot * (size_t)g.tree_words;
    const long long a0 = __ldg(g.indptr + a), a1 = __ldg(g.indptr + a + 1);
    // T(a) = h(a) + sum of the children's T: lane l chains entries a0 + l, a0 + l + 32, ..., then a xor butterfly (T is 0
    // for nodes that are not reached)
    double s = 0.0;
    for (long long e = a0 + lane; e < a1; e += 32)
        if (tree_bit(tb, e)) s = __dadd_rn(s, g.T[o + (size_t)__ldg(g.adj + e)]);
    const double Ta = __dadd_rn(g.h[o + a], warp_dsum(s));
    if (lane == 0) g.T[o + a] = Ta;
    for (long long e = a0 + lane; e < a1; e += 32) {
        if (!tree_bit(tb, e)) continue;
        const int x = __ldg(g.adj + e);
        if (g.father[o + x] != a) continue;                  // not reached: every w of x is 0
        const double Tx = g.T[o + x];
        g.w_in[o + x] = __dsub_rn(Tx, __dmul_rn(g.w_in[o + x], Ta));                // w_a(x) = T(x) - pi_a(x) T(a)
        g.w_stop[o + x] = __dsub_rn(g.h[o + x], __dmul_rn(g.w_stop[o + x], Tx));    // w_x(a) = h(x) - pi_x(a) T(x)
    }
}

// deepest level first, a warp per item, one grid barrier per level
__global__ void __launch_bounds__(VG_THREADS) tsum_kernel(const VgArgs g) {
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((long long)gridDim.x * blockDim.x) >> 5;
    const int n_lev = (int)*g.n_lev;
    for (int lev = n_lev - 1; lev >= 0; --lev) {
        const long long i0 = g.lev_off[lev], i1 = g.lev_off[lev + 1];
        for (long long i = i0 + gw; i < i1; i += nw) tsum_item(g, g.items[i], lane);
        grid.sync();
    }
}

// chain_q of node a in root slot k (see the top of the file): s[i] for coordinate lane + 32 i, sb for the bias.  The
// children's (x, c_e, w_x(a)) are broadcast from the lanes that found them; four rows are in flight.
template <int CPL>
__device__ __forceinline__ void child_chain(const VgArgs &g, size_t o, const uint32_t *tb, int a, long long a0, long long a1,
                                            int q, int lane, double (&s)[CPL], double &sb) {
    constexpr int LD = 32 * CPL;
#pragma unroll
    for (int i = 0; i < CPL; ++i) s[i] = 0.0;
    sb = 0.0;
    for (long long b0 = a0 + CHAIN_BLOCK * q; b0 < a1; b0 += CHAIN_BLOCK * VG_CHAINS) {
        const long long b1 = b0 + CHAIN_BLOCK < a1 ? b0 + CHAIN_BLOCK : a1;
        for (long long e0 = b0; e0 < b1; e0 += 32) {
            const long long e = e0 + lane;
            int x = -1;
            double cx = 0.0, wx = 0.0;
            if (e < b1 && tree_bit(tb, e)) {
                x = __ldg(g.adj + e);
                if (g.father[o + x] == a) {
                    wx = g.w_stop[o + x];
                    cx = __dadd_rn(g.w_in[o + x], wx);      // c_e = w_a(x) + w_x(a)
                } else {
                    x = -1;
                }
            }
            unsigned mk = __ballot_sync(FULL, x >= 0);
            while (mk) {
                int src[4], xs[4];
                double cs[4], ws[4];
                float ev[4][CPL];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    src[u] = mk ? __ffs(mk) - 1 : -1;
                    mk &= mk - 1u;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    xs[u] = __shfl_sync(FULL, x, src[u] & 31);
                    cs[u] = __shfl_sync(FULL, cx, src[u] & 31);
                    ws[u] = __shfl_sync(FULL, wx, src[u] & 31);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
#pragma unroll
                    for (int i = 0; i < CPL; ++i)
                        ev[u][i] = src[u] >= 0 ? __ldg(g.emb + (size_t)xs[u] * LD + lane + 32 * i) : 0.0f;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (src[u] < 0) break;                    // warp-uniform
#pragma unroll
                    for (int i = 0; i < CPL; ++i) s[i] = __fma_rn(cs[u], (double)ev[u][i], s[i]);
                    sb = __dadd_rn(sb, ws[u]);
                }
            }
        }
    }
}

// Work items: first one CTA per big node (a hub's 13 828 entries start first), then groups of 8 nodes, a warp per node
// (big nodes skipped).  Each item runs the roots in order and stores its rows once.
template <int CPL>
__global__ void __launch_bounds__(VG_THREADS) gather_kernel(const VgArgs g) {
    constexpr int LD = 32 * CPL;
    extern __shared__ __align__(16) unsigned char vg_smem[];
    double *s_ch = reinterpret_cast<double *>(vg_smem);   // [VG_CHAINS, LD] chain sums, then [VG_CHAINS] bias chains
    double *s_chb = s_ch + VG_CHAINS * LD;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long n_big = *g.big_cnt, n_groups = (g.n_node + VG_CHAINS - 1) / VG_CHAINS;
    for (long long item = blockIdx.x; item < n_big + n_groups; item += gridDim.x) {
        if (item < n_big) {
            // ---- a big node: warp q runs chain_q; thread t owns coordinates t, t + 256
            const int a = g.big[item];
            const long long a0 = __ldg(g.indptr + a), a1 = __ldg(g.indptr + a + 1);
            double acc[2], accb = 0.0;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int j = threadIdx.x + VG_THREADS * r;
                acc[r] = j < LD ? g.grad_emb[(size_t)a * LD + j] : 0.0;
            }
            if (threadIdx.x == 0) accb = g.grad_bias[a];
            for (long long k = 0; k < g.n_roots; ++k) {
                if (__ldg(g.ok + k) != 1) continue;
                const size_t o = (size_t)k * (size_t)g.n_node;
                const int fa = (__ldg(g.roots + k) == a) ? -1 : g.father[o + a];
                if (fa < 0 && __ldg(g.roots + k) != a) continue;          // not reached from this root
                double s[CPL], sb;
                child_chain<CPL>(g, o, g.tree_bits + (size_t)k * (size_t)g.tree_words, a, a0, a1, wid, lane, s, sb);
#pragma unroll
                for (int i = 0; i < CPL; ++i) s_ch[wid * LD + lane + 32 * i] = s[i];
                if (lane == 0) s_chb[wid] = sb;
                __syncthreads();
                const double wi = fa >= 0 ? g.w_in[o + a] : 0.0;
                const double cf = fa >= 0 ? __dadd_rn(wi, g.w_stop[o + a]) : 0.0;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int j = threadIdx.x + VG_THREADS * r;
                    if (j >= LD) continue;
                    double ch = s_ch[j];
                    for (int q = 1; q < VG_CHAINS; ++q) ch = __dadd_rn(ch, s_ch[q * LD + j]);
                    const double tf = fa >= 0 ? __dmul_rn(cf, (double)__ldg(g.emb + (size_t)fa * LD + j)) : 0.0;
                    acc[r] = __dsub_rn(acc[r], __dadd_rn(tf, ch));
                }
                if (threadIdx.x == 0) {
                    double chb = s_chb[0];
                    for (int q = 1; q < VG_CHAINS; ++q) chb = __dadd_rn(chb, s_chb[q]);
                    accb = __dsub_rn(accb, __dadd_rn(wi, chb));
                }
                __syncthreads();
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int j = threadIdx.x + VG_THREADS * r;
                if (j < LD) g.grad_emb[(size_t)a * LD + j] = acc[r];
            }
            if (threadIdx.x == 0) g.grad_bias[a] = accb;
            continue;
        }
        // ---- a group of 8 nodes, a warp per node: chain_0 only
        const long long a = (item - n_big) * VG_CHAINS + wid;
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
            const int fa = is_root ? -1 : g.father[o + a];
            if (fa < 0 && !is_root) continue;
            double s[CPL], sb;
            child_chain<CPL>(g, o, g.tree_bits + (size_t)k * (size_t)g.tree_words, (int)a, a0, a1, 0, lane, s, sb);
            const double wi = fa >= 0 ? g.w_in[o + a] : 0.0;
            const double cf = fa >= 0 ? __dadd_rn(wi, g.w_stop[o + a]) : 0.0;
#pragma unroll
            for (int i = 0; i < CPL; ++i) {
                const double tf = fa >= 0 ? __dmul_rn(cf, (double)__ldg(g.emb + (size_t)fa * LD + lane + 32 * i)) : 0.0;
                acc[i] = __dsub_rn(acc[i], __dadd_rn(tf, s[i]));
            }
            accb = __dsub_rn(accb, __dadd_rn(wi, sb));
        }
#pragma unroll
        for (int i = 0; i < CPL; ++i) g.grad_emb[(size_t)a * LD + lane + 32 * i] = acc[i];
        if (lane == 0) g.grad_bias[a] = accb;
    }
}

struct VgLayout {
    void *rec;                                 // gdist_rec_layout's part
    double *dist, *h, *T, *pi_in, *pi_stop, *partial;
    int *father, *root_ok, *big;
    unsigned *big_cnt;
    size_t partial_bytes;
};

size_t vg_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, VgLayout *v) {
    const size_t rn = (size_t)n_roots * (size_t)n_node;
    int64_t partial = 0;
    gg_game_value_scratch_bytes(n_node, n_roots, &partial);
    Slab s(buf);
    VgLayout t;
    t.rec = s.take<unsigned char>(gdist_rec_layout(nullptr, n_node, nnz_words, n_roots, nullptr));
    t.dist = s.take<double>(rn);
    t.h = s.take<double>(rn);
    t.T = s.take<double>(rn);
    t.pi_in = s.take<double>(rn);
    t.pi_stop = s.take<double>(rn);
    t.father = s.take<int>(rn);
    t.root_ok = s.take<int>((size_t)n_roots);
    t.partial = s.take<double>((size_t)partial / sizeof(double));
    t.partial_bytes = (size_t)partial;
    t.big = s.take<int>((size_t)n_node);
    t.big_cnt = s.take<unsigned>(1);
    if (buf && v) *v = t;
    return s.off;
}

}  // namespace

// the nodes with more than CHAIN_BLOCK entries, in any order (each is one independent item)
__global__ void big_nodes_kernel(long long n_node, const long long *indptr, int *big, unsigned *big_cnt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_node) return;
    if (__ldg(indptr + i + 1) - __ldg(indptr + i) > CHAIN_BLOCK) big[atomicAdd(big_cnt, 1u)] = (int)i;
}

int big_nodes_launch(long long n_node, const long long *indptr, int *big, unsigned *big_cnt, cudaStream_t st) {
    big_nodes_kernel<<<(unsigned)((n_node + 255) / 256), 256, 0, st>>>(n_node, indptr, big, big_cnt);
    return check_cuda(cudaGetLastError(), "big-node list launch");
}

}  // namespace gg

extern "C" int gg_game_value_grad_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0 && n_roots >= 0, "bad arguments");
    *bytes = (int64_t)gg::vg_layout(nullptr, n_node, (nnz + 31) / 32, n_roots, nullptr);
    return 0;
}

extern "C" int gg_game_value_grad(const gg_walk_desc *gp, const float *d_emb, const float *d_bias, const int64_t *raw_indptr,
                                  const int32_t *raw_adj, double *pos, double *neg, int32_t *ok, double *grad_emb,
                                  double *grad_bias, void *scratch, int64_t scratch_bytes, void *stream) {
    int rc = gg::check_law_desc(gp);
    if (rc || gp->n_roots == 0) return rc;
    const gg_walk_desc &d = *gp;
    GG_REQUIRE(d_emb && d_bias && raw_indptr && raw_adj, "null discriminator or raw graph pointer");
    GG_REQUIRE(pos && neg && ok && grad_emb && grad_bias && scratch, "null output or scratch pointer");
    gg::VgLayout v;
    const size_t need = gg::vg_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, &v);
    GG_REQUIRE(scratch_bytes >= (int64_t)need, "scratch too small (gg_game_value_grad_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t rn = (size_t)d.n_roots * (size_t)d.n_node;
    GG_CHECK(cudaMemsetAsync(v.dist, 0, rn * sizeof(double), st));
    GG_CHECK(cudaMemsetAsync(v.root_ok, 0, (size_t)d.n_roots * sizeof(int), st));
    GG_CHECK(cudaMemsetAsync(v.T, 0, rn * sizeof(double), st));
    GG_CHECK(cudaMemsetAsync(v.pi_stop, 0, rn * sizeof(double), st));
    GG_CHECK(cudaMemsetAsync(v.father, 0xff, rn * sizeof(int), st));
    GG_CHECK(cudaMemsetAsync(v.big_cnt, 0, sizeof(unsigned), st));
    gg::GdRec rec;
    rec.pi_in = v.pi_in; rec.pi_stop = v.pi_stop; rec.father = v.father;
    gg::gdist_rec_layout(v.rec, d.n_node, d.tree_words - 1, d.n_roots, &rec);
    rc = gg::gdist_rec_launch(d, v.dist, v.root_ok, rec, v.rec, st);
    if (rc) return rc;
    rc = gg_game_value(d.n_node, d.ld, d_emb, d_bias, raw_indptr, raw_adj, d.n_roots, d.roots, v.dist, v.root_ok, pos, neg,
                       ok, v.partial, (int64_t)v.partial_bytes, stream);
    if (rc) return rc;
    rc = gg::value_h_launch(d.n_node, d.ld, d_emb, d_bias, d.n_roots, d.roots, v.dist, v.h, st);
    if (rc) return rc;
    gg::VgArgs g;
    g.n_node = d.n_node; g.n_roots = d.n_roots; g.tree_words = d.tree_words; g.ld = d.ld;
    g.indptr = (const long long *)d.indptr; g.adj = d.adj; g.roots = d.roots; g.ok = ok; g.tree_bits = d.tree_bits;
    g.emb = d.emb; g.h = v.h; g.T = v.T; g.w_in = v.pi_in; g.w_stop = v.pi_stop; g.father = v.father;
    g.items = rec.items; g.lev_off = rec.lev_off; g.n_lev = rec.n_lev; g.big = v.big; g.big_cnt = v.big_cnt;
    g.grad_emb = grad_emb; g.grad_bias = grad_bias;
    void *args[] = {(void *)&g};
    rc = gg::coop_launch((const void *)gg::tsum_kernel, gg::VG_THREADS, 0, 0, args, st, "value gradient tsum");
    if (rc) return rc;
    rc = gg::big_nodes_launch(d.n_node, g.indptr, v.big, v.big_cnt, st);
    if (rc) return rc;
    return gg::with_cpl(d.ld, [&](auto c) {
        const size_t smem = (size_t)gg::VG_CHAINS * (32 * c + 1) * sizeof(double);
        unsigned grid = 0;
        const long long n_groups = (g.n_node + gg::VG_CHAINS - 1) / gg::VG_CHAINS;
        int rc = gg::fill_grid((const void *)gg::gather_kernel<c>, gg::VG_THREADS, smem, n_groups + g.n_node,
                               "value gradient gather", &grid);
        if (rc) return rc;
        gg::gather_kernel<c><<<grid, gg::VG_THREADS, smem, st>>>(g);
        return gg::check_cuda(cudaGetLastError(), "value gradient gather launch");
    });
}
