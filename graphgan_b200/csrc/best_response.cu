// best_response.cu -- the game value against the best discriminator, V*_c(G) = max_D V_c(G, D)
// = 2 JSD(p_true(.|c) || G(.|c)) - log 4, per root, and its generator gradient (DESIGN.md section 5.8).
//
// p_true(.|c) lives on c's neighbours, which are exactly the depth-1 nodes of c's BFS tree, and D* = p / (p + G) is 0
// everywhere else, so V*_c needs the root's list and the lists [c] + children(a) of its depth-1 nodes a only:
//   G(a)    = fl(pi_c(a) pi_a(c))                        (the bits of gg_generator_dist's dist[k, a])
//   p(a)    = n_ca / deg_c                               (n_ca: a's count in the raw list graph[c])
//   h*(a)   = G(a) log1p(p(a) / G(a))                    (0 where G(a) = 0)
//   vstar_c = -sum_a (p(a) log1p(G(a) / p(a)) + h*(a)),  hit_c = sum_a G(a),  H_c = sum_a h*(a)
// The gradient is section 5.3's policy gradient with h replaced by h* (envelope theorem: D* held fixed), whose w terms
// reduce to w_c(a) = h*(a) - pi_c(a) H_c, w_a(c) = h*(a) (1 - pi_a(c)) and w_a(x) = -pi_a(x) h*(a) for a's tree children.
//
// One cooperative launch per chunk of roots (best_response_kernel): level 0 (a warp per root: its list, pi_c), the
// depth-1 items (a warp per (root, reached depth-1 node): G, h*, and with the gradient pi_a of a's children), the per-root
// sums (a warp per root), then with the gradient one grid barrier per ok root: the root's coefficient terms, one per
// walk-CSR entry at most, added to the caller's per-entry accumulators (acc_coef: the edge coefficient c_e on both
// entries of the edge; acc_bias: the bias coefficient on the receiving node's entry).  best_response_spmm_kernel turns the
// accumulators into the gradient once per call.
#include <cooperative_groups.h>
#include <math.h>

#include "exact.cuh"

namespace gg {
namespace {

namespace cg = cooperative_groups;

constexpr long long BR_BLOCK = 256;        // entries of a depth-1 node's row per unit of the coefficient pass

struct BrView {
    int4 *items;                           // depth-1 items (root slot, node, entry (root -> node), father removed)
    unsigned *cnt;                         // their number
    int *pool_ids;                         // per root slot, pool_stride entries: node a's list at indptr[a] + a when it
    float *pool_sc;                        //   does not fit in the warp's shared buffers (as gdist.cu)
    long long pool_stride;
    double *pi_ca, *G, *hs, *pt;           // [R, N] at the depth-1 nodes: pi_c(a), G(a), h*(a), p(a) log1p(G(a) / p(a))
    double *wac, *pi_x;                    // [R, N], gradient only: w_a(c) at depth 1, pi_father(x)(x) at depth 2
    int *boff;                             // [R, N], gradient only: first unit of the root's row entry j
    int *nunit;                            // [R] units of the root's coefficient pass
    double *H;                             // [R]
    int *root_ok;                          // [R]: section 5.1's root_ok (-1 while a void is found)
};

struct BrArgs {
    const long long *raw_indptr;
    const int *mult, *rev;                 // per walk-CSR entry: n_ca of (c -> a), the reverse entry
    double *vstar, *hit;
    int *ok;
    double *acc_coef, *acc_bias;           // per walk-CSR entry (gradient only)
};

size_t br_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, bool grad, BrView *v) {
    const long long stride = 32 * nnz_words + n_node;   // >= nnz + n_node (nnz_words = gg_tree_words(nnz) - 1)
    const size_t rn = (size_t)n_roots * (size_t)n_node;
    Slab s(buf);
    BrView t;
    t.cnt = s.take<unsigned>(1);
    t.items = s.take<int4>(rn);
    t.pool_ids = s.take<int>((size_t)n_roots * (size_t)stride);
    t.pool_sc = s.take<float>((size_t)n_roots * (size_t)stride);
    t.pool_stride = stride;
    t.pi_ca = s.take<double>(rn);
    t.G = s.take<double>(rn);
    t.hs = s.take<double>(rn);
    t.pt = s.take<double>(rn);
    t.root_ok = s.take<int>((size_t)n_roots);
    t.H = s.take<double>((size_t)n_roots);
    t.wac = grad ? s.take<double>(rn) : nullptr;
    t.pi_x = grad ? s.take<double>(rn) : nullptr;
    t.boff = grad ? s.take<int>(rn) : nullptr;
    t.nunit = grad ? s.take<int>((size_t)n_roots) : nullptr;
    if (buf && v) *v = t;
    return s.off;
}

// level 0: the root's list (its children), pi_c of every child; the reached children become depth-1 items
template <int CPL>
__device__ __forceinline__ void br_root_item(const gg_walk_desc &d, const BrView &v, int slot, int *s_ids, float *s_sc,
                                             int lane, unsigned long long &rows, unsigned int (&cyc)[7], Stage &stg) {
    const int c = __ldg(d.roots + slot);
    const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
    const size_t o = (size_t)slot * (size_t)d.n_node;
    const long long a0 = d.indptr[c], a1 = d.indptr[c + 1];
    int *g_ids = v.pool_ids + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + c);
    float *g_sc = v.pool_sc + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + c);
    ListLaw L = list_law<CPL>(d, tb, c, -1, false, s_ids, s_sc, g_ids, g_sc, lane, rows, cyc, stg);
    if (L.n == 0) return;                                    // no children: every walk voids, root_ok stays 0
    if (lane == 0) v.root_ok[slot] = 1;
    list_norm(L, lane);
    double carry = 0.0, k_prev = 0.0;
    for (int t0 = 0; t0 < L.n; t0 += 32) {
        const double pi = L.n > 1 ? pi_tile(L, t0, lane, carry, k_prev) : 1.0;
        const int j = t0 + lane;
        if (j < L.n) {
            const size_t x = o + (size_t)L.ids[j];
            v.pi_ca[x] = pi;                                 // reach(a) = fl(1 * pi_c(a)) = pi_c(a)
            v.G[x] = 0.0; v.hs[x] = 0.0; v.pt[x] = 0.0;     // (the item of a reached child overwrites them)
            if (v.wac) v.wac[x] = 0.0;
        }
    }
    __syncwarp();
    for (long long e0 = a0; e0 < a1; e0 += 32) {
        const long long e = e0 + lane;
        bool take = false;
        int child = -1, rm = 0;
        if (e < a1 && tree_bit(tb, e)) {
            child = __ldg(d.adj + e);
            take = v.pi_ca[o + child] > 0.0;
            rm = d.d1_bits ? (int)((__ldg(d.d1_bits + (e >> 5)) >> (e & 31)) & 1u) : 0;
        }
        warp_append(take, v.items, v.cnt, make_int4(slot, child, (int)e, rm), lane);
    }
}

// a depth-1 item: G(a), h*(a), p(a) log1p(G / p); with GRAD also w_a(c) and pi_a(x) of a's children.  A node whose father
// entry is removed has G(a) = 0 and only matters through ok: an empty list voids the root's walks.
template <int CPL, bool GRAD>
__device__ __forceinline__ void br_d1_item(const gg_walk_desc &d, const BrArgs &ar, const BrView &v, const int4 it,
                                           int *s_ids, float *s_sc, int lane, unsigned long long &rows,
                                           unsigned int (&cyc)[7], Stage &stg) {
    const int slot = it.x, a = it.y;
    const long long e_ca = it.z;
    const int c = __ldg(d.roots + slot);
    const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
    const size_t o = (size_t)slot * (size_t)d.n_node;
    const long long a0 = d.indptr[a], a1 = d.indptr[a + 1];
    if (it.w) {
        bool any = false;
        for (long long e = a0 + lane; e < a1 && !any; e += 32) any = tree_bit(tb, e);
        if (!__any_sync(FULL, any) && lane == 0) v.root_ok[slot] = -1;
        return;
    }
    int *g_ids = v.pool_ids + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + a);
    float *g_sc = v.pool_sc + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + a);
    ListLaw L = list_law<CPL>(d, tb, a, c, true, s_ids, s_sc, g_ids, g_sc, lane, rows, cyc, stg);   // n >= 1
    list_norm(L, lane);
    double carry = 0.0, k_prev = 0.0, pi_ac = 0.0;
    for (int t0 = 0; t0 < L.n; t0 += 32) {
        const double pi = L.n > 1 ? pi_tile(L, t0, lane, carry, k_prev) : 1.0;
        const int j = t0 + lane;
        if (j == 0) pi_ac = pi;                              // the father's candidate: the stop step
        if constexpr (GRAD) {
            if (j > 0 && j < L.n) v.pi_x[o + (size_t)L.ids[j]] = pi;
        }
    }
    if (lane != 0) return;
    const double G = __dmul_rn(__ldcg(v.pi_ca + o + a), pi_ac);
    const double p = __ddiv_rn((double)__ldg(ar.mult + e_ca), (double)(__ldg(ar.raw_indptr + c + 1) - __ldg(ar.raw_indptr + c)));
    double hs = 0.0, pt = 0.0;
    if (G > 0.0) {
        hs = __dmul_rn(G, log1p(__ddiv_rn(p, G)));
        pt = __dmul_rn(p, log1p(__ddiv_rn(G, p)));
    }
    v.G[o + a] = G;
    v.hs[o + a] = hs;
    v.pt[o + a] = pt;
    if constexpr (GRAD) v.wac[o + a] = __dmul_rn(hs, __dsub_rn(1.0, pi_ac));
}

// the per-root sums over the root's row entries (lane l chains entries a0 + l, a0 + l + 32, ...; then warp_dsum);
// with GRAD the unit offsets of the coefficient pass
template <bool GRAD>
__device__ __forceinline__ void br_root_sum(const gg_walk_desc &d, const BrArgs &ar, const BrView &v, int slot, int lane) {
    const int c = __ldg(d.roots + slot);
    const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
    const size_t o = (size_t)slot * (size_t)d.n_node;
    const long long a0 = d.indptr[c], a1 = d.indptr[c + 1];
    const bool ok = __ldcg(v.root_ok + slot) == 1 && __ldg(ar.raw_indptr + c + 1) > __ldg(ar.raw_indptr + c);
    double sg = 0.0, sh = 0.0, sv = 0.0;
    if (ok) {
        for (long long e = a0 + lane; e < a1; e += 32) {
            if (!tree_bit(tb, e)) continue;
            const size_t x = o + (size_t)__ldg(d.adj + e);
            const double g = __ldcg(v.G + x), h = __ldcg(v.hs + x);
            sg = __dadd_rn(sg, g);
            sh = __dadd_rn(sh, h);
            sv = __dadd_rn(sv, __dadd_rn(__ldcg(v.pt + x), h));
        }
    }
    sg = warp_dsum(sg);
    sh = warp_dsum(sh);
    sv = warp_dsum(sv);
    if (lane == 0) {
        ar.ok[slot] = ok ? 1 : 0;
        ar.vstar[slot] = ok ? __dsub_rn(0.0, sv) : 0.0;
        ar.hit[slot] = ok ? sg : 0.0;
        v.H[slot] = ok ? sh : 0.0;
    }
    if constexpr (GRAD) {
        // units of entry j: 1 (the edge (c, a)) or, when h*(a) != 0, one per BR_BLOCK entries of a's row
        int base = 0;
        for (long long e0 = a0; e0 < a1; e0 += 32) {
            const long long e = e0 + lane;
            int nb = 0;
            if (ok && e < a1 && tree_bit(tb, e)) {
                const int x = __ldg(d.adj + e);
                nb = 1;
                if (__ldcg(v.hs + o + x) != 0.0) {
                    const long long dx = d.indptr[x + 1] - d.indptr[x];
                    nb = dx > BR_BLOCK ? (int)((dx + BR_BLOCK - 1) / BR_BLOCK) : 1;
                }
            }
            int inc = nb;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const int y = __shfl_up_sync(FULL, inc, off);
                if (lane >= off) inc += y;
            }
            if (e < a1) v.boff[o + (size_t)(e - a0)] = base + inc - nb;
            base += __shfl_sync(FULL, inc, 31);
        }
        if (lane == 0) v.nunit[slot] = base;
    }
}

__device__ __forceinline__ void br_acc_add(double *p, double t) { __stcg(p, __dadd_rn(__ldcg(p), t)); }

// unit u of root slot k's coefficient pass: entry j of the root's row with boff[j] <= u < boff[j] + units(j); its
// unit 0 adds the edge (c, a)'s terms, unit b the terms of a's children at a's entries [BR_BLOCK b, BR_BLOCK (b + 1))
__device__ __forceinline__ void br_apply_unit(const gg_walk_desc &d, const BrArgs &ar, const BrView &v, long long k, int u,
                                              int lane) {
    const int c = __ldg(d.roots + k);
    const uint32_t *tb = d.tree_bits + (size_t)k * (size_t)d.tree_words;
    const size_t o = (size_t)k * (size_t)d.n_node;
    const long long c0 = d.indptr[c];
    long long lo = 0, hi = d.indptr[c + 1] - c0;             // boff[lo] <= u < boff[hi] (boff[deg] = the unit count)
    while (hi - lo > 1) {
        const long long mid = (lo + hi) >> 1;
        if (__ldcg(v.boff + o + mid) <= u) lo = mid;
        else hi = mid;
    }
    const long long e = c0 + lo;
    const int a = __ldg(d.adj + e);
    const int b = u - __ldcg(v.boff + o + lo);
    const double h = __ldcg(v.hs + o + a);
    if (b == 0 && lane == 0) {
        const double wca = __dsub_rn(h, __dmul_rn(__ldcg(v.pi_ca + o + a), __ldcg(v.H + k)));
        const double wac = __ldcg(v.wac + o + a);
        const double ce = __dadd_rn(wca, wac);
        const long long re = __ldg(ar.rev + e);
        if (ce != 0.0) {
            br_acc_add(ar.acc_coef + e, ce);
            br_acc_add(ar.acc_coef + re, ce);
        }
        if (wca != 0.0) br_acc_add(ar.acc_bias + re, wca);   // grad_b[a] -= w_c(a): a's entry (a -> c)
        if (wac != 0.0) br_acc_add(ar.acc_bias + e, wac);    // grad_b[c] -= w_a(c): c's entry (c -> a)
    }
    if (h == 0.0) return;
    const long long x0 = d.indptr[a] + BR_BLOCK * b, xe = d.indptr[a + 1];
    const long long x1 = x0 + BR_BLOCK < xe ? x0 + BR_BLOCK : xe;
    for (long long e2 = x0 + lane; e2 < x1; e2 += 32) {
        if (!tree_bit(tb, e2)) continue;
        const double p = __ldcg(v.pi_x + o + (size_t)__ldg(d.adj + e2));
        if (p == 0.0) continue;
        const double t = -__dmul_rn(p, h);                   // w_a(x); w_x(a) = 0 at depth 2
        const long long r2 = __ldg(ar.rev + e2);
        br_acc_add(ar.acc_coef + e2, t);
        br_acc_add(ar.acc_coef + r2, t);
        br_acc_add(ar.acc_bias + r2, t);                     // grad_b[x] -= w_a(x): x's entry (x -> a)
    }
}

template <int CPL, bool GRAD>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL))
best_response_kernel(const __grid_constant__ gg_walk_desc d, const BrArgs ar, const BrView v) {
    extern __shared__ __align__(16) unsigned char walk_smem[];
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *s_sc = reinterpret_cast<float *>(walk_smem + (size_t)wid * WALK_SMEM_PER_WARP);   // the walk kernels' layout
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    Stage stg;
    stg.buf = s_sc; stg.bar = nullptr; stg.phase = 0u; stg.on = false;   // hub lists: plain loads
    const long long gw = (long long)blockIdx.x * WARPS_PER_CTA + wid, nw = (long long)gridDim.x * WARPS_PER_CTA;
    unsigned long long rows = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (long long k = gw; k < d.n_roots; k += nw) br_root_item<CPL>(d, v, (int)k, s_ids, s_sc, lane, rows, cyc, stg);
    grid.sync();
    const unsigned n_items = *(volatile unsigned *)v.cnt;
    for (long long i = gw; i < (long long)n_items; i += nw)
        br_d1_item<CPL, GRAD>(d, ar, v, v.items[i], s_ids, s_sc, lane, rows, cyc, stg);
    grid.sync();
    for (long long k = gw; k < d.n_roots; k += nw) br_root_sum<GRAD>(d, ar, v, (int)k, lane);
    if constexpr (GRAD) {
        // the roots in slot order, one barrier each: every accumulator entry takes at most one term per root
        grid.sync();
        for (long long k = 0; k < d.n_roots; ++k) {
            if (__ldcg(ar.ok + k) != 1) continue;            // grid-uniform
            const int nu = __ldcg(v.nunit + k);
            for (long long u = gw; u < nu; u += nw) br_apply_unit(d, ar, v, k, (int)u, lane);
            grid.sync();
        }
    }
    if (lane == 0 && rows && d.counters) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows);
}

// row y of the gradient: grad_emb[y] -= sum_e acc_coef[e] emb[adj[e]], grad_bias[y] -= sum_e acc_bias[e], over y's
// entries in entry order, one fp64 chain per coordinate continued from the caller's value (zero coefficients skipped).
// A warp per row; the nonzero entries of each 32-entry tile are broadcast four at a time.
template <int CPL>
__global__ void __launch_bounds__(256) best_response_spmm_kernel(long long n_node, const long long *__restrict__ indptr,
                                                                 const int *__restrict__ adj, const float *__restrict__ emb,
                                                                 const double *__restrict__ acc_coef,
                                                                 const double *__restrict__ acc_bias,
                                                                 double *__restrict__ grad_emb, double *__restrict__ grad_bias) {
    constexpr int LD = 32 * CPL;
    const int lane = threadIdx.x & 31;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long y = gw; y < n_node; y += nw) {
        const long long y0 = __ldg(indptr + y), y1 = __ldg(indptr + y + 1);
        double acc[CPL];
#pragma unroll
        for (int i = 0; i < CPL; ++i) acc[i] = grad_emb[(size_t)y * LD + lane + 32 * i];
        double accb = grad_bias[y];
        for (long long e0 = y0; e0 < y1; e0 += 32) {
            const long long e = e0 + lane;
            double cc = 0.0, cb = 0.0;
            int z = 0;
            if (e < y1) {
                cc = __ldg(acc_coef + e);
                cb = __ldg(acc_bias + e);
                z = __ldg(adj + e);
            }
            unsigned mk = __ballot_sync(FULL, cc != 0.0 || cb != 0.0);
            while (mk) {
                int src[4], zs[4];
                double cs[4], bs[4];
                float ev[4][CPL];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    src[u] = mk ? __ffs(mk) - 1 : -1;
                    mk &= mk - 1u;
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    zs[u] = __shfl_sync(FULL, z, src[u] & 31);
                    cs[u] = __shfl_sync(FULL, cc, src[u] & 31);
                    bs[u] = __shfl_sync(FULL, cb, src[u] & 31);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
#pragma unroll
                    for (int i = 0; i < CPL; ++i)
                        ev[u][i] = (src[u] >= 0 && cs[u] != 0.0) ? __ldg(emb + (size_t)zs[u] * LD + lane + 32 * i) : 0.0f;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (src[u] < 0) break;                   // warp-uniform
                    if (cs[u] != 0.0) {
#pragma unroll
                        for (int i = 0; i < CPL; ++i) acc[i] = __fma_rn(-cs[u], (double)ev[u][i], acc[i]);
                    }
                    if (bs[u] != 0.0) accb = __dsub_rn(accb, bs[u]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < CPL; ++i) grad_emb[(size_t)y * LD + lane + 32 * i] = acc[i];
        if (lane == 0) grad_bias[y] = accb;
    }
}

int br_run(const gg_walk_desc &d, const int64_t *raw_indptr, const int32_t *mult, const int32_t *rev, double *vstar,
           double *hit, int32_t *ok, double *acc_coef, double *acc_bias, void *scratch, int64_t scratch_bytes, bool grad,
           void *stream) {
    BrView v;
    const size_t need = br_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, grad, &v);
    GG_REQUIRE(scratch_bytes >= (int64_t)need,
               grad ? "scratch too small (gg_best_response_grad_scratch_bytes)" : "scratch too small (gg_best_response_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(v.cnt, 0, sizeof(unsigned), st));
    GG_CHECK(cudaMemsetAsync(v.root_ok, 0, (size_t)d.n_roots * sizeof(int), st));
    BrArgs ar;
    ar.raw_indptr = (const long long *)raw_indptr; ar.mult = mult; ar.rev = rev;
    ar.vstar = vstar; ar.hit = hit; ar.ok = ok; ar.acc_coef = acc_coef; ar.acc_bias = acc_bias;
    const void *kern = with_cpl(d.ld, [grad](auto c) {
        return grad ? (const void *)best_response_kernel<c, true> : (const void *)best_response_kernel<c, false>;
    });
    const int cpl = d.ld / 32;
    void *args[] = {(void *)&d, (void *)&ar, (void *)&v};
    return coop_launch(kern, WARPS_PER_CTA * 32, walk_smem_bytes(cpl, WARPS_PER_CTA), walk_min_ctas(cpl), args, st,
                       "best-response");
}

}  // namespace
}  // namespace gg

extern "C" int gg_best_response_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0 && n_roots >= 0, "bad arguments");
    *bytes = (int64_t)gg::br_layout(nullptr, n_node, (nnz + 31) / 32, n_roots, false, nullptr);
    return 0;
}

extern "C" int gg_best_response_grad_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0 && n_roots >= 0, "bad arguments");
    *bytes = (int64_t)gg::br_layout(nullptr, n_node, (nnz + 31) / 32, n_roots, true, nullptr);
    return 0;
}

extern "C" int gg_best_response(const gg_walk_desc *g, const int64_t *raw_indptr, const int32_t *mult, double *vstar,
                                double *hit, int32_t *ok, void *scratch, int64_t scratch_bytes, void *stream) {
    int rc = gg::check_law_desc(g);
    if (rc || g->n_roots == 0) return rc;
    GG_REQUIRE(raw_indptr && mult, "null raw graph or multiplicity pointer");
    GG_REQUIRE(vstar && hit && ok && scratch, "null output or scratch pointer");
    return gg::br_run(*g, raw_indptr, mult, nullptr, vstar, hit, ok, nullptr, nullptr, scratch, scratch_bytes, false, stream);
}

extern "C" int gg_best_response_grad(const gg_walk_desc *g, const int64_t *raw_indptr, const int32_t *mult,
                                     const int32_t *rev, double *vstar, double *hit, int32_t *ok, double *acc_coef,
                                     double *acc_bias, void *scratch, int64_t scratch_bytes, void *stream) {
    int rc = gg::check_law_desc(g);
    if (rc || g->n_roots == 0) return rc;
    GG_REQUIRE(raw_indptr && mult && rev, "null raw graph, multiplicity or reverse-entry pointer");
    GG_REQUIRE(vstar && hit && ok && acc_coef && acc_bias && scratch, "null output, accumulator or scratch pointer");
    return gg::br_run(*g, raw_indptr, mult, rev, vstar, hit, ok, acc_coef, acc_bias, scratch, scratch_bytes, true, stream);
}

extern "C" int gg_best_response_spmm(int64_t n_node, int32_t ld, const int64_t *indptr, const int32_t *adj, const float *emb,
                                     const double *acc_coef, const double *acc_bias, double *grad_emb, double *grad_bias,
                                     void *stream) {
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(n_node >= 0, "n_node must be >= 0");
    if (n_node == 0) return 0;
    GG_REQUIRE(indptr && adj && emb && acc_coef && acc_bias && grad_emb && grad_bias, "null pointer");
    return gg::with_cpl(ld, [&](auto c) {
        unsigned grid = 0;
        int rc = gg::fill_grid((const void *)gg::best_response_spmm_kernel<c>, 256, 0, (n_node + 7) / 8, "best-response SpMM",
                               &grid);
        if (rc) return rc;
        gg::best_response_spmm_kernel<c><<<grid, 256, 0, (cudaStream_t)stream>>>(n_node, (const long long *)indptr, adj, emb,
                                                                                 acc_coef, acc_bias, grad_emb, grad_bias);
        return gg::check_cuda(cudaGetLastError(), "best-response SpMM launch");
    });
}
