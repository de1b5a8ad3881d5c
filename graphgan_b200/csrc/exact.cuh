// exact.cuh -- the shared pieces of the exact-game kernels (DESIGN.md section 5): gdist.cu, value.cu, value_grad.cu,
// value_dgrad.cu, value_gref.cu and best_response.cu.
#pragma once
#include <type_traits>

#include "walk_list.cuh"

namespace gg {

// ---------------------------------------------------------------- device helpers

__device__ __forceinline__ bool tree_bit(const uint32_t *tb, long long e) { return (__ldg(tb + (e >> 5)) >> (e & 31)) & 1u; }

// lane l's value, then the xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same bits)
__device__ __forceinline__ double warp_dsum(double x) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) x = __dadd_rn(x, __shfl_xor_sync(FULL, x, off));
    return x;
}

constexpr double TWO53 = 9007199254740992.0;

// A node's candidate list (build_list: n candidates, ids, scores sc and their max m), then (list_norm, n >= 2 only) its
// canonical softmax sum S and CDF total.  A list of one candidate draws it with probability 1 and has neither.
struct ListLaw {
    int n;
    int *ids;
    float *sc;
    float m, S;
    double total;
};

template <int CPL>
__device__ __forceinline__ ListLaw list_law(const gg_walk_desc &d, const uint32_t *tb, int cur, int prev, bool inc_father,
                                            int *s_ids, float *s_sc, int *g_ids, float *g_sc, int lane,
                                            unsigned long long &rows, unsigned int (&cyc)[7], Stage &stg) {
    ListLaw L;
    build_list<CPL, UNR>(d, tb, cur, prev, inc_father, s_ids, s_sc, g_ids, g_sc, lane, L.n, L.m, L.ids, L.sc, rows, cyc, stg);
    return L;
}

__device__ __forceinline__ void list_norm(ListLaw &L, int lane) {
    L.S = 0.0f;
    L.total = 0.0;
    if (L.n > 1) {
        double car[2];
        L.S = softmax_exp_sum<UNR_S1>(L.sc, L.n, L.m, lane);
        L.total = cdf_total<UNR_S1>(L.sc, L.n, L.S, lane, car);
    }
}

// pi of candidate j = t0 + lane of a list with n > 1 candidates, the exact law of one draw (DESIGN.md section 5.1): the
// canonical CDF q_j picks j for the uniforms k / 2^53 with q_{j-1} <= u < q_j, so pi_j = (ceil(q_j 2^53) -
// ceil(q_{j-1} 2^53)) / 2^53.  carry / k_prev carry the tiles (start both at 0).
__device__ __forceinline__ double pi_tile(const ListLaw &L, int t0, int lane, double &carry, double &k_prev) {
    const int j = t0 + lane;
    double x = (j < L.n) ? (double)__fdiv_rn(L.sc[j], L.S) : 0.0;
    x = warp_scan_ks(x, lane);
    const double q = __ddiv_rn(__dadd_rn(carry, x), L.total);   // q_j as cdf_store / cdf_pick_from compute it
    const double k = ceil(__dmul_rn(q, TWO53));                  // #{u = k / 2^53 : u < q_j}, exact
    double kb = __shfl_up_sync(FULL, k, 1);
    if (lane == 0) kb = k_prev;
    const double pi = __dmul_rn(__dsub_rn(k, kb), 1.0 / TWO53);
    k_prev = __shfl_sync(FULL, k, 31);
    carry = __dadd_rn(carry, __shfl_sync(FULL, x, 31));
    return pi;
}

// ---------------------------------------------------------------- host helpers

// f(std::integral_constant<int, CPL>) for the row stride ld = 32 CPL (ld checked by the caller: ld_supported)
template <class F>
auto with_cpl(int ld, F &&f) {
    switch (ld / 32) {
        case 1: return f(std::integral_constant<int, 1>());
        case 2: return f(std::integral_constant<int, 2>());
        case 4: return f(std::integral_constant<int, 4>());
        case 8: return f(std::integral_constant<int, 8>());
        default: return f(std::integral_constant<int, 16>());
    }
}

// cooperative launch of `kern` over the whole device: as many CTAs per SM as fit, at most per_sm_cap (0: no cap)
inline int coop_launch(const void *kern, int threads, int smem, int per_sm_cap, void **args, cudaStream_t st,
                       const char *what) {
    int dev = 0, coop = 0;
    GG_CHECK(cudaGetDevice(&dev));
    GG_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    GG_REQUIRE(coop, "device does not support cooperative launches");
    GG_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int per_sm = 0;
    GG_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    if (per_sm < 1) {
        set_error("%s: %s kernel does not fit on an SM", __func__, what);
        return 2;
    }
    if (per_sm_cap > 0 && per_sm > per_sm_cap) per_sm = per_sm_cap;
    GG_CHECK(cudaLaunchCooperativeKernel(kern, dim3((unsigned)(sm_count() * per_sm)), dim3(threads), args, (size_t)smem, st));
    return 0;
}

// *grid = min(SMs x the CTAs of `kern` that fit on an SM, n_items): one pass of the device over a grid-stride item loop
inline int fill_grid(const void *kern, int threads, size_t smem, long long n_items, const char *what, unsigned *grid) {
    int per_sm = 0;
    GG_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    if (per_sm < 1) {
        set_error("%s: %s kernel does not fit on an SM", __func__, what);
        return 2;
    }
    const long long g = (long long)sm_count() * per_sm;
    *grid = (unsigned)(g < n_items ? g : n_items);
    return 0;
}

// The checks of an entry point that takes the walk descriptor of the generator's law, in this order: the row stride,
// n_roots >= 0; then, for n_roots > 0 only (no pointer is looked at without roots), the descriptor's pointers,
// tree_words, n_roots * n_node < 2^31 and the hub threshold.  The caller returns 0 for n_roots == 0.
inline int check_law_desc(const gg_walk_desc *dp) {
    GG_REQUIRE(dp, "null descriptor");
    const gg_walk_desc &d = *dp;
    GG_REQUIRE(ld_supported(d.ld), GG_LD_MESSAGE);
    GG_REQUIRE(d.n_roots >= 0, "n_roots must be >= 0");
    if (d.n_roots == 0) return 0;
    GG_REQUIRE(d.n_node > 0 && d.emb && d.bias && d.indptr && d.adj && d.roots && d.tree_bits, "null graph/embedding pointer");
    GG_REQUIRE(d.tree_words > 0, "tree_words missing (gg_tree_words)");
    GG_REQUIRE(d.n_roots * d.n_node < (1ll << 31), "n_roots * n_node must be below 2^31 (process the roots in chunks)");
    GG_REQUIRE(!d.edge_score || (d.hub_threshold > 0 && d.hub_threshold < SMEM_CAP), "hub_threshold out of range");
    return 0;
}

// Carves a scratch buffer into slabs in order, each starting 256-byte aligned.  With a null base it only counts: `off`
// ends as the bytes the layout needs, and every slab is null.
struct Slab {
    unsigned char *base;
    size_t off = 0;
    explicit Slab(void *buf) : base(static_cast<unsigned char *>(buf)) {}
    template <class T>
    T *take(size_t count) {
        const size_t o = off;
        off += (count * sizeof(T) + 255) & ~(size_t)255;
        return base ? reinterpret_cast<T *>(base + o) : nullptr;
    }
};

// ---------------------------------------------------------------- what the gradients take from gdist.cu and value.cu

// Per (root slot, node), [n_roots, n_node] row-major, written by the recording variant of the section 5.1 kernel for the
// nodes it reaches: pi_in (the node's probability in its father's list), pi_stop (its father's probability in its own
// list; the caller clears it to 0), father (the caller clears it to -1).  items / lev_off / n_lev live in the scratch
// (gdist_rec_layout): every level's items, level L at [lev_off[L], lev_off[L + 1]), n_lev levels.
struct GdRec {
    double *pi_in = nullptr, *pi_stop = nullptr;
    int *father = nullptr;
    int4 *items = nullptr;
    unsigned *lev_off = nullptr, *n_lev = nullptr;
};

// bytes of the recording kernel's scratch; fills rec->{items, lev_off, n_lev} when `buf` is given
size_t gdist_rec_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, GdRec *rec);
// dist / root_ok with the bits of gg_generator_dist, plus the records (dist and root_ok cleared by the caller)
int gdist_rec_launch(const gg_walk_desc &d, double *dist, int *root_ok, GdRec rec, void *scratch, cudaStream_t st);
// h[k, v] = dist[k, v] * bce(s(roots[k], v), 0) (0 where dist is 0): the products the value kernel adds into neg
int value_h_launch(long long n_node, int ld, const float *emb, const float *bias, long long n_roots, const int *roots,
                   const double *dist, double *h, cudaStream_t st);
// W[k, v] = dV_{c_k} / ds(c_k, v) = mult[k, v] sigma(-s) / |graph[c_k]| - dist[k, v] sigma(s), 0 for roots with ok_k = 0
// (the discriminator gradient, value_dgrad.cu, DESIGN.md section 5.4); mult: v's count in graph[c_k]
int value_w_launch(long long n_node, int ld, const float *emb, const float *bias, const long long *raw_indptr,
                   long long n_roots, const int *roots, const double *dist, const int *root_ok, const int *mult, double *W,
                   cudaStream_t st);
// W_ref[k, v] = fl(fl(|graph[c_k]| accept[k]) dgrad_w(mult, |graph[c_k]|, Q, s)), Q = dist_d[k, v] / (1 - p_void[k]):
// the expected reference D step per (root, node) (value_dgrad.cu, DESIGN.md section 5.7), 0 for roots with ok_ref = 0
int value_wref_launch(long long n_node, int ld, const float *emb, const float *bias, const long long *raw_indptr,
                      long long n_roots, const int *roots, const double *dist_d, const double *p_void, const int *ok_ref,
                      const double *accept, const int *mult, double *W, cudaStream_t st);
// entries per chain block of the gradients' node-major gathers (value_grad.cu, value_gref.cu): a list of at most this
// many entries is one warp's item, a longer one ("big") a CTA's
constexpr long long CHAIN_BLOCK = 256;
// big[0 .. *big_cnt) = the nodes with more than CHAIN_BLOCK entries, in any order (the caller clears big_cnt)
int big_nodes_launch(long long n_node, const long long *indptr, int *big, unsigned *big_cnt, cudaStream_t st);

}  // namespace gg
