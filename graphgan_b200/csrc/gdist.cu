// gdist.cu -- the exact generator distribution G(v | root) of the graph-softmax walk (G mode; DESIGN.md section 5.1).
//
// The walk of graph_gan.py:225-270 from `root` stops at v with probability
//   P(v) = reach(v) * pi_v(father(v)),   reach(root) = 1,   reach(child) = reach(a) * pi_a(child)
// where pi_a is the exact law of ONE draw from a's candidate list: the canonical CDF q_j (DESIGN.md section 3) picks j for
// the uniforms u = k / 2^53 with q_{j-1} <= u < q_j, i.e. pi_a(x_j) = (ceil(q_j 2^53) - ceil(q_{j-1} 2^53)) / 2^53 -- a
// dyadic rational, exact in fp64.  Every reach / P is one fixed chain of fp64 products from the root, so the result is
// the same bits whatever order the nodes are visited in.
//
// One cooperative launch per batch of roots, level-synchronous over the trees: level L holds the items (root slot, node)
// of depth L of every root; a warp per item builds the node's candidate list with the walk sampler's own code
// (walk_list.cuh: children from the tree bits, on-demand or cached hub scores), runs the canonical softmax + CDF
// (walk_common.cuh), turns q into pi, writes reach(child) for every child and P(node) for the stop step, and appends the
// children to level L + 1.  reach(node) waits in dist[slot, node] until the node's own item replaces it with P(node).
#include <cooperative_groups.h>
#include <math.h>

#include "exact.cuh"

namespace gg {
namespace {

namespace cg = cooperative_groups;

// Items: int4 (root slot, node, father or -1 for the root itself, 1 = the node's father entry was removed by a D pass).
struct GdView {
    int4 *list[2];        // the items of levels L (list[L & 1]) and L + 1
    unsigned *cnt;        // [3]: items of level L in cnt[L % 3]; cnt[(L + 2) % 3] is cleared during level L
    int *pool_ids;        // per root slot, pool_stride entries: node a's list at indptr[a] + a when it does not fit in the
    float *pool_sc;       //   warp's shared buffers (the walk kernels' per-warp g_ids / g_sc)
    long long pool_stride;
};

// G: the G-mode law.  Rec: the same law, also recording the step law of every list per node (DESIGN.md section 5.3) and
// every level's items.  D: the D-mode law (section 5.7).
enum class GdMode { G, Rec, D };

// The bytes of the scratch layout: the counters, the items (Rec: every level's items and their offsets, else the two
// level lists), the list pools.  Fills `v` (and `rec`'s items / lev_off / n_lev) when `buf` is given.
size_t gdist_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, bool keep_levels, GdView *v,
                    GdRec *rec) {
    const long long stride = 32 * nnz_words + n_node;   // >= nnz + n_node (nnz_words = gg_tree_words(nnz) - 1)
    const size_t rn = (size_t)n_roots * (size_t)n_node;
    Slab s(buf);
    GdView t;
    GdRec r;
    t.cnt = s.take<unsigned>(3);
    if (keep_levels) {
        t.list[0] = t.list[1] = nullptr;
        r.items = s.take<int4>(rn);
        r.lev_off = s.take<unsigned>((size_t)n_node + 2);
        r.n_lev = s.take<unsigned>(1);
    } else {
        t.list[0] = s.take<int4>(rn);
        t.list[1] = s.take<int4>(rn);
    }
    t.pool_ids = s.take<int>((size_t)n_roots * (size_t)stride);
    t.pool_sc = s.take<float>((size_t)n_roots * (size_t)stride);
    t.pool_stride = stride;
    if (buf && v) *v = t;
    if (buf && rec) {
        rec->items = r.items;
        rec->lev_off = r.lev_off;
        rec->n_lev = r.n_lev;
    }
    return s.off;
}

// One item: the law of the walk's step from node it.y of root slot it.x.  Rec: also record the step law of the item's
// list per node: pi_in of every reached child, pi_stop of the node, the child's father.  D: every depth-1 item goes
// without its father whatever d1_bits holds, and a depth-1 leaf adds its reach to p_void[slot] (the walk voids the root's
// pass) instead of voiding the row.
template <int CPL, GdMode MODE>
__device__ __forceinline__ void gdist_item(const gg_walk_desc &d, double *__restrict__ dist, int *__restrict__ root_ok,
                                           const GdView &v, const int4 it, int4 *out, unsigned *out_cnt, int *s_ids,
                                           float *s_sc, int lane, unsigned long long &rows, unsigned int (&cyc)[7],
                                           Stage &stg, const GdRec &rec, double *p_void) {
    const int slot = it.x, a = it.y, fa = it.z;
    const bool is_root = fa < 0, removed = it.w != 0;
    const bool inc_father = !is_root && !removed;           // graph_gan.py:250-259, G mode (d1 bits: :258-259)
    const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
    double *row = dist + (size_t)slot * (size_t)d.n_node;
    const double reach = is_root ? 1.0 : row[a];             // written by the father's item one level up
    const long long a0 = d.indptr[a], a1 = d.indptr[a + 1];
    int *g_ids = v.pool_ids + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + a);
    float *g_sc = v.pool_sc + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + a);
    ListLaw L = list_law<CPL>(d, tb, a, fa, inc_father, s_ids, s_sc, g_ids, g_sc, lane, rows, cyc, stg);
    if (L.n == 0) {
        // a root without children voids every walk (graph_gan.py:252-253): root_ok stays 0.  Elsewhere only a node whose
        // father entry was removed can have an empty list (a D pass never leaves one): walks reaching it void the root.
        if constexpr (MODE == GdMode::D) {
            // D mode: only a depth-1 leaf has an empty list (graph_gan.py:255-257); its reach is the root's void mass,
            // a multiple of 2^-53 whose sum is exact in any order
            if (lane == 0 && !is_root) {
                atomicAdd(p_void + slot, reach);
                row[a] = 0.0;
            }
            return;
        }
        if (lane == 0 && !is_root) {
            row[a] = 0.0;
            root_ok[slot] = -1;                              // (row cleared at the end of the launch)
        }
        return;
    }
    if (lane == 0) {
        if (is_root) root_ok[slot] = 1;
        else if (removed) row[a] = 0.0;                      // no stop step: P = 0
    }
    list_norm(L, lane);
    double carry = 0.0, k_prev = 0.0;
    for (int t0 = 0; t0 < L.n; t0 += 32) {
        const int j = t0 + lane;
        const double pi = L.n > 1 ? pi_tile(L, t0, lane, carry, k_prev) : 1.0;
        const double r = __dmul_rn(reach, pi);
        const bool valid = j < L.n, stop = valid && inc_father && j == 0;
        if (stop) row[a] = r;                                // P(a): the walk draws its father (graph_gan.py:264-266)
        const int child = (valid && !stop) ? L.ids[j] : -1;
        const bool take = child >= 0 && r > 0.0;             // (a child never reached has no law below it: all zero)
        if (take) row[child] = r;
        if constexpr (MODE == GdMode::Rec) {
            const size_t o = (size_t)slot * (size_t)d.n_node;
            if (stop) rec.pi_stop[o + a] = pi;
            if (take) { rec.pi_in[o + child] = pi; rec.father[o + child] = a; }
        }
        if (!is_root) warp_append(take, out, out_cnt, make_int4(slot, child, a, 0), lane);
    }
    if (!is_root) return;
    // the root's children go to level 1 with their father-removal bit, which belongs to the entry (root -> child)
    __syncwarp();
    for (long long e0 = a0; e0 < a1; e0 += 32) {
        const long long e = e0 + lane;
        bool take = false;
        int child = -1, rm = 0;
        if (e < a1 && tree_bit(tb, e)) {
            child = __ldg(d.adj + e);
            take = row[child] > 0.0;
            if constexpr (MODE == GdMode::D) rm = 1;        // graph_gan.py:258-259: D mode always removes the root
            else rm = d.d1_bits ? (int)((__ldg(d.d1_bits + (e >> 5)) >> (e & 31)) & 1u) : 0;
        }
        warp_append(take, out, out_cnt, make_int4(slot, child, a, rm), lane);
    }
}

// The levels of one launch.  G and D keep two level lists; Rec keeps every level: level L holds items [lev_off[L],
// lev_off[L + 1]) of rec.items, so that the gradients' passes can replay the levels (the item order does not enter any
// value).  G and Rec clear the rows of roots whose walks can void; no D root voids its row, so root_ok ends 1 (the root
// has children) or 0 there.
template <int CPL, GdMode MODE>
__device__ __forceinline__ void gdist_levels(const gg_walk_desc &d, double *__restrict__ dist, int *__restrict__ root_ok,
                                             const GdView &v, const GdRec &rec, double *p_void) {
    constexpr bool REC = MODE == GdMode::Rec;
    extern __shared__ __align__(16) unsigned char walk_smem[];
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *s_sc = reinterpret_cast<float *>(walk_smem + (size_t)wid * WALK_SMEM_PER_WARP);   // the walk kernels' layout
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    Stage stg;
    stg.buf = s_sc; stg.bar = nullptr; stg.phase = 0u; stg.on = false;   // hub lists: plain loads
    const long long gw = (long long)blockIdx.x * WARPS_PER_CTA + wid, nw = (long long)gridDim.x * WARPS_PER_CTA;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
    unsigned long long rows = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    int4 *seed = REC ? rec.items : v.list[0];
    for (long long k = tid; k < d.n_roots; k += nt) seed[k] = make_int4((int)k, __ldg(d.roots + k), -1, 0);
    if (tid == 0) v.cnt[0] = (unsigned)d.n_roots;
    grid.sync();
    unsigned start = 0;                                      // Rec: first item of level lev
    for (int lev = 0;; ++lev) {
        const unsigned n_items = *(volatile unsigned *)(v.cnt + lev % 3);
        if (REC && tid == 0) rec.lev_off[lev] = start;
        if (n_items == 0) {
            if (REC && tid == 0) *rec.n_lev = (unsigned)lev;
            break;
        }
        if (tid == 0) v.cnt[(lev + 2) % 3] = 0;
        const int4 *in = REC ? rec.items + start : v.list[lev & 1];
        int4 *out = REC ? rec.items + start + n_items : v.list[(lev + 1) & 1];
        for (long long i = gw; i < (long long)n_items; i += nw)
            gdist_item<CPL, MODE>(d, dist, root_ok, v, in[i], out, v.cnt + (lev + 1) % 3, s_ids, s_sc, lane, rows, cyc, stg,
                                  rec, p_void);
        start += n_items;
        grid.sync();
    }
    if constexpr (MODE != GdMode::D) {
        // roots whose walks can void have no law: all-zero rows
        for (long long k = blockIdx.x; k < d.n_roots; k += gridDim.x) {
            if (root_ok[k] >= 0) continue;
            double *row = dist + (size_t)k * (size_t)d.n_node;
            for (long long i = threadIdx.x; i < d.n_node; i += blockDim.x) row[i] = 0.0;
            __syncthreads();
            if (threadIdx.x == 0) root_ok[k] = 0;
        }
    }
    if (lane == 0 && rows && d.counters) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows);
}

template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL))
gdist_kernel(const __grid_constant__ gg_walk_desc d, double *__restrict__ dist, int *__restrict__ root_ok, const GdView v) {
    gdist_levels<CPL, GdMode::G>(d, dist, root_ok, v, GdRec(), nullptr);
}

// p_void[slot] collects the reach of the depth-1 leaves
template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL))
gdist_d_kernel(const __grid_constant__ gg_walk_desc d, double *__restrict__ dist, int *__restrict__ root_ok,
               double *__restrict__ p_void, const GdView v) {
    gdist_levels<CPL, GdMode::D>(d, dist, root_ok, v, GdRec(), p_void);
}

template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL))
gdist_rec_kernel(const __grid_constant__ gg_walk_desc d, double *__restrict__ dist, int *__restrict__ root_ok, const GdView v,
                 const GdRec rec) {
    gdist_levels<CPL, GdMode::Rec>(d, dist, root_ok, v, rec, nullptr);
}

// cooperative launch of one of the three kernels over the whole device
int launch_gdist(const void *kern, const gg_walk_desc &d, void **args, cudaStream_t st) {
    const int cpl = d.ld / 32;
    return coop_launch(kern, WARPS_PER_CTA * 32, walk_smem_bytes(cpl, WARPS_PER_CTA), walk_min_ctas(cpl), args, st,
                       "generator distribution");
}

// gg_generator_dist, and with d_mode gg_generator_dist_d
int gdist_run(const gg_walk_desc *dp, double *dist, double *p_void, int32_t *root_ok, void *scratch, int64_t scratch_bytes,
              void *stream, bool d_mode) {
    int rc = check_law_desc(dp);
    if (rc || dp->n_roots == 0) return rc;
    const gg_walk_desc &d = *dp;
    GG_REQUIRE(dist && (p_void || !d_mode) && root_ok && scratch, "null output or scratch pointer");
    GdView v;
    const size_t need = gdist_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, false, &v, nullptr);
    GG_REQUIRE(scratch_bytes >= (int64_t)need, "scratch too small (gg_generator_dist_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(dist, 0, sizeof(double) * (size_t)d.n_roots * (size_t)d.n_node, st));
    if (d_mode) GG_CHECK(cudaMemsetAsync(p_void, 0, sizeof(double) * (size_t)d.n_roots, st));
    GG_CHECK(cudaMemsetAsync(root_ok, 0, sizeof(int32_t) * (size_t)d.n_roots, st));
    GG_CHECK(cudaMemsetAsync(v.cnt, 0, 3 * sizeof(unsigned), st));
    if (d_mode) {
        const void *kern = with_cpl(d.ld, [](auto c) { return (const void *)gdist_d_kernel<c>; });
        void *args[] = {(void *)&d, (void *)&dist, (void *)&root_ok, (void *)&p_void, (void *)&v};
        return launch_gdist(kern, d, args, st);
    }
    const void *kern = with_cpl(d.ld, [](auto c) { return (const void *)gdist_kernel<c>; });
    void *args[] = {(void *)&d, (void *)&dist, (void *)&root_ok, (void *)&v};
    return launch_gdist(kern, d, args, st);
}

}  // namespace

size_t gdist_rec_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, GdRec *rec) {
    return gdist_layout(buf, n_node, nnz_words, n_roots, true, nullptr, rec);
}

int gdist_rec_launch(const gg_walk_desc &d, double *dist, int *root_ok, GdRec rec, void *scratch, cudaStream_t st) {
    GdView v;
    gdist_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, true, &v, &rec);
    GG_CHECK(cudaMemsetAsync(v.cnt, 0, 3 * sizeof(unsigned), st));
    const void *kern = with_cpl(d.ld, [](auto c) { return (const void *)gdist_rec_kernel<c>; });
    void *args[] = {(void *)&d, (void *)&dist, (void *)&root_ok, (void *)&v, (void *)&rec};
    return launch_gdist(kern, d, args, st);
}

}  // namespace gg

extern "C" int gg_generator_dist_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0 && n_roots >= 0, "bad arguments");
    *bytes = (int64_t)gg::gdist_layout(nullptr, n_node, (nnz + 31) / 32, n_roots, false, nullptr, nullptr);
    return 0;
}

extern "C" int gg_generator_dist(const gg_walk_desc *dp, double *dist, int32_t *root_ok, void *scratch, int64_t scratch_bytes,
                                 void *stream) {
    return gg::gdist_run(dp, dist, nullptr, root_ok, scratch, scratch_bytes, stream, false);
}

extern "C" int gg_generator_dist_d(const gg_walk_desc *dp, double *dist, double *p_void, int32_t *root_ok, void *scratch,
                                   int64_t scratch_bytes, void *stream) {
    return gg::gdist_run(dp, dist, p_void, root_ok, scratch, scratch_bytes, stream, true);
}
