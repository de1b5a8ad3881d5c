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

#include "walk_list.cuh"
#include "value_grad.cuh"

namespace gg {
namespace {

namespace cg = cooperative_groups;

constexpr double TWO53 = 9007199254740992.0;

// Items: int4 (root slot, node, father or -1 for the root itself, 1 = the node's father entry was removed by a D pass).
struct GdView {
    int4 *list[2];        // the items of levels L (list[L & 1]) and L + 1
    unsigned *cnt;        // [3]: items of level L in cnt[L % 3]; cnt[(L + 2) % 3] is cleared during level L
    int *pool_ids;        // per root slot, pool_stride entries: node a's list at indptr[a] + a when it does not fit in the
    float *pool_sc;       //   warp's shared buffers (the walk kernels' per-warp g_ids / g_sc)
    long long pool_stride;
};

// the bytes of the scratch layout; fills `v` when `buf` is given
size_t gdist_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, GdView *v) {
    const long long stride = 32 * nnz_words + n_node;   // >= nnz + n_node (nnz_words = gg_tree_words(nnz) - 1)
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    const size_t o_cnt = take(3 * sizeof(unsigned));
    const size_t o_l0 = take((size_t)n_roots * (size_t)n_node * sizeof(int4));
    const size_t o_l1 = take((size_t)n_roots * (size_t)n_node * sizeof(int4));
    const size_t o_ids = take((size_t)n_roots * (size_t)stride * sizeof(int));
    const size_t o_sc = take((size_t)n_roots * (size_t)stride * sizeof(float));
    if (buf && v) {
        unsigned char *b = static_cast<unsigned char *>(buf);
        v->cnt = reinterpret_cast<unsigned *>(b + o_cnt);
        v->list[0] = reinterpret_cast<int4 *>(b + o_l0);
        v->list[1] = reinterpret_cast<int4 *>(b + o_l1);
        v->pool_ids = reinterpret_cast<int *>(b + o_ids);
        v->pool_sc = reinterpret_cast<float *>(b + o_sc);
        v->pool_stride = stride;
    }
    return off;
}

// One item: the law of the walk's step from node it.y of root slot it.x.  REC: also record the step law of the item's
// list per node (DESIGN.md section 5.3): pi_in of every reached child, pi_stop of the node, the child's father.
// DM: the D-mode law (section 5.7): every depth-1 item goes without its father whatever d1_bits holds, and a depth-1
// leaf adds its reach to p_void[slot] (the walk voids the root's pass) instead of voiding the row.
template <int CPL, bool REC = false, bool DM = false>
__device__ __forceinline__ void gdist_item(const gg_walk_desc &d, double *__restrict__ dist, int *__restrict__ root_ok,
                                           const GdView &v, const int4 it, int4 *out, unsigned *out_cnt, int *s_ids,
                                           float *s_sc, int lane, unsigned long long &rows, unsigned int (&cyc)[7],
                                           Stage &stg, const GdRec &rec = GdRec(), double *p_void = nullptr) {
    const int slot = it.x, a = it.y, fa = it.z;
    const bool is_root = fa < 0, removed = it.w != 0;
    const bool inc_father = !is_root && !removed;           // graph_gan.py:250-259, G mode (d1 bits: :258-259)
    const uint32_t *tb = d.tree_bits + (size_t)slot * (size_t)d.tree_words;
    double *row = dist + (size_t)slot * (size_t)d.n_node;
    const double reach = is_root ? 1.0 : row[a];             // written by the father's item one level up
    const long long a0 = d.indptr[a], a1 = d.indptr[a + 1];
    int *g_ids = v.pool_ids + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + a);
    float *g_sc = v.pool_sc + (size_t)slot * (size_t)v.pool_stride + (size_t)(a0 + a);
    int n;
    float m;
    int *ids;
    float *sc;
    build_list<CPL, UNR>(d, tb, a, fa, inc_father, s_ids, s_sc, g_ids, g_sc, lane, n, m, ids, sc, rows, cyc, stg);
    if (n == 0) {
        // a root without children voids every walk (graph_gan.py:252-253): root_ok stays 0.  Elsewhere only a node whose
        // father entry was removed can have an empty list (a D pass never leaves one): walks reaching it void the root.
        if constexpr (DM) {
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
    // softmax + CDF (n >= 2; one candidate is drawn with probability 1), then pi_j tile by tile
    float S = 0.0f;
    double total = 0.0;
    if (n > 1) {
        double car[2];
        S = softmax_exp_sum<UNR_S1>(sc, n, m, lane);
        total = cdf_total<UNR_S1>(sc, n, S, lane, car);
    }
    double carry = 0.0, k_prev = 0.0;                        // k_prev = ceil(q_{j-1} 2^53), q_{-1} = 0
    for (int t0 = 0; t0 < n; t0 += 32) {
        const int j = t0 + lane;
        double pi = 1.0;
        if (n > 1) {
            double x = (j < n) ? (double)__fdiv_rn(sc[j], S) : 0.0;
            x = warp_scan_ks(x, lane);
            const double q = __ddiv_rn(__dadd_rn(carry, x), total);   // q_j as cdf_store / cdf_pick_from compute it
            const double k = ceil(__dmul_rn(q, TWO53));               // #{u = k / 2^53 : u < q_j}, exact
            double kb = __shfl_up_sync(FULL, k, 1);
            if (lane == 0) kb = k_prev;
            pi = __dmul_rn(__dsub_rn(k, kb), 1.0 / TWO53);
            k_prev = __shfl_sync(FULL, k, 31);
            carry = __dadd_rn(carry, __shfl_sync(FULL, x, 31));
        }
        const double r = __dmul_rn(reach, pi);
        const bool valid = j < n, stop = valid && inc_father && j == 0;
        if (stop) row[a] = r;                                // P(a): the walk draws its father (graph_gan.py:264-266)
        const int child = (valid && !stop) ? ids[j] : -1;
        const bool take = child >= 0 && r > 0.0;             // (a child never reached has no law below it: all zero)
        if (take) row[child] = r;
        if constexpr (REC) {
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
        if (e < a1 && ((__ldg(tb + (e >> 5)) >> (e & 31)) & 1u)) {
            child = __ldg(d.adj + e);
            take = row[child] > 0.0;
            if constexpr (DM) rm = 1;                        // graph_gan.py:258-259: D mode always removes the root
            else rm = d.d1_bits ? (int)((__ldg(d.d1_bits + (e >> 5)) >> (e & 31)) & 1u) : 0;
        }
        warp_append(take, out, out_cnt, make_int4(slot, child, a, rm), lane);
    }
}

template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL))
gdist_kernel(const __grid_constant__ gg_walk_desc d, double *__restrict__ dist, int *__restrict__ root_ok, const GdView v) {
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
    for (long long k = tid; k < d.n_roots; k += nt) v.list[0][k] = make_int4((int)k, __ldg(d.roots + k), -1, 0);
    if (tid == 0) v.cnt[0] = (unsigned)d.n_roots;
    grid.sync();
    for (int lev = 0;; ++lev) {
        const unsigned n_items = *(volatile unsigned *)(v.cnt + lev % 3);
        if (n_items == 0) break;
        if (tid == 0) v.cnt[(lev + 2) % 3] = 0;
        const int4 *in = v.list[lev & 1];
        int4 *out = v.list[(lev + 1) & 1];
        for (long long i = gw; i < (long long)n_items; i += nw)
            gdist_item<CPL>(d, dist, root_ok, v, in[i], out, v.cnt + (lev + 1) % 3, s_ids, s_sc, lane, rows, cyc, stg);
        grid.sync();
    }
    // roots whose walks can void have no law: all-zero rows
    for (long long k = blockIdx.x; k < d.n_roots; k += gridDim.x) {
        if (root_ok[k] >= 0) continue;
        double *row = dist + (size_t)k * (size_t)d.n_node;
        for (long long i = threadIdx.x; i < d.n_node; i += blockDim.x) row[i] = 0.0;
        __syncthreads();
        if (threadIdx.x == 0) root_ok[k] = 0;
    }
    if (lane == 0 && rows && d.counters) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows);
}

// The D-mode law (DESIGN.md section 5.7): gdist_kernel's levels with the D-mode item; p_void[slot] collects the reach of
// the depth-1 leaves.  No root voids its row, so root_ok ends 1 (the root has children) or 0.
template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL))
gdist_d_kernel(const __grid_constant__ gg_walk_desc d, double *__restrict__ dist, int *__restrict__ root_ok,
               double *__restrict__ p_void, const GdView v) {
    extern __shared__ __align__(16) unsigned char walk_smem[];
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *s_sc = reinterpret_cast<float *>(walk_smem + (size_t)wid * WALK_SMEM_PER_WARP);
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    Stage stg;
    stg.buf = s_sc; stg.bar = nullptr; stg.phase = 0u; stg.on = false;
    const long long gw = (long long)blockIdx.x * WARPS_PER_CTA + wid, nw = (long long)gridDim.x * WARPS_PER_CTA;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
    unsigned long long rows = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (long long k = tid; k < d.n_roots; k += nt) v.list[0][k] = make_int4((int)k, __ldg(d.roots + k), -1, 0);
    if (tid == 0) v.cnt[0] = (unsigned)d.n_roots;
    grid.sync();
    for (int lev = 0;; ++lev) {
        const unsigned n_items = *(volatile unsigned *)(v.cnt + lev % 3);
        if (n_items == 0) break;
        if (tid == 0) v.cnt[(lev + 2) % 3] = 0;
        const int4 *in = v.list[lev & 1];
        int4 *out = v.list[(lev + 1) & 1];
        for (long long i = gw; i < (long long)n_items; i += nw)
            gdist_item<CPL, false, true>(d, dist, root_ok, v, in[i], out, v.cnt + (lev + 1) % 3, s_ids, s_sc, lane, rows,
                                         cyc, stg, GdRec(), p_void);
        grid.sync();
    }
    if (lane == 0 && rows && d.counters) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows);
}

// The same law, keeping every level: level L holds items [lev_off[L], lev_off[L + 1]) of rec.items, so that the
// bottom-up pass of the value gradient (value_grad.cu) can replay the levels deepest first.  dist and root_ok are the bits
// of gdist_kernel (the same item function; the item order does not enter any value).
template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, walk_min_ctas(CPL))
gdist_rec_kernel(const __grid_constant__ gg_walk_desc d, double *__restrict__ dist, int *__restrict__ root_ok, const GdView v,
                 const GdRec rec) {
    extern __shared__ __align__(16) unsigned char walk_smem[];
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float *s_sc = reinterpret_cast<float *>(walk_smem + (size_t)wid * WALK_SMEM_PER_WARP);
    int *s_ids = reinterpret_cast<int *>(s_sc + SC_CAP);
    Stage stg;
    stg.buf = s_sc; stg.bar = nullptr; stg.phase = 0u; stg.on = false;
    const long long gw = (long long)blockIdx.x * WARPS_PER_CTA + wid, nw = (long long)gridDim.x * WARPS_PER_CTA;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
    unsigned long long rows = 0;
    unsigned int cyc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (long long k = tid; k < d.n_roots; k += nt) rec.items[k] = make_int4((int)k, __ldg(d.roots + k), -1, 0);
    if (tid == 0) v.cnt[0] = (unsigned)d.n_roots;
    grid.sync();
    unsigned start = 0;                                      // first item of level lev
    for (int lev = 0;; ++lev) {
        const unsigned n_items = *(volatile unsigned *)(v.cnt + lev % 3);
        if (tid == 0) rec.lev_off[lev] = start;
        if (n_items == 0) {
            if (tid == 0) *rec.n_lev = (unsigned)lev;
            break;
        }
        if (tid == 0) v.cnt[(lev + 2) % 3] = 0;
        const int4 *in = rec.items + start;
        int4 *out = rec.items + start + n_items;
        for (long long i = gw; i < (long long)n_items; i += nw)
            gdist_item<CPL, true>(d, dist, root_ok, v, in[i], out, v.cnt + (lev + 1) % 3, s_ids, s_sc, lane, rows, cyc, stg,
                                  rec);
        start += n_items;
        grid.sync();
    }
    for (long long k = blockIdx.x; k < d.n_roots; k += gridDim.x) {
        if (root_ok[k] >= 0) continue;
        double *row = dist + (size_t)k * (size_t)d.n_node;
        for (long long i = threadIdx.x; i < d.n_node; i += blockDim.x) row[i] = 0.0;
        __syncthreads();
        if (threadIdx.x == 0) root_ok[k] = 0;
    }
    if (lane == 0 && rows && d.counters) atomicAdd(d.counters + GG_CNT_ROWS_GATHERED, rows);
}

// cooperative launch of `kern` (gdist_kernel / gdist_rec_kernel) over the whole device
int launch_gdist(const void *kern, const gg_walk_desc &d, void **args, cudaStream_t st) {
    int dev = 0, coop = 0;
    GG_CHECK(cudaGetDevice(&dev));
    GG_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    GG_REQUIRE(coop, "device does not support cooperative launches");
    const int cpl = d.ld / 32, nt = WARPS_PER_CTA * 32;
    const int smem = walk_smem_bytes(cpl, WARPS_PER_CTA);
    GG_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int per_sm = 0;
    GG_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, nt, smem));
    GG_REQUIRE(per_sm >= 1, "generator distribution kernel does not fit on an SM");
    if (per_sm > walk_min_ctas(cpl)) per_sm = walk_min_ctas(cpl);
    GG_CHECK(cudaLaunchCooperativeKernel(kern, dim3((unsigned)(sm_count() * per_sm)), dim3(nt), args, (size_t)smem, st));
    return 0;
}

// the recording variant's scratch: counters, every level's items and their offsets, the list pools of gdist_layout
size_t rec_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, GdRec *rec, GdView *v) {
    const long long stride = 32 * nnz_words + n_node;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    const size_t o_cnt = take(3 * sizeof(unsigned));
    const size_t o_items = take((size_t)n_roots * (size_t)n_node * sizeof(int4));
    const size_t o_lev = take(((size_t)n_node + 2) * sizeof(unsigned));
    const size_t o_nlev = take(sizeof(unsigned));
    const size_t o_ids = take((size_t)n_roots * (size_t)stride * sizeof(int));
    const size_t o_sc = take((size_t)n_roots * (size_t)stride * sizeof(float));
    unsigned char *b = static_cast<unsigned char *>(buf);
    if (b && rec) {
        rec->items = reinterpret_cast<int4 *>(b + o_items);
        rec->lev_off = reinterpret_cast<unsigned *>(b + o_lev);
        rec->n_lev = reinterpret_cast<unsigned *>(b + o_nlev);
    }
    if (b && v) {
        v->cnt = reinterpret_cast<unsigned *>(b + o_cnt);
        v->list[0] = v->list[1] = nullptr;
        v->pool_ids = reinterpret_cast<int *>(b + o_ids);
        v->pool_sc = reinterpret_cast<float *>(b + o_sc);
        v->pool_stride = stride;
    }
    return off;
}

}  // namespace

size_t gdist_rec_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, GdRec *rec) {
    return rec_layout(buf, n_node, nnz_words, n_roots, rec, nullptr);
}

int gdist_rec_launch(const gg_walk_desc &d, double *dist, int *root_ok, GdRec rec, void *scratch, cudaStream_t st) {
    GdView v;
    rec_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, &rec, &v);
    GG_CHECK(cudaMemsetAsync(v.cnt, 0, 3 * sizeof(unsigned), st));
    const void *kern;
    switch (d.ld / 32) {
        case 1: kern = (const void *)gdist_rec_kernel<1>; break;
        case 2: kern = (const void *)gdist_rec_kernel<2>; break;
        case 4: kern = (const void *)gdist_rec_kernel<4>; break;
        case 8: kern = (const void *)gdist_rec_kernel<8>; break;
        default: kern = (const void *)gdist_rec_kernel<16>; break;
    }
    double *dist_p = dist;
    int *ok_p = root_ok;
    void *args[] = {(void *)&d, (void *)&dist_p, (void *)&ok_p, (void *)&v, (void *)&rec};
    return launch_gdist(kern, d, args, st);
}

}  // namespace gg

extern "C" int gg_generator_dist_scratch_bytes(int64_t n_node, int64_t nnz, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && nnz >= 0 && n_roots >= 0, "bad arguments");
    *bytes = (int64_t)gg::gdist_layout(nullptr, n_node, (nnz + 31) / 32, n_roots, nullptr);
    return 0;
}

extern "C" int gg_generator_dist(const gg_walk_desc *dp, double *dist, int32_t *root_ok, void *scratch, int64_t scratch_bytes,
                                 void *stream) {
    GG_REQUIRE(dp, "null descriptor");
    const gg_walk_desc &d = *dp;
    GG_REQUIRE(gg::ld_supported(d.ld), GG_LD_MESSAGE);
    if (d.n_roots == 0) return 0;
    GG_REQUIRE(d.n_node > 0 && d.emb && d.bias && d.indptr && d.adj && d.roots && d.tree_bits, "null graph/embedding pointer");
    GG_REQUIRE(d.tree_words > 0, "tree_words missing (gg_tree_words)");
    GG_REQUIRE(dist && root_ok && scratch, "null output or scratch pointer");
    GG_REQUIRE(d.n_roots * d.n_node < (1ll << 31), "n_roots * n_node must be below 2^31 (process the roots in chunks)");
    GG_REQUIRE(!d.edge_score || (d.hub_threshold > 0 && d.hub_threshold < gg::SMEM_CAP), "hub_threshold out of range");
    gg::GdView v;
    const size_t need = gg::gdist_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, &v);
    GG_REQUIRE(scratch_bytes >= (int64_t)need, "scratch too small (gg_generator_dist_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(dist, 0, sizeof(double) * (size_t)d.n_roots * (size_t)d.n_node, st));
    GG_CHECK(cudaMemsetAsync(root_ok, 0, sizeof(int32_t) * (size_t)d.n_roots, st));
    GG_CHECK(cudaMemsetAsync(v.cnt, 0, 3 * sizeof(unsigned), st));
    const void *kern;
    switch (d.ld / 32) {
        case 1: kern = (const void *)gg::gdist_kernel<1>; break;
        case 2: kern = (const void *)gg::gdist_kernel<2>; break;
        case 4: kern = (const void *)gg::gdist_kernel<4>; break;
        case 8: kern = (const void *)gg::gdist_kernel<8>; break;
        case 16: kern = (const void *)gg::gdist_kernel<16>; break;
        default: gg::set_error("gg_generator_dist: unsupported ld %d (supported: 32, 64, 128, 256, 512)", d.ld); return 2;
    }
    double *dist_p = dist;
    int *ok_p = root_ok;
    void *args[] = {(void *)&d, (void *)&dist_p, (void *)&ok_p, (void *)&v};
    return gg::launch_gdist(kern, d, args, st);
}

extern "C" int gg_generator_dist_d(const gg_walk_desc *dp, double *dist, double *p_void, int32_t *root_ok, void *scratch,
                                   int64_t scratch_bytes, void *stream) {
    GG_REQUIRE(dp, "null descriptor");
    const gg_walk_desc &d = *dp;
    GG_REQUIRE(gg::ld_supported(d.ld), GG_LD_MESSAGE);
    if (d.n_roots == 0) return 0;
    GG_REQUIRE(d.n_node > 0 && d.emb && d.bias && d.indptr && d.adj && d.roots && d.tree_bits, "null graph/embedding pointer");
    GG_REQUIRE(d.tree_words > 0, "tree_words missing (gg_tree_words)");
    GG_REQUIRE(dist && p_void && root_ok && scratch, "null output or scratch pointer");
    GG_REQUIRE(d.n_roots * d.n_node < (1ll << 31), "n_roots * n_node must be below 2^31 (process the roots in chunks)");
    GG_REQUIRE(!d.edge_score || (d.hub_threshold > 0 && d.hub_threshold < gg::SMEM_CAP), "hub_threshold out of range");
    gg::GdView v;
    const size_t need = gg::gdist_layout(scratch, d.n_node, d.tree_words - 1, d.n_roots, &v);
    GG_REQUIRE(scratch_bytes >= (int64_t)need, "scratch too small (gg_generator_dist_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(dist, 0, sizeof(double) * (size_t)d.n_roots * (size_t)d.n_node, st));
    GG_CHECK(cudaMemsetAsync(p_void, 0, sizeof(double) * (size_t)d.n_roots, st));
    GG_CHECK(cudaMemsetAsync(root_ok, 0, sizeof(int32_t) * (size_t)d.n_roots, st));
    GG_CHECK(cudaMemsetAsync(v.cnt, 0, 3 * sizeof(unsigned), st));
    const void *kern;
    switch (d.ld / 32) {
        case 1: kern = (const void *)gg::gdist_d_kernel<1>; break;
        case 2: kern = (const void *)gg::gdist_d_kernel<2>; break;
        case 4: kern = (const void *)gg::gdist_d_kernel<4>; break;
        case 8: kern = (const void *)gg::gdist_d_kernel<8>; break;
        default: kern = (const void *)gg::gdist_d_kernel<16>; break;
    }
    double *dist_p = dist, *pv_p = p_void;
    int *ok_p = root_ok;
    void *args[] = {(void *)&d, (void *)&dist_p, (void *)&ok_p, (void *)&pv_p, (void *)&v};
    return gg::launch_gdist(kern, d, args, st);
}
