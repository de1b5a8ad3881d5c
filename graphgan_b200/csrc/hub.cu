// hub.cu -- per-pass precomputation that removes the walk's redundant work (sm_90a).
//
// The reference recomputes E.E^T + b for EVERY root (graph_gan.py:238) and re-derives the same
// root-step softmax for each of the root's sample_num walks (:260-262).  Two exact reuses:
//
//  * hub_score_tm_kernel: all_score[u, v] for the adjacency of high-degree nodes u.  A score does
//    not depend on the root, only the candidate SET does (children of u in that root's tree),
//    so one pass over a hub's neighbour rows serves every walk that ever stands on u.  The pass
//    runs target-major: each target row is read once, the (few, L2-resident) hub rows many times.
//  * root_cdf_kernel: the root step's candidate list is tree[root][1:] = all neighbours of the
//    root for every walk of that root, so its normalised CDF is built once per root and each
//    walk only draws u and inverts it (walk.cu: cdf_search).
//
// Both produce exactly the floats the on-demand path produces (same canonical arithmetic),
// so sampled indices are unchanged; tests run the walk with and without them.
#include "walk_common.cuh"

namespace gg {
namespace {

// ld = 512: the warp's current row in dynamic shared memory (WIDE_ROW_BYTES per warp; walk_common.cuh)
__device__ __forceinline__ float *hub_wide_row() {
    extern __shared__ __align__(16) unsigned char hub_smem[];
    return reinterpret_cast<float *>(hub_smem + (size_t)(threadIdx.x >> 5) * WIDE_ROW_BYTES);
}

// ld = 512, target-major hub scores: the 8-lane group's target row (4 per warp)
__device__ __forceinline__ float *hub_group_row(int grp) {
    extern __shared__ __align__(16) unsigned char hub_smem[];
    return reinterpret_cast<float *>(hub_smem + (size_t)(4 * (threadIdx.x >> 5) + grp) * WIDE_ROW_BYTES);
}

// CTAs per SM the kernel is compiled for: as many as the source-major kernel's registers allowed (ld 512: shared memory)
constexpr int hub_tm_min_ctas(int cpl) { return cpl <= 2 ? 5 : cpl == 4 ? 4 : 3; }

// Target-major: item t = (v, first, count, -) covers pairs[first, first + count), hub entries e = (u -> v) of ONE target v
// stored as (u, e) (graph.py: DeviceGraph.hub_tiles).  Each 8-lane group takes one item: E[v] is read from DRAM once
// per pass for all of v's hub entries, and the hub rows E[u] -- a few MB for all hubs together, touched by every SM all
// the time -- stream past it from L2.  Source-major (a hub's row held, its targets gathered) read each target row once
// per hub that lists it.
template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32, hub_tm_min_ctas(CPL))
hub_score_tm_kernel(long long n_items, const int4 *__restrict__ items, const int2 *__restrict__ pairs,
                    const float *__restrict__ emb, const float *__restrict__ bias, int ld, float *__restrict__ edge_score) {
    const int lane = threadIdx.x & 31, grp = lane >> 3;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long t0 = 4 * warp; t0 < n_items; t0 += 4 * nwarps) {   // (t0: warp-uniform)
        const int4 it = (t0 + grp < n_items) ? __ldg(items + t0 + grp) : make_int4(0, 0, 0, 0);
        const int v = it.x, n = it.z;
        const int n_warp = __reduce_max_sync(FULL, n);
        const float bv = __ldg(bias + v);
        if constexpr (CPL == WIDE_CPL) {
            float *s_row = hub_group_row(grp);
            load_row_group_wide(emb, ld, v, s_row, lane & 7);
            score_pairs_wide(emb, ld, s_row, bv, pairs + it.y, n, n_warp, edge_score, v, lane);
        } else {
            float4 c4[CPL];
            load_row<CPL>(emb, ld, v, lane & 7, c4);
            score_pairs<CPL>(emb, ld, c4, bv, pairs + it.y, n, n_warp, edge_score, v, lane);
        }
    }
}

template <int CPL>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32)
root_cdf_kernel(const __grid_constant__ gg_walk_desc d, float *__restrict__ root_sc, double *__restrict__ root_q) {
    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long slot = warp; slot < d.n_roots; slot += nwarps) {
        const int root = d.roots[slot];
        const long long a0 = d.indptr[root], a1 = d.indptr[root + 1], o = d.rq_ptr[slot];
        const int n = (int)(a1 - a0);
        if (n == 0) continue;
        float *sc = root_sc + o;
        if (d.edge_score && n >= d.hub_threshold) {
            for (int i = lane; i < n; i += 32) sc[i] = __ldg(d.edge_score + a0 + i);
            __syncwarp();
        } else {
            if constexpr (CPL == WIDE_CPL) {
                float *s_row = hub_wide_row();
                load_row_wide(d.emb, d.ld, root, s_row, lane);
                score_edges_wide(d.emb, d.bias, d.ld, s_row, d.adj, a0, n, sc, root, lane);
            } else {
                float4 c4[CPL];
                load_row<CPL>(d.emb, d.ld, root, lane & 7, c4);
                score_edges<CPL>(d.emb, d.bias, d.ld, c4, d.adj, a0, n, sc, root, lane);
            }
        }
        cdf_store(sc, n, root_q + o, lane);
    }
}

// dynamic shared memory of a root_cdf_kernel launch (only ld = 512 keeps the current row there)
constexpr int hub_smem_bytes(int cpl) { return cpl == WIDE_CPL ? WARPS_PER_CTA * WIDE_ROW_BYTES : 0; }
// ... and of a hub_score_tm_kernel launch (one row per group)
constexpr int hub_tm_smem_bytes(int cpl) { return cpl == WIDE_CPL ? 4 * WARPS_PER_CTA * WIDE_ROW_BYTES : 0; }

}  // namespace
}  // namespace gg

extern "C" int gg_hub_scores(int64_t n_items, const int32_t *items, const int32_t *pairs, const float *emb, const float *bias,
                             int32_t ld, float *edge_score, void *stream) {
    if (n_items == 0) return 0;
    GG_REQUIRE(items && pairs && emb && bias && edge_score, "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    long long blocks = (n_items + 4 * gg::WARPS_PER_CTA - 1) / (4 * gg::WARPS_PER_CTA);
    const long long cap = (long long)gg::sm_count() * 8;
    if (blocks > cap) blocks = cap;
    cudaStream_t st = (cudaStream_t)stream;
    const int4 *it = reinterpret_cast<const int4 *>(items);
    const int2 *pr = reinterpret_cast<const int2 *>(pairs);
    if (ld == 512) {
        static_assert(gg::hub_tm_smem_bytes(gg::WIDE_CPL) > 48 * 1024, "the attribute is needed");
        GG_CHECK(cudaFuncSetAttribute(gg::hub_score_tm_kernel<gg::WIDE_CPL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      gg::hub_tm_smem_bytes(gg::WIDE_CPL)));
    }
#define GG_LAUNCH(C)                                                                                           \
    gg::hub_score_tm_kernel<C><<<(unsigned)blocks, gg::WARPS_PER_CTA * 32, gg::hub_tm_smem_bytes(C), st>>>(    \
        n_items, it, pr, emb, bias, ld, edge_score)
    switch (ld / 32) {
        case 1: GG_LAUNCH(1); break;
        case 2: GG_LAUNCH(2); break;
        case 4: GG_LAUNCH(4); break;
        case 8: GG_LAUNCH(8); break;
        case 16: GG_LAUNCH(16); break;
        default: gg::set_error("gg_hub_scores: unsupported ld %d (supported: 32, 64, 128, 256, 512)", ld); return 2;
    }
#undef GG_LAUNCH
    return gg::check_cuda(cudaGetLastError(), "hub score kernel launch");
}

extern "C" int gg_root_cdf(const gg_walk_desc *dp, float *root_sc, double *root_q, void *stream) {
    GG_REQUIRE(dp, "null descriptor");
    if (dp->n_roots == 0) return 0;
    GG_REQUIRE(root_sc && root_q, "null pointer");
    const gg_walk_desc &d = *dp;
    GG_REQUIRE(d.roots && d.indptr && d.adj && d.emb && d.bias && d.rq_ptr, "null pointer in descriptor");
    GG_REQUIRE(gg::ld_supported(d.ld), GG_LD_MESSAGE);
    if (d.n_roots == 0) return 0;
    long long blocks = (d.n_roots + gg::WARPS_PER_CTA - 1) / gg::WARPS_PER_CTA;
    const long long cap = (long long)gg::sm_count() * 8;
    if (blocks > cap) blocks = cap;
    cudaStream_t st = (cudaStream_t)stream;
    switch (d.ld / 32) {
        case 1: gg::root_cdf_kernel<1><<<(unsigned)blocks, gg::WARPS_PER_CTA * 32, 0, st>>>(d, root_sc, root_q); break;
        case 2: gg::root_cdf_kernel<2><<<(unsigned)blocks, gg::WARPS_PER_CTA * 32, 0, st>>>(d, root_sc, root_q); break;
        case 4: gg::root_cdf_kernel<4><<<(unsigned)blocks, gg::WARPS_PER_CTA * 32, 0, st>>>(d, root_sc, root_q); break;
        case 8: gg::root_cdf_kernel<8><<<(unsigned)blocks, gg::WARPS_PER_CTA * 32, 0, st>>>(d, root_sc, root_q); break;
        case 16:
            gg::root_cdf_kernel<16><<<(unsigned)blocks, gg::WARPS_PER_CTA * 32, gg::hub_smem_bytes(16), st>>>(d, root_sc, root_q);
            break;
        default: gg::set_error("gg_root_cdf: unsupported ld %d (supported: 32, 64, 128, 256, 512)", d.ld); return 2;
    }
    return gg::check_cuda(cudaGetLastError(), "root cdf kernel launch");
}
