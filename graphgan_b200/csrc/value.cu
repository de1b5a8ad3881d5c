// value.cu -- the GraphGAN game value V_c(G, D) per root, exactly (DESIGN.md section 5.2).
//
//   V_c  = pos_c + neg_c
//   pos_c = -(1 / |graph[c]|) sum_k bce(s(c, graph[c][k]), 1)      raw adjacency, entry order, duplicates and self-loops
//   neg_c = -sum_v G(v | c) bce(s(c, v), 0)                         G(v | c): gg_generator_dist's rows (G mode)
//   s(c, v) = __fadd_rn(canonical 8-lane dot(E_D[c], E_D[v]), b_D[v])  (fp32, the bits of reward_kernel's score)
//   bce(s, y) = (max(s, 0) - s y) + log1p(exp(-|s|))                  (fp64 from the fp32 s; discriminator.py:26-30)
//
// Every sum has one fixed order, so the bits depend on the inputs only (not on the grid, the chunk of roots or the
// order of the roots):
//   neg: nodes in tiles of VAL_TILE; inside a tile, 8-lane group q takes nodes q, q + 32, ... (one fp64 chain each), the
//        32 group partials of a root are added as ((q0 + q1) + (q2 + q3)) per warp (xor 8, 16) and then warp 0 .. 7 in
//        order; value_reduce_kernel adds a root's tile partials with lane l chaining tiles l, l + 32, ... and a xor
//        butterfly over the lanes.
//   pos: one CTA per root (its neighbour list can be the 13 828 entries of a hub); group q chains entries q, q + 32, ...,
//        then the same warp and CTA combination.
#include <math.h>

#include "exact.cuh"

namespace gg {
namespace {

constexpr int VAL_THREADS = 256;                   // 8 warps = 32 8-lane groups
constexpr int VAL_GROUPS = VAL_THREADS / 8;
constexpr int VAL_NPG = 16;                        // nodes per group and tile
constexpr long long VAL_TILE = VAL_GROUPS * VAL_NPG;   // 512 nodes
// roots per root tile: their rows sit in shared memory (32 KB at ld >= 128), and each lane keeps RT / 8 fp64 sums
__host__ __device__ constexpr int val_root_tile(int cpl) { return cpl <= 4 ? 64 : 256 / cpl; }
__host__ __device__ constexpr size_t val_smem_bytes(int cpl) {
    return (size_t)val_root_tile(cpl) * 32 * cpl * sizeof(float) + (size_t)(VAL_THREADS / 32) * val_root_tile(cpl) * sizeof(double);
}
long long val_tiles(long long n_node) { return (n_node + VAL_TILE - 1) / VAL_TILE; }

struct ValArgs {
    long long n_node, n_roots, n_tiles;
    const float *emb, *bias;
    const long long *raw_indptr;
    const int *raw_adj, *roots, *root_ok;
    const double *dist;
    double *pos, *partial;                          // partial: [n_roots, n_tiles]
};

// bce(s, y) of TF's sigmoid_cross_entropy_with_logits, in fp64 from the fp32 logit
__device__ __forceinline__ double bce_logits(float s, bool y) {
    const double x = (double)s;
    const double m = fmax(x, 0.0);
    return __dadd_rn(y ? __dsub_rn(m, x) : m, log1p(exp(-fabs(x))));
}

__device__ __forceinline__ bool value_ok(const ValArgs &a, long long k, long long &lo, long long &deg) {
    const int c = __ldg(a.roots + k);
    lo = __ldg(a.raw_indptr + c);
    deg = __ldg(a.raw_indptr + c + 1) - lo;
    return deg > 0 && __ldg(a.root_ok + k) == 1;
}

// group8_sum of eight dots at once: lane g of the group returns dot g.  Each dot goes through group8_sum's own tree
// (xor 4, then 2, then 1; the adds only swap operands), so the bits are the same, with 7 shuffles instead of 24.
__device__ __forceinline__ float group8_sum8(const float (&s)[8], int g) {
    const bool h4 = (g & 4) != 0, h2 = (g & 2) != 0, h1 = (g & 1) != 0;
    float t[4], u[2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {                    // t[j]: dot j + 4 h4
        const float keep = h4 ? s[j + 4] : s[j], send = h4 ? s[j] : s[j + 4];
        t[j] = __fadd_rn(keep, __shfl_xor_sync(FULL, send, 4));
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {                    // u[j]: dot j + 2 h2 + 4 h4
        const float keep = h2 ? t[j + 2] : t[j], send = h2 ? t[j] : t[j + 2];
        u[j] = __fadd_rn(keep, __shfl_xor_sync(FULL, send, 2));
    }
    const float keep = h1 ? u[1] : u[0], send = h1 ? u[0] : u[1];
    return __fadd_rn(keep, __shfl_xor_sync(FULL, send, 1));
}

// ((q0 + q1) + (q2 + q3)) over the four 8-lane groups of a warp: lane g of every group returns the sum of the groups'
// lane-g values
__device__ __forceinline__ double warp_groups_sum(double x) {
    x = __dadd_rn(x, __shfl_xor_sync(FULL, x, 8));
    return __dadd_rn(x, __shfl_xor_sync(FULL, x, 16));
}

// pos_c for root slot k: one CTA
template <int CPL>
__device__ void pos_item(const ValArgs &a, long long k, double *s_part) {
    constexpr int LD = 32 * CPL;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, g = lane & 7, grp = threadIdx.x >> 3;
    long long lo, deg;
    const bool ok = value_ok(a, k, lo, deg);          // uniform over the CTA
    if (!ok) {
        if (threadIdx.x == 0) a.pos[k] = 0.0;
        return;
    }
    const int c = __ldg(a.roots + k);
    float4 rc[CPL];
#pragma unroll
    for (int j = 0; j < CPL; ++j) rc[j] = ldg4(a.emb + (size_t)c * LD + 4 * g + 32 * j);
    double acc = 0.0;
#pragma unroll 4
    for (long long e0 = 0; e0 < deg; e0 += VAL_GROUPS) {
        const long long e = e0 + grp;
        const bool valid = e < deg;
        const int v = valid ? __ldg(a.raw_adj + lo + e) : c;
        float s = 0.0f;
#pragma unroll
        for (int j = 0; j < CPL; ++j) s = fma4(rc[j], ldg4(a.emb + (size_t)v * LD + 4 * g + 32 * j), s);
        s = __fadd_rn(group8_sum(s), __ldg(a.bias + v));
        if (valid) acc = __dadd_rn(acc, bce_logits(s, true));
    }
    acc = warp_groups_sum(acc);
    if (lane == 0) s_part[wid] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double x = s_part[0];
        for (int w = 1; w < VAL_THREADS / 32; ++w) x = __dadd_rn(x, s_part[w]);
        a.pos[k] = -__ddiv_rn(x, (double)deg);
    }
    __syncthreads();
}

// dV_c / ds(c, v) = m sigma(-s) / deg_c - G sigma(s) (DESIGN.md section 5.4): m the multiplicity of v in graph[c], G the
// law's dist[k, v]; sigma(|s|) = 1 / (1 + e), sigma(-|s|) = e sigma(|s|), e = exp(-|s|), in fp64 from the fp32 s
__device__ __forceinline__ double dgrad_w(int m, double deg, double G, float s) {
    if (m == 0 && G == 0.0) return 0.0;
    const double x = (double)s, e = exp(-fabs(x));
    const double big = __drcp_rn(__dadd_rn(1.0, e)), small = __dmul_rn(e, big);
    const double sp = x >= 0.0 ? big : small, sn = x >= 0.0 ? small : big;
    const double pos = m != 0 ? __ddiv_rn(__dmul_rn((double)m, sn), deg) : 0.0;
    return __dsub_rn(pos, G != 0.0 ? __dmul_rn(G, sp) : 0.0);
}

enum class NegOut { Chain, H, W, WRef };

// The tile partials of neg for root tile rt (roots rt * RT ..) and node tile t; the root rows are in s_root.  OUT = H: each
// product h[k, v] = dist[k, v] * bce(s(c_k, v), 0) is stored instead of added (the value gradient, DESIGN.md section 5.3).
// OUT = W: h[k, v] = dgrad_w of the multiplicity mult[k, v] and dist[k, v] is stored, 0 for roots with ok_k = 0 (the
// discriminator gradient, section 5.4).  OUT = WRef: dist holds the D-mode law P_D and h[k, v] = fl(a_k dgrad_w(mult,
// deg, Q, s)) with Q = P_D / (1 - p_void[k]) and a_k = fl(deg accept[k]) (the expected reference D step, section 5.7).
template <int CPL, NegOut OUT = NegOut::Chain>
__device__ void neg_item(const ValArgs &a, int rt, long long t, const float *s_root, double *s_part, double *h = nullptr,
                         const int *mult = nullptr, const double *p_void = nullptr, const double *accept = nullptr) {
    constexpr int LD = 32 * CPL, RT = val_root_tile(CPL), RJ = RT / 8;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, g = lane & 7, grp = threadIdx.x >> 3;
    const long long k0 = (long long)rt * RT;
    double acc[RJ];
#pragma unroll
    for (int j = 0; j < RJ; ++j) acc[j] = 0.0;
    constexpr bool WW = OUT == NegOut::W || OUT == NegOut::WRef;
    double rdeg[WW ? RJ : 1];                        // W: |graph[c_k]| of lane g's roots, 0 when ok_k = 0
    double rq[OUT == NegOut::WRef ? RJ : 1], ra[OUT == NegOut::WRef ? RJ : 1];   // WRef: 1 - p_void, a_k
    if constexpr (WW) {
#pragma unroll
        for (int j = 0; j < RJ; ++j) {
            const long long k = k0 + 8 * j + g;
            long long lo, deg;
            rdeg[j] = (k < a.n_roots && value_ok(a, k, lo, deg)) ? (double)deg : 0.0;
            if constexpr (OUT == NegOut::WRef) {
                rq[j] = rdeg[j] > 0.0 ? __dsub_rn(1.0, __ldg(p_void + k)) : 1.0;
                ra[j] = rdeg[j] > 0.0 ? __dmul_rn(rdeg[j], __ldg(accept + k)) : 0.0;
            }
        }
    }
    for (int i = 0; i < VAL_NPG; ++i) {
        const long long v = t * VAL_TILE + grp + (long long)VAL_GROUPS * i;
        const bool valid = v < a.n_node;
        const long long vv = valid ? v : 0;
        float4 row[CPL];
#pragma unroll
        for (int j = 0; j < CPL; ++j) row[j] = ldg4(a.emb + (size_t)vv * LD + 4 * g + 32 * j);
        const float bv = __ldg(a.bias + vv);
        double w[RJ];                                // lane g weighs root k0 + 8 j + g
#pragma unroll
        for (int j = 0; j < RJ; ++j) {
            const long long k = k0 + 8 * j + g;
            w[j] = (valid && k < a.n_roots) ? __ldg(a.dist + (size_t)k * (size_t)a.n_node + (size_t)v) : 0.0;
        }
#pragma unroll
        for (int j = 0; j < RJ; ++j) {
            float s[8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float *rr = s_root + (8 * j + r) * LD + 4 * g;
                float x = 0.0f;
#pragma unroll
                for (int c = 0; c < CPL; ++c) x = fma4(*reinterpret_cast<const float4 *>(rr + 32 * c), row[c], x);
                s[r] = x;
            }
            const float sc = __fadd_rn(group8_sum8(s, g), bv);
            if constexpr (OUT == NegOut::H) {
                const long long k = k0 + 8 * j + g;
                if (valid && k < a.n_roots)
                    h[(size_t)k * (size_t)a.n_node + (size_t)v] = (w[j] != 0.0) ? __dmul_rn(w[j], bce_logits(sc, false)) : 0.0;
            } else if constexpr (OUT == NegOut::W) {
                const long long k = k0 + 8 * j + g;
                if (valid && k < a.n_roots) {
                    const size_t o = (size_t)k * (size_t)a.n_node + (size_t)v;
                    h[o] = rdeg[j] > 0.0 ? dgrad_w(__ldg(mult + o), rdeg[j], w[j], sc) : 0.0;
                }
            } else if constexpr (OUT == NegOut::WRef) {
                const long long k = k0 + 8 * j + g;
                if (valid && k < a.n_roots) {
                    const size_t o = (size_t)k * (size_t)a.n_node + (size_t)v;
                    const double q = w[j] != 0.0 ? __ddiv_rn(w[j], rq[j]) : 0.0;
                    h[o] = rdeg[j] > 0.0 ? __dmul_rn(ra[j], dgrad_w(__ldg(mult + o), rdeg[j], q, sc)) : 0.0;
                }
            } else {
                if (w[j] != 0.0) acc[j] = __dadd_rn(acc[j], __dmul_rn(w[j], bce_logits(sc, false)));
            }
        }
    }
    if constexpr (OUT == NegOut::Chain) {
#pragma unroll
        for (int j = 0; j < RJ; ++j) {
            const double x = warp_groups_sum(acc[j]);
            if (lane < 8) s_part[wid * RT + 8 * j + lane] = x;
        }
        __syncthreads();
        if (threadIdx.x < RT && k0 + threadIdx.x < a.n_roots) {
            double x = s_part[threadIdx.x];
            for (int w = 1; w < VAL_THREADS / 32; ++w) x = __dadd_rn(x, s_part[w * RT + threadIdx.x]);
            a.partial[(size_t)(k0 + threadIdx.x) * (size_t)a.n_tiles + (size_t)t] = x;
        }
        __syncthreads();
    }
}

// s_root = the embedding rows of root tile rt (zero rows past the last root), between two CTA barriers
template <int CPL>
__device__ __forceinline__ void stage_root_tile(const ValArgs &a, long long rt, float *s_root) {
    constexpr int LD = 32 * CPL, RT = val_root_tile(CPL);
    __syncthreads();
    for (int i = threadIdx.x; i < RT * LD / 4; i += VAL_THREADS) {
        const long long k = rt * RT + i / (LD / 4);
        float4 x = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (k < a.n_roots) x = ldg4(a.emb + (size_t)__ldg(a.roots + k) * LD + 4 * (i % (LD / 4)));
        reinterpret_cast<float4 *>(s_root)[i] = x;
    }
    __syncthreads();
}

// Work items: first one pos item per root (a hub root's list is the longest single item, so it starts first), then the
// (root tile, node tile) items of neg, node tile fastest so that a CTA keeps its root rows across items.
template <int CPL>
__global__ void __launch_bounds__(VAL_THREADS) value_kernel(const ValArgs a) {
    constexpr int LD = 32 * CPL, RT = val_root_tile(CPL);
    extern __shared__ __align__(16) unsigned char val_smem[];
    float *s_root = reinterpret_cast<float *>(val_smem);                                   // [RT, LD]
    double *s_part = reinterpret_cast<double *>(val_smem + (size_t)RT * LD * sizeof(float));   // [8 warps, RT]
    const long long n_rt = (a.n_roots + RT - 1) / RT, n_items = a.n_roots + n_rt * a.n_tiles;
    long long cur_rt = -1;
    for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
        if (item < a.n_roots) {
            pos_item<CPL>(a, item, s_part);
            continue;
        }
        const long long ni = item - a.n_roots, rt = ni / a.n_tiles, t = ni % a.n_tiles;
        if (rt != cur_rt) {
            stage_root_tile<CPL>(a, rt, s_root);
            cur_rt = rt;
        }
        neg_item<CPL>(a, (int)rt, t, s_root, s_part);
    }
}

// value_kernel's neg items with a store of each (root, node) product instead of the chain (OUT: see neg_item)
template <int CPL, NegOut OUT>
__device__ __forceinline__ void neg_store_items(const ValArgs &a, double *h, const int *mult = nullptr,
                                                const double *p_void = nullptr, const double *accept = nullptr) {
    constexpr int LD = 32 * CPL, RT = val_root_tile(CPL);
    extern __shared__ __align__(16) unsigned char val_smem[];
    float *s_root = reinterpret_cast<float *>(val_smem);
    double *s_part = reinterpret_cast<double *>(val_smem + (size_t)RT * LD * sizeof(float));
    const long long n_items = (a.n_roots + RT - 1) / RT * a.n_tiles;
    long long cur_rt = -1;
    for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
        const long long rt = item / a.n_tiles, t = item % a.n_tiles;
        if (rt != cur_rt) {
            stage_root_tile<CPL>(a, rt, s_root);
            cur_rt = rt;
        }
        neg_item<CPL, OUT>(a, (int)rt, t, s_root, s_part, h, mult, p_void, accept);
    }
}

// h[k, v] for every (root, node) pair
template <int CPL>
__global__ void __launch_bounds__(VAL_THREADS) value_h_kernel(const ValArgs a, double *__restrict__ h) {
    neg_store_items<CPL, NegOut::H>(a, h);
}

// W[k, v] = dV_{c_k} / ds(c_k, v) for every (root, node) pair
template <int CPL>
__global__ void __launch_bounds__(VAL_THREADS) value_w_kernel(const ValArgs a, const int *__restrict__ mult,
                                                              double *__restrict__ W) {
    neg_store_items<CPL, NegOut::W>(a, W, mult);
}

// W_ref[k, v] for every (root, node) pair (DESIGN.md section 5.7): value_w_kernel with the D-mode law and the acceptance
template <int CPL>
__global__ void __launch_bounds__(VAL_THREADS) value_wref_kernel(const ValArgs a, const int *__restrict__ mult,
                                                                 const double *__restrict__ p_void,
                                                                 const double *__restrict__ accept, double *__restrict__ W) {
    neg_store_items<CPL, NegOut::WRef>(a, W, mult, p_void, accept);
}

// neg_c = -(sum of the root's tile partials); warp per root
__global__ void __launch_bounds__(256) value_reduce_kernel(const ValArgs a, double *__restrict__ neg, int *__restrict__ ok) {
    const int lane = threadIdx.x & 31;
    const long long k = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= a.n_roots) return;
    const double *p = a.partial + (size_t)k * (size_t)a.n_tiles;
    double x = 0.0;
    for (long long t = lane; t < a.n_tiles; t += 32) x = __dadd_rn(x, p[t]);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) x = __dadd_rn(x, __shfl_xor_sync(FULL, x, off));
    if (lane == 0) {
        long long lo, deg;
        const bool good = value_ok(a, k, lo, deg);
        neg[k] = good ? -x : 0.0;
        ok[k] = good ? 1 : 0;
    }
}

// value_kernel (with_pos: its pos items first) or one of its store variants, over a grid that fills the device
template <int CPL, class K, class... A>
int launch_value(K kern, const ValArgs &a, bool with_pos, const char *what, cudaStream_t st, A... args) {
    const size_t smem = val_smem_bytes(CPL);
    const long long RT = val_root_tile(CPL);
    const long long n_items = (with_pos ? a.n_roots : 0) + (a.n_roots + RT - 1) / RT * a.n_tiles;
    unsigned grid = 0;
    int rc = fill_grid((const void *)kern, VAL_THREADS, smem, n_items, "game value", &grid);
    if (rc) return rc;
    kern<<<grid, VAL_THREADS, smem, st>>>(a, args...);
    return check_cuda(cudaGetLastError(), what);
}

// the ValArgs of the store variants
ValArgs store_args(long long n_node, const float *emb, const float *bias, const long long *raw_indptr, long long n_roots,
                   const int *roots, const double *dist, const int *root_ok) {
    ValArgs a = {};
    a.n_node = n_node; a.n_roots = n_roots; a.n_tiles = val_tiles(n_node);
    a.emb = emb; a.bias = bias; a.raw_indptr = raw_indptr; a.roots = roots; a.dist = dist; a.root_ok = root_ok;
    return a;
}

}  // namespace

int value_wref_launch(long long n_node, int ld, const float *emb, const float *bias, const long long *raw_indptr,
                      long long n_roots, const int *roots, const double *dist_d, const double *p_void, const int *ok_ref,
                      const double *accept, const int *mult, double *W, cudaStream_t st) {
    if (n_roots == 0) return 0;
    const ValArgs a = store_args(n_node, emb, bias, raw_indptr, n_roots, roots, dist_d, ok_ref);
    return with_cpl(ld, [&](auto c) {
        return launch_value<c>(value_wref_kernel<c>, a, false, "expected D step W launch", st, mult, p_void, accept, W);
    });
}

int value_w_launch(long long n_node, int ld, const float *emb, const float *bias, const long long *raw_indptr,
                   long long n_roots, const int *roots, const double *dist, const int *root_ok, const int *mult, double *W,
                   cudaStream_t st) {
    if (n_roots == 0) return 0;
    const ValArgs a = store_args(n_node, emb, bias, raw_indptr, n_roots, roots, dist, root_ok);
    return with_cpl(ld, [&](auto c) {
        return launch_value<c>(value_w_kernel<c>, a, false, "game value W launch", st, mult, W);
    });
}

int value_h_launch(long long n_node, int ld, const float *emb, const float *bias, long long n_roots, const int *roots,
                   const double *dist, double *h, cudaStream_t st) {
    if (n_roots == 0) return 0;
    const ValArgs a = store_args(n_node, emb, bias, nullptr, n_roots, roots, dist, nullptr);
    return with_cpl(ld, [&](auto c) { return launch_value<c>(value_h_kernel<c>, a, false, "game value h launch", st, h); });
}

}  // namespace gg

extern "C" int gg_game_value_scratch_bytes(int64_t n_node, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && n_roots >= 0, "bad arguments");
    *bytes = (int64_t)(sizeof(double) * (size_t)n_roots * (size_t)gg::val_tiles(n_node));
    return 0;
}

extern "C" int gg_game_value(int64_t n_node, int32_t ld, const float *emb, const float *bias, const int64_t *raw_indptr,
                             const int32_t *raw_adj, int64_t n_roots, const int32_t *roots, const double *dist,
                             const int32_t *root_ok, double *pos, double *neg, int32_t *ok, void *scratch,
                             int64_t scratch_bytes, void *stream) {
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(n_node > 0 && n_node < (1ll << 31), "n_node must lie in [1, 2^31)");
    GG_REQUIRE(n_roots >= 0, "n_roots must be >= 0");
    if (n_roots == 0) return 0;
    GG_REQUIRE(emb && bias && raw_indptr && raw_adj && roots, "null graph/embedding pointer");
    GG_REQUIRE(dist && root_ok, "null generator distribution pointer");
    GG_REQUIRE(pos && neg && ok && scratch, "null output or scratch pointer");
    int64_t need = 0;
    gg_game_value_scratch_bytes(n_node, n_roots, &need);
    GG_REQUIRE(scratch_bytes >= need, "scratch too small (gg_game_value_scratch_bytes)");
    gg::ValArgs a;
    a.n_node = n_node; a.n_roots = n_roots; a.n_tiles = gg::val_tiles(n_node);
    a.emb = emb; a.bias = bias; a.raw_indptr = (const long long *)raw_indptr; a.raw_adj = raw_adj; a.roots = roots;
    a.root_ok = root_ok; a.dist = dist; a.pos = pos; a.partial = static_cast<double *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = gg::with_cpl(ld, [&](auto c) {
        return gg::launch_value<c>(gg::value_kernel<c>, a, true, "game value launch", st);
    });
    if (rc) return rc;
    gg::value_reduce_kernel<<<(unsigned)((n_roots + 7) / 8), 256, 0, st>>>(a, neg, ok);
    return gg::check_cuda(cudaGetLastError(), "game value reduce launch");
}
