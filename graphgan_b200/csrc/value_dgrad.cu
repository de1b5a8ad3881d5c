// value_dgrad.cu -- the exact discriminator gradient of the game value, grad_D sum_c V_c(G, D) (DESIGN.md section 5.4).
//
// Per root c = c_k with ok_k = 1 (section 5.2), s(c, v) = E_D[c] . E_D[v] + b_D[v] the canonical fp32 score:
//   W[k, v] = dV_c / ds(c, v) = n_kv sigma(-s) / deg_c - G(v | c) sigma(s)      (n_kv: v's count in the raw list graph[c])
//   grad_b[v] += W[k, v],  grad_E[v] += W[k, v] E_D[c]  (node side),  grad_E[c] += C_k = sum_v W[k, v] E_D[v]  (centre side)
// G does not depend on D, so the law is a fixed weight.  Roots with ok_k = 0 add nothing.
//
// Per chunk of roots: mult_kernel counts n_kv into an int32 [R, N] plane (integer atomics over the raw lists, cleared per
// chunk); value_w_kernel (value.cu, the value kernel's node tiling) stores W [R, N]; cen_kernel forms C_k per fixed tile
// of CEN_TILE nodes (each coordinate one fma chain over the tile's nodes in order from +0) and cen_reduce_kernel adds a
// root's tile partials in tile order; node_kernel, node-major, adds each root's contribution to each row.
//
// Order (the bits depend on the inputs only): row r, coordinate i, takes the roots in the order given (WalkSampler sorts
// them by id) as one fp64 chain continued from the caller's accumulator; per root k with ok_k = 1:
//   acc = fma(W[k, r], E_D[c_k][i], acc) when W[k, r] != 0,  then acc = acc + C_k[i] when c_k = r;
// the bias chain is accb = accb + W[k, r] when W[k, r] != 0.
//
// The expected reference D step of one pass (gg_expected_d_grad, DESIGN.md section 5.7) runs the same passes with
// W_ref (value.cu's WRef store) in place of W and ok_ref in place of ok, after accept_kernel has formed P_acc and ok_ref.
#include "exact.cuh"

namespace gg {
namespace {

constexpr int DG_THREADS = 256;                 // 8 warps
constexpr long long CEN_TILE = 2048;            // nodes per centre tile: the C_k partials are fixed by N alone

long long cen_tiles(long long n_node) { return (n_node + CEN_TILE - 1) / CEN_TILE; }

struct DgArgs {
    long long n_node, n_roots, n_ctiles;
    const float *emb;
    const long long *raw_indptr;
    const int *raw_adj, *roots, *root_ok;
    int *mult;
    const double *W;
    double *partial, *C;                        // partial: [n_roots, n_ctiles, ld]; C: [n_roots, ld]
    double *grad_emb, *grad_bias;
};

__device__ __forceinline__ bool root_ok_k(const DgArgs &a, long long k) {
    const int c = __ldg(a.roots + k);
    return __ldg(a.raw_indptr + c + 1) > __ldg(a.raw_indptr + c) && __ldg(a.root_ok + k) == 1;
}

// n_kv: a CTA per root, a thread per raw entry
__global__ void __launch_bounds__(DG_THREADS) mult_kernel(const DgArgs a) {
    const long long k = blockIdx.x;
    if (!root_ok_k(a, k)) return;
    const int c = __ldg(a.roots + k);
    const long long lo = __ldg(a.raw_indptr + c), hi = __ldg(a.raw_indptr + c + 1);
    for (long long e = lo + threadIdx.x; e < hi; e += DG_THREADS)
        atomicAdd(a.mult + (size_t)k * (size_t)a.n_node + (size_t)__ldg(a.raw_adj + e), 1);
}

// roots per warp in the centre pass: every lane keeps RW x CPL fp64 sums (16)
__host__ __device__ constexpr int cen_rw(int cpl) { return cpl >= 16 ? 1 : 16 / cpl; }

// C_k partials: items (centre tile t, root tile), the root tile fastest so that concurrent CTAs share the tile's rows in
// L2; warp w owns roots rt * 8 RW + w RW + [0, RW), lane l the coordinates l + 32 i
template <int CPL>
__global__ void __launch_bounds__(DG_THREADS) cen_kernel(const DgArgs a) {
    constexpr int LD = 32 * CPL, RW = cen_rw(CPL), CRT = 8 * RW;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long n_rt = (a.n_roots + CRT - 1) / CRT, n_items = n_rt * a.n_ctiles;
    for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
        const long long t = item / n_rt, k0 = (item % n_rt) * CRT + (long long)wid * RW;
        if (k0 >= a.n_roots) continue;                                  // warp-uniform
        const long long v0 = t * CEN_TILE, v1 = v0 + CEN_TILE < a.n_node ? v0 + CEN_TILE : a.n_node;
        const double *wr[RW];
#pragma unroll
        for (int r = 0; r < RW; ++r) wr[r] = a.W + (size_t)(k0 + r < a.n_roots ? k0 + r : k0) * (size_t)a.n_node;
        double acc[RW][CPL];
#pragma unroll
        for (int r = 0; r < RW; ++r)
#pragma unroll
            for (int i = 0; i < CPL; ++i) acc[r][i] = 0.0;
#pragma unroll 2
        for (long long v = v0; v < v1; ++v) {
            float e[CPL];
#pragma unroll
            for (int i = 0; i < CPL; ++i) e[i] = __ldg(a.emb + (size_t)v * LD + lane + 32 * i);
#pragma unroll
            for (int r = 0; r < RW; ++r) {
                const double w = __ldg(wr[r] + v);
#pragma unroll
                for (int i = 0; i < CPL; ++i) acc[r][i] = __fma_rn(w, (double)e[i], acc[r][i]);
            }
        }
#pragma unroll
        for (int r = 0; r < RW; ++r) {
            if (k0 + r >= a.n_roots) break;
            double *p = a.partial + ((size_t)(k0 + r) * (size_t)a.n_ctiles + (size_t)t) * LD;
#pragma unroll
            for (int i = 0; i < CPL; ++i) p[lane + 32 * i] = acc[r][i];
        }
    }
}

// C_k[i] = the tile partials of (k, i) added in tile order from the first; a thread per (k, i)
__global__ void __launch_bounds__(256) cen_reduce_kernel(const DgArgs a, int ld) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.n_roots * ld) return;
    const long long k = j / ld, i = j % ld;
    const double *p = a.partial + (size_t)k * (size_t)a.n_ctiles * ld + i;
    double x = p[0];
#pragma unroll 8
    for (long long t = 1; t < a.n_ctiles; ++t) x = __dadd_rn(x, p[(size_t)t * ld]);
    a.C[j] = x;
}

// the node pass: nodes per warp (every lane keeps NPW x CPL fp64 sums, 16), roots per shared-memory tile (16 KB of rows)
__host__ __device__ constexpr int node_npw(int cpl) { return cpl >= 16 ? 1 : 16 / cpl; }
__host__ __device__ constexpr int node_rt(int cpl) { return cpl <= 4 ? 32 : 128 / cpl; }
__host__ __device__ constexpr size_t node_smem_bytes(int cpl) {
    return (size_t)node_rt(cpl) * 32 * cpl * sizeof(float) + (size_t)node_rt(cpl) * 8 * node_npw(cpl) * sizeof(double) +
           (size_t)node_rt(cpl) * sizeof(int);
}

// Items: blocks of 8 NPW consecutive nodes, warp w owning nodes w NPW + [0, NPW), lane l the coordinates l + 32 i.  Each
// item runs the roots in order, a root tile at a time (rows E_D[c_k], W[k, block] and c_k in shared memory), and stores its
// rows once.
template <int CPL>
__global__ void __launch_bounds__(DG_THREADS) node_kernel(const DgArgs a) {
    constexpr int LD = 32 * CPL, NPW = node_npw(CPL), NB = 8 * NPW, RT = node_rt(CPL);
    extern __shared__ __align__(16) unsigned char dg_smem[];
    float *s_row = reinterpret_cast<float *>(dg_smem);                                         // [RT, LD]
    double *s_w = reinterpret_cast<double *>(dg_smem + (size_t)RT * LD * sizeof(float));       // [RT, NB]
    int *s_c = reinterpret_cast<int *>(s_w + RT * NB);                                         // [RT]: c_k, -1 when ok_k = 0
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long n_items = (a.n_node + NB - 1) / NB;
    for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
        const long long vb = item * NB, v0 = vb + (long long)wid * NPW;
        double acc[NPW][CPL], accb[NPW];
#pragma unroll
        for (int u = 0; u < NPW; ++u) {
            const bool in = v0 + u < a.n_node;
#pragma unroll
            for (int i = 0; i < CPL; ++i) acc[u][i] = in ? a.grad_emb[(size_t)(v0 + u) * LD + lane + 32 * i] : 0.0;
            accb[u] = in ? a.grad_bias[v0 + u] : 0.0;
        }
        for (long long r0 = 0; r0 < a.n_roots; r0 += RT) {
            const int nr = a.n_roots - r0 < RT ? (int)(a.n_roots - r0) : RT;
            __syncthreads();
            for (int x = threadIdx.x; x < nr * LD / 4; x += DG_THREADS)
                reinterpret_cast<float4 *>(s_row)[x] = ldg4(a.emb + (size_t)__ldg(a.roots + r0 + x / (LD / 4)) * LD + 4 * (x % (LD / 4)));
            for (int x = threadIdx.x; x < nr * NB; x += DG_THREADS) {
                const long long v = vb + x % NB;
                s_w[x] = v < a.n_node ? __ldg(a.W + (size_t)(r0 + x / NB) * (size_t)a.n_node + (size_t)v) : 0.0;
            }
            for (int x = threadIdx.x; x < nr; x += DG_THREADS) s_c[x] = root_ok_k(a, r0 + x) ? __ldg(a.roots + r0 + x) : -1;
            __syncthreads();
            for (int j = 0; j < nr; ++j) {
                const int c = s_c[j];
                if (c < 0) continue;                                    // uniform over the CTA
                float e[CPL];
#pragma unroll
                for (int i = 0; i < CPL; ++i) e[i] = s_row[j * LD + lane + 32 * i];
#pragma unroll
                for (int u = 0; u < NPW; ++u) {
                    const double w = s_w[j * NB + wid * NPW + u];       // uniform over the warp
                    if (w != 0.0) {
#pragma unroll
                        for (int i = 0; i < CPL; ++i) acc[u][i] = __fma_rn(w, (double)e[i], acc[u][i]);
                        accb[u] = __dadd_rn(accb[u], w);
                    }
                    if (c == v0 + u) {
                        const double *ck = a.C + (size_t)(r0 + j) * LD;
#pragma unroll
                        for (int i = 0; i < CPL; ++i) acc[u][i] = __dadd_rn(acc[u][i], ck[lane + 32 * i]);
                    }
                }
            }
        }
#pragma unroll
        for (int u = 0; u < NPW; ++u) {
            if (v0 + u >= a.n_node) break;
#pragma unroll
            for (int i = 0; i < CPL; ++i) a.grad_emb[(size_t)(v0 + u) * LD + lane + 32 * i] = acc[u][i];
            if (lane == 0) a.grad_bias[v0 + u] = accb[u];
        }
    }
}

// P_acc = (1 - p_void)^deg_c by square-and-multiply from the least significant bit of deg_c, one __dmul_rn per step;
// ok_ref = deg_c > 0, the root has children (root_ok = 1) and P_acc > 0.  accept is 0 where ok_ref is 0.
__global__ void __launch_bounds__(256) accept_kernel(long long n_roots, const long long *__restrict__ raw_indptr,
                                                     const int *__restrict__ roots, const double *__restrict__ p_void,
                                                     const int *__restrict__ root_ok, double *__restrict__ accept,
                                                     int *__restrict__ ok_ref) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_roots) return;
    const int c = __ldg(roots + k);
    long long e = __ldg(raw_indptr + c + 1) - __ldg(raw_indptr + c);
    double p = 0.0;
    if (e > 0 && __ldg(root_ok + k) == 1) {
        double base = __dsub_rn(1.0, __ldg(p_void + k));
        p = 1.0;
        for (; e > 0; e >>= 1) {
            if (e & 1) p = __dmul_rn(p, base);
            base = __dmul_rn(base, base);
        }
    }
    accept[k] = p;
    ok_ref[k] = p > 0.0 ? 1 : 0;
}

template <int CPL>
int launch_passes(const DgArgs &a, cudaStream_t st) {
    constexpr long long CRT = 8 * cen_rw(CPL), NB = 8 * node_npw(CPL);
    unsigned grid = 0;
    int rc = fill_grid((const void *)cen_kernel<CPL>, DG_THREADS, 0, (a.n_roots + CRT - 1) / CRT * a.n_ctiles,
                       "discriminator gradient centre", &grid);
    if (rc) return rc;
    cen_kernel<CPL><<<grid, DG_THREADS, 0, st>>>(a);
    GG_CHECK(cudaGetLastError());
    const long long n = a.n_roots * 32 * CPL;
    cen_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, 32 * CPL);
    GG_CHECK(cudaGetLastError());
    const size_t smem = node_smem_bytes(CPL);
    rc = fill_grid((const void *)node_kernel<CPL>, DG_THREADS, smem, (a.n_node + NB - 1) / NB, "discriminator gradient node",
                   &grid);
    if (rc) return rc;
    node_kernel<CPL><<<grid, DG_THREADS, smem, st>>>(a);
    return check_cuda(cudaGetLastError(), "discriminator gradient node launch");
}

struct DgLayout {
    int *mult;
    double *W, *partial, *C;
    int *ok_ref;                                // gg_expected_d_grad only
};

// gg_game_value_grad_d's scratch; with ok_ref (gg_expected_d_grad), then ok_ref [n_roots]
size_t dg_layout(void *buf, long long n_node, int ld, long long n_roots, bool ok_ref, DgLayout *v) {
    const size_t rn = (size_t)n_roots * (size_t)n_node;
    Slab s(buf);
    DgLayout t;
    t.mult = s.take<int>(rn);
    t.W = s.take<double>(rn);
    t.partial = s.take<double>((size_t)n_roots * (size_t)cen_tiles(n_node) * (size_t)ld);
    t.C = s.take<double>((size_t)n_roots * (size_t)ld);
    t.ok_ref = ok_ref ? s.take<int>((size_t)n_roots) : nullptr;
    if (buf && v) *v = t;
    return s.off;
}

}  // namespace
}  // namespace gg

extern "C" int gg_game_value_grad_d_scratch_bytes(int64_t n_node, int32_t ld, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && n_roots >= 0, "bad arguments");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    *bytes = (int64_t)gg::dg_layout(nullptr, n_node, ld, n_roots, false, nullptr);
    return 0;
}

extern "C" int gg_game_value_grad_d(int64_t n_node, int32_t ld, const float *emb, const float *bias,
                                    const int64_t *raw_indptr, const int32_t *raw_adj, int64_t n_roots, const int32_t *roots,
                                    const double *dist, const int32_t *root_ok, double *grad_emb, double *grad_bias,
                                    void *scratch, int64_t scratch_bytes, void *stream) {
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(n_node > 0 && n_node < (1ll << 31), "n_node must lie in [1, 2^31)");
    GG_REQUIRE(n_roots >= 0, "n_roots must be >= 0");
    if (n_roots == 0) return 0;
    GG_REQUIRE(emb && bias && raw_indptr && raw_adj && roots, "null graph/embedding pointer");
    GG_REQUIRE(dist && root_ok, "null generator distribution pointer");
    GG_REQUIRE(grad_emb && grad_bias && scratch, "null output or scratch pointer");
    gg::DgLayout v;
    const size_t need = gg::dg_layout(scratch, n_node, ld, n_roots, false, &v);
    GG_REQUIRE(scratch_bytes >= (int64_t)need, "scratch too small (gg_game_value_grad_d_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    gg::DgArgs a;
    a.n_node = n_node; a.n_roots = n_roots; a.n_ctiles = gg::cen_tiles(n_node);
    a.emb = emb; a.raw_indptr = (const long long *)raw_indptr; a.raw_adj = raw_adj; a.roots = roots; a.root_ok = root_ok;
    a.mult = v.mult; a.W = v.W; a.partial = v.partial; a.C = v.C; a.grad_emb = grad_emb; a.grad_bias = grad_bias;
    GG_CHECK(cudaMemsetAsync(v.mult, 0, (size_t)n_roots * (size_t)n_node * sizeof(int), st));
    gg::mult_kernel<<<(unsigned)n_roots, gg::DG_THREADS, 0, st>>>(a);
    GG_CHECK(cudaGetLastError());
    int rc = gg::value_w_launch(n_node, ld, emb, bias, a.raw_indptr, n_roots, roots, dist, root_ok, v.mult, v.W, st);
    if (rc) return rc;
    return gg::with_cpl(ld, [&](auto c) { return gg::launch_passes<c>(a, st); });
}

extern "C" int gg_expected_d_grad_scratch_bytes(int64_t n_node, int32_t ld, int64_t n_roots, int64_t *bytes) {
    GG_REQUIRE(bytes && n_node >= 0 && n_roots >= 0, "bad arguments");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    *bytes = (int64_t)gg::dg_layout(nullptr, n_node, ld, n_roots, true, nullptr);
    return 0;
}

extern "C" int gg_expected_d_grad(int64_t n_node, int32_t ld, const float *emb, const float *bias, const int64_t *raw_indptr,
                                  const int32_t *raw_adj, int64_t n_roots, const int32_t *roots, const double *dist_d,
                                  const double *p_void, const int32_t *root_ok, double *accept, double *grad_emb,
                                  double *grad_bias, void *scratch, int64_t scratch_bytes, void *stream) {
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(n_node > 0 && n_node < (1ll << 31), "n_node must lie in [1, 2^31)");
    GG_REQUIRE(n_roots >= 0, "n_roots must be >= 0");
    if (n_roots == 0) return 0;
    GG_REQUIRE(emb && bias && raw_indptr && raw_adj && roots, "null graph/embedding pointer");
    GG_REQUIRE(dist_d && p_void && root_ok, "null D-mode law pointer");
    GG_REQUIRE(accept && grad_emb && grad_bias && scratch, "null output or scratch pointer");
    gg::DgLayout v;
    const size_t need = gg::dg_layout(scratch, n_node, ld, n_roots, true, &v);
    int *ok_ref = v.ok_ref;
    GG_REQUIRE(scratch_bytes >= (int64_t)need, "scratch too small (gg_expected_d_grad_scratch_bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    const long long *rip = (const long long *)raw_indptr;
    gg::accept_kernel<<<(unsigned)((n_roots + 255) / 256), 256, 0, st>>>(n_roots, rip, roots, p_void, root_ok, accept, ok_ref);
    GG_CHECK(cudaGetLastError());
    gg::DgArgs a;
    a.n_node = n_node; a.n_roots = n_roots; a.n_ctiles = gg::cen_tiles(n_node);
    a.emb = emb; a.raw_indptr = rip; a.raw_adj = raw_adj; a.roots = roots; a.root_ok = ok_ref;
    a.mult = v.mult; a.W = v.W; a.partial = v.partial; a.C = v.C; a.grad_emb = grad_emb; a.grad_bias = grad_bias;
    GG_CHECK(cudaMemsetAsync(v.mult, 0, (size_t)n_roots * (size_t)n_node * sizeof(int), st));
    gg::mult_kernel<<<(unsigned)n_roots, gg::DG_THREADS, 0, st>>>(a);
    GG_CHECK(cudaGetLastError());
    int rc = gg::value_wref_launch(n_node, ld, emb, bias, rip, n_roots, roots, dist_d, p_void, ok_ref, accept, v.mult, v.W, st);
    if (rc) return rc;
    return gg::with_cpl(ld, [&](auto c) { return gg::launch_passes<c>(a, st); });
}
