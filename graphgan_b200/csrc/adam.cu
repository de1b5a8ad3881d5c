// adam.cu -- K3: TF1.8 AdamOptimizer "sparse" apply, which is dense (sm_90a).
//
// generator.py:30-31 / discriminator.py:31-32 call tf.train.AdamOptimizer(lr).minimize(loss)
// on variables whose gradients are IndexedSlices.  TF 1.8's _apply_sparse_shared does
//     m <- m * beta1;  m[idx] += (1 - beta1) * g          (every row decays)
//     v <- v * beta2;  v[idx] += (1 - beta2) * g * g
//     var <- var - lr_t * m / (sqrt(v) + eps)              (every row moves)
// with lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t) computed by the host wrapper.  So one
// 64-pair step streams all of E, m, v: 24 * N * ld bytes -- a pure HBM-bandwidth kernel.
// A warp sweeps 512-byte segments, two in flight, 32 warps per SM (update_dev.cuh: adam_rows; the IEEE div / sqrt
// chains of the update are what the warps wait on -- ncu: fixed-latency dependency stalls -- so occupancy beats
// deeper unrolling: 4 in flight at 112 registers ran at 45 % of DRAM peak); the row -> gradient-slot map
// written by gg_pair_grad tells whether the row has a gradient, and is reset here.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "update_dev.cuh"

namespace gg {
namespace {

__global__ void __launch_bounds__(256, 4) adam_kernel(long long n_node, int ld, float *__restrict__ emb,
                                                   float *__restrict__ m_emb, float *__restrict__ v_emb,
                                                   float *__restrict__ bias, float *__restrict__ m_bias,
                                                   float *__restrict__ v_bias, const float *__restrict__ grad_rows,
                                                   const float *__restrict__ grad_bias, int *__restrict__ row_slot,
                                                   float lr_t, float b1, float b2, float eps) {
    adam_rows<false, 2>(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, grad_rows, grad_bias, row_slot, lr_t, b1, b2, eps);
}

// ld = 512: a row is four segments, so a warp keeps four in flight -- the whole row.  The lane that clears the row's slot
// then does so after every lane that reads the slot has read it (the __syncwarp in adam_rows); with two segments per warp
// the other half of the row would belong to another warp, which could find the slot already cleared.  (Four segments in
// flight need the registers of 2 CTAs per SM; at 4 the kernel spills.)
__global__ void __launch_bounds__(256, 2) adam_wide_kernel(long long n_node, int ld, float *__restrict__ emb,
                                                        float *__restrict__ m_emb, float *__restrict__ v_emb,
                                                        float *__restrict__ bias, float *__restrict__ m_bias,
                                                        float *__restrict__ v_bias, const float *__restrict__ grad_rows,
                                                        const float *__restrict__ grad_bias, int *__restrict__ row_slot,
                                                        float lr_t, float b1, float b2, float eps) {
    adam_rows<false, ADAM_WIDE_UNR>(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, grad_rows, grad_bias, row_slot, lr_t, b1,
                                    b2, eps);
}

// ---------------------------------------------------------------- the same sweep with TMA bulk copies (sm_90+)
// The sweep is a pure stream (24 * N * ld bytes per step), so it is fed by the copy engine instead of per-thread loads:
// one elected thread issues cp.async.bulk (global -> shared, completion on an mbarrier) for a tile of E, m and v, all
// 256 threads update the tile in shared memory (the identical per-element operation sequence as adam_rows), and one
// thread sends it back with cp.async.bulk (shared -> global).  Two tiles load, one computes and one stores per CTA, so the
// IEEE div / sqrt chains of one tile overlap the transfers of the next ones with no registers spent on the pipeline.
constexpr int ADAM_TILE = 2048;                   // floats per array per tile (8 KB): 64 / 32 / 16 / 8 rows
constexpr int ADAM_STAGES = 4;
constexpr size_t ADAM_TMA_SMEM = (size_t)ADAM_STAGES * 3 * ADAM_TILE * 4 + 64;   // + the full / done mbarriers

template <int ADAM_THREADS, int MINB>
__global__ void __launch_bounds__(ADAM_THREADS, MINB)
adam_tma_kernel(long long n_node, int ld, float *__restrict__ emb, float *__restrict__ m_emb, float *__restrict__ v_emb,
                float *__restrict__ bias, float *__restrict__ m_bias, float *__restrict__ v_bias,
                const float *__restrict__ grad_rows, const float *__restrict__ grad_bias, int *__restrict__ row_slot,
                float lr_t, float b1, float b2, float eps) {
    extern __shared__ __align__(128) unsigned char adam_smem[];
    float *buf = reinterpret_cast<float *>(adam_smem);                       // [STAGES][3][TILE]
    unsigned long long *full = reinterpret_cast<unsigned long long *>(adam_smem + (size_t)ADAM_STAGES * 3 * ADAM_TILE * 4);
    const int tid = threadIdx.x;
    const long long total = n_node * (long long)ld;
    const long long n_tiles = (total + ADAM_TILE - 1) / ADAM_TILE;
    const long long my_tiles = (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const float omb1 = 1.0f - b1, omb2 = 1.0f - b2;
    const int rows_per_tile = ADAM_TILE / ld;
    if (tid == 0) {
        for (int s = 0; s < ADAM_STAGES; ++s) mbar_init(full + s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](long long k) {               // thread 0: the three loads of my k-th tile
        const int s = (int)(k % ADAM_STAGES);
        const long long t = blockIdx.x + k * gridDim.x;
        const long long at = t * ADAM_TILE;
        const unsigned bytes = (unsigned)(((total - at) < ADAM_TILE ? (total - at) : ADAM_TILE) * 4);
        float *sb = buf + (size_t)s * 3 * ADAM_TILE;
        mbar_expect_tx(full + s, 3 * bytes);
        bulk_g2s(sb, emb + at, bytes, full + s);
        bulk_g2s(sb + ADAM_TILE, m_emb + at, bytes, full + s);
        bulk_g2s(sb + 2 * ADAM_TILE, v_emb + at, bytes, full + s);
    };
    if (tid == 0)
        for (long long k = 0; k < ADAM_STAGES - 2 && k < my_tiles; ++k) issue(k);
    for (long long k = 0; k < my_tiles; ++k) {
        const int s = (int)(k % ADAM_STAGES);
        const unsigned parity = (unsigned)((k / ADAM_STAGES) & 1);
        if (tid == 0 && k + ADAM_STAGES - 2 < my_tiles) {
            // the stage about to be refilled held tile k - 2, stored two iterations ago: the copy engine must have
            // finished READING it; the store of tile k - 1 may still be in flight (one pending group allowed)
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            issue(k + ADAM_STAGES - 2);
        }
        const long long t = blockIdx.x + k * gridDim.x;
        const long long at = t * ADAM_TILE;
        const int nfl = (int)((total - at) < ADAM_TILE ? (total - at) : ADAM_TILE);
        const long long row0 = at / ld;
        float *sx = buf + (size_t)s * 3 * ADAM_TILE, *sm = sx + ADAM_TILE, *sv = sx + 2 * ADAM_TILE;
        // slots of my rows (independent of the tile data: issued before the wait)
        int slot[ADAM_TILE / (4 * ADAM_THREADS)];
#pragma unroll
        for (int p = 0; p < ADAM_TILE / (4 * ADAM_THREADS); ++p) {
            const int e = 4 * (tid + ADAM_THREADS * p);
            slot[p] = (e < nfl) ? row_slot[row0 + e / ld] : -1;
        }
        mbar_wait(full + s, parity);
#define GG_ADAM_E(f)                                                                                  \
    m4.f = __fadd_rn(__fmul_rn(m4.f, b1), __fmul_rn(omb1, g.f));                                      \
    v4.f = __fadd_rn(__fmul_rn(v4.f, b2), __fmul_rn(__fmul_rn(g.f, g.f), omb2));                      \
    x4.f = __fsub_rn(x4.f, __fdiv_rn(__fmul_rn(lr_t, m4.f), __fadd_rn(__fsqrt_rn(v4.f), eps)));
#pragma unroll
        for (int p = 0; p < ADAM_TILE / (4 * ADAM_THREADS); ++p) {
            const int e = 4 * (tid + ADAM_THREADS * p);
            if (e >= nfl) continue;
            const int r = e / ld, c = e - r * ld;
            float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
            if (slot[p] >= 0) g = *reinterpret_cast<const float4 *>(grad_rows + (size_t)slot[p] * ld + c);
            float4 x4 = *reinterpret_cast<float4 *>(sx + e), m4 = *reinterpret_cast<float4 *>(sm + e),
                   v4 = *reinterpret_cast<float4 *>(sv + e);
            GG_ADAM_E(x) GG_ADAM_E(y) GG_ADAM_E(z) GG_ADAM_E(w)
            *reinterpret_cast<float4 *>(sx + e) = x4;
            *reinterpret_cast<float4 *>(sm + e) = m4;
            *reinterpret_cast<float4 *>(sv + e) = v4;
            if (c == 0) {                         // this thread owns the row's bias (and its slot, cleared below)
                const long long row = row0 + r;
                const float gb = slot[p] >= 0 ? grad_bias[slot[p]] : 0.0f;
                const float mm = __fadd_rn(__fmul_rn(m_bias[row], b1), __fmul_rn(omb1, gb));
                const float vv = __fadd_rn(__fmul_rn(v_bias[row], b2), __fmul_rn(__fmul_rn(gb, gb), omb2));
                m_bias[row] = mm; v_bias[row] = vv;
                bias[row] = __fsub_rn(bias[row], __fdiv_rn(__fmul_rn(lr_t, mm), __fadd_rn(__fsqrt_rn(vv), eps)));
            }
        }
#undef GG_ADAM_E
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // my shared-memory writes -> visible to the copy engine
        __syncthreads();                                                 // (also: every thread has read its rows' slots)
#pragma unroll
        for (int p = 0; p < ADAM_TILE / (4 * ADAM_THREADS); ++p) {
            const int e = 4 * (tid + ADAM_THREADS * p);
            if (e < nfl && slot[p] >= 0 && e % ld == 0) row_slot[row0 + e / ld] = -1;
        }
        if (tid == 0) {
            bulk_s2g(emb + at, sx, (unsigned)nfl * 4);
            bulk_s2g(m_emb + at, sm, (unsigned)nfl * 4);
            bulk_s2g(v_emb + at, sv, (unsigned)nfl * 4);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        (void)rows_per_tile;
    }
    if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all stores complete before the CTA retires
}

// ---------------------------------------------------------------- warp-specialised TMA sweep
// The CTA-wide barrier per tile of adam_tma_kernel serialises load -> compute -> store; here one PRODUCER warp owns the
// copy engine (loads two tiles ahead, stores two tiles behind) and NCW consumer warps only ever wait on mbarriers:
//   full[s]  (count 1 + tx bytes) : tile s has landed           producer -> consumers
//   done[s]  (count NCW)          : every consumer warp is done   consumers -> producer (which then stores the tile)
// so the div / sqrt chains of one tile overlap the transfers of the neighbouring ones without any thread idling at a
// block barrier.  The row -> slot map is read by the consumers before they wait and cleared by the producer warp once
// the tile is done (no consumer of that tile can still need it).
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <int NCW, int MINB>
__global__ void __launch_bounds__((NCW + 1) * 32, MINB)
adam_ws_kernel(long long n_node, int ld, float *__restrict__ emb, float *__restrict__ m_emb, float *__restrict__ v_emb,
               float *__restrict__ bias, float *__restrict__ m_bias, float *__restrict__ v_bias,
               const float *__restrict__ grad_rows, const float *__restrict__ grad_bias, int *__restrict__ row_slot,
               float lr_t, float b1, float b2, float eps) {
    constexpr int NCT = NCW * 32, LAG = 2;
    constexpr int PER = ADAM_TILE / (4 * NCT);                           // float4 per consumer thread per array per tile
    static_assert(PER >= 1 && PER * 4 * NCT == ADAM_TILE, "tile must split evenly over the consumer threads");
    extern __shared__ __align__(128) unsigned char adam_smem[];
    float *buf = reinterpret_cast<float *>(adam_smem);                   // [STAGES][3][TILE]
    unsigned long long *full = reinterpret_cast<unsigned long long *>(adam_smem + (size_t)ADAM_STAGES * 3 * ADAM_TILE * 4);
    unsigned long long *done = full + ADAM_STAGES;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long total = n_node * (long long)ld;
    const long long n_tiles = (total + ADAM_TILE - 1) / ADAM_TILE;
    const long long my_tiles = (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (tid == 0) {
        for (int s = 0; s < ADAM_STAGES; ++s) { mbar_init(full + s, 1); mbar_init(done + s, NCW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (wid == NCW) {
        // ---------------- producer warp
        for (long long it = 0; it < my_tiles + LAG; ++it) {
            if (it < my_tiles && lane == 0) {
                if (it >= ADAM_STAGES) asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(ADAM_STAGES - 1 - LAG) : "memory");
                const int s = (int)(it % ADAM_STAGES);
                const long long at = (blockIdx.x + it * gridDim.x) * (long long)ADAM_TILE;
                const unsigned bytes = (unsigned)(((total - at) < ADAM_TILE ? (total - at) : ADAM_TILE) * 4);
                float *sb = buf + (size_t)s * 3 * ADAM_TILE;
                mbar_expect_tx(full + s, 3 * bytes);
                bulk_g2s(sb, emb + at, bytes, full + s);
                bulk_g2s(sb + ADAM_TILE, m_emb + at, bytes, full + s);
                bulk_g2s(sb + 2 * ADAM_TILE, v_emb + at, bytes, full + s);
            }
            const long long j = it - LAG;
            if (j >= 0) {
                const int s = (int)(j % ADAM_STAGES);
                mbar_wait(done + s, (unsigned)((j / ADAM_STAGES) & 1));
                const long long at = (blockIdx.x + j * gridDim.x) * (long long)ADAM_TILE;
                const int nfl = (int)((total - at) < ADAM_TILE ? (total - at) : ADAM_TILE);
                const long long row0 = at / ld;
                for (int r = lane; r < nfl / ld; r += 32)            // the tile's gradient slots are consumed: clear them
                    if (row_slot[row0 + r] >= 0) row_slot[row0 + r] = -1;
                if (lane == 0) {
                    float *sb = buf + (size_t)s * 3 * ADAM_TILE;
                    bulk_s2g(emb + at, sb, (unsigned)nfl * 4);
                    bulk_s2g(m_emb + at, sb + ADAM_TILE, (unsigned)nfl * 4);
                    bulk_s2g(v_emb + at, sb + 2 * ADAM_TILE, (unsigned)nfl * 4);
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
            }
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        return;
    }
    // ---------------- consumer warps
    const float omb1 = 1.0f - b1, omb2 = 1.0f - b2;
    for (long long k = 0; k < my_tiles; ++k) {
        const int s = (int)(k % ADAM_STAGES);
        const long long at = (blockIdx.x + k * gridDim.x) * (long long)ADAM_TILE;
        const int nfl = (int)((total - at) < ADAM_TILE ? (total - at) : ADAM_TILE);
        const long long row0 = at / ld;
        float *sx = buf + (size_t)s * 3 * ADAM_TILE, *sm = sx + ADAM_TILE, *sv = sx + 2 * ADAM_TILE;
        int slot[PER];
#pragma unroll
        for (int p = 0; p < PER; ++p) {
            const int e = 4 * (tid + NCT * p);
            slot[p] = (e < nfl) ? row_slot[row0 + e / ld] : -1;
        }
        mbar_wait(full + s, (unsigned)((k / ADAM_STAGES) & 1));
#define GG_ADAM_E(f)                                                                                  \
    m4.f = __fadd_rn(__fmul_rn(m4.f, b1), __fmul_rn(omb1, g.f));                                      \
    v4.f = __fadd_rn(__fmul_rn(v4.f, b2), __fmul_rn(__fmul_rn(g.f, g.f), omb2));                      \
    x4.f = __fsub_rn(x4.f, __fdiv_rn(__fmul_rn(lr_t, m4.f), __fadd_rn(__fsqrt_rn(v4.f), eps)));
#pragma unroll
        for (int p = 0; p < PER; ++p) {
            const int e = 4 * (tid + NCT * p);
            if (e >= nfl) continue;
            const int r = e / ld, c = e - r * ld;
            float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
            if (slot[p] >= 0) g = *reinterpret_cast<const float4 *>(grad_rows + (size_t)slot[p] * ld + c);
            float4 x4 = *reinterpret_cast<float4 *>(sx + e), m4 = *reinterpret_cast<float4 *>(sm + e),
                   v4 = *reinterpret_cast<float4 *>(sv + e);
            GG_ADAM_E(x) GG_ADAM_E(y) GG_ADAM_E(z) GG_ADAM_E(w)
            *reinterpret_cast<float4 *>(sx + e) = x4;
            *reinterpret_cast<float4 *>(sm + e) = m4;
            *reinterpret_cast<float4 *>(sv + e) = v4;
            if (c == 0) {                         // this thread owns the row's bias
                const long long row = row0 + r;
                const float gb = slot[p] >= 0 ? grad_bias[slot[p]] : 0.0f;
                const float mm = __fadd_rn(__fmul_rn(m_bias[row], b1), __fmul_rn(omb1, gb));
                const float vv = __fadd_rn(__fmul_rn(v_bias[row], b2), __fmul_rn(__fmul_rn(gb, gb), omb2));
                m_bias[row] = mm; v_bias[row] = vv;
                bias[row] = __fsub_rn(bias[row], __fdiv_rn(__fmul_rn(lr_t, mm), __fadd_rn(__fsqrt_rn(vv), eps)));
            }
        }
#undef GG_ADAM_E
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // my shared-memory writes -> visible to the copy engine
        __syncwarp();
        if (lane == 0) mbar_arrive(done + s);
    }
}

// ---------------------------------------------------------------- dense-gradient step of the exact game (DESIGN.md 5.5)
// The sweep of adam_rows with a gradient for every element: the fp64 accumulators that gg_game_value_grad{,_d} fill,
// g = f32(scale * acc + lambda * x) in fp64 (mul, mul, add: no contraction), then the GG_ADAM1 sequence.  A pure stream
// of 32 bytes per element (acc 8, E / m / v 24).  A warp owns segments of 32 float4 (the element order of adam_rows)
// and keeps UNR of them in flight; the lane holding a row's first columns also steps the row's bias.
template <int UNR>
__device__ __forceinline__ void adam_dense_rows(long long n_node, int ld, float *emb, float *m_emb, float *v_emb,
                                                float *bias, float *m_bias, float *v_bias, const double *acc_emb,
                                                const double *acc_bias, double scale, float lam_e, float lam_b,
                                                float lr_t, float b1, float b2, float eps) {
    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const float omb1 = 1.0f - b1, omb2 = 1.0f - b2;
    const int q = ld >> 2, qs = __ffs(q) - 1;     // float4 per row (a power of two) and its log2
    const long long n4 = n_node * q;              // float4 in the whole matrix
    const long long nseg = (n4 + 31) >> 5;
    const double le = (double)lam_e, lb = (double)lam_b;
#define GG_DENSE_G(a, xx) __double2float_rn(__dadd_rn(__dmul_rn(scale, (a)), __dmul_rn(le, (double)(xx))))
#define GG_ADAM1(f)                                                                                   \
    m[k].f = __fadd_rn(__fmul_rn(m[k].f, b1), __fmul_rn(omb1, g.f));                                  \
    v[k].f = __fadd_rn(__fmul_rn(v[k].f, b2), __fmul_rn(__fmul_rn(g.f, g.f), omb2));                  \
    x[k].f = __fsub_rn(x[k].f, __fdiv_rn(__fmul_rn(lr_t, m[k].f), __fadd_rn(__fsqrt_rn(v[k].f), eps)));
    for (long long s0 = warp * UNR; s0 < nseg; s0 += nwarps * UNR) {
        long long e4[UNR];                         // my float4 of segment s0 + k, or -1
        float4 m[UNR], v[UNR], x[UNR];
        double2 a0[UNR], a1[UNR];
#pragma unroll
        for (int k = 0; k < UNR; ++k) {
            const long long e = ((s0 + k) << 5) + lane;
            e4[k] = (s0 + k < nseg && e < n4) ? e : -1;
            if (e4[k] >= 0) {
                const size_t at = (size_t)e << 2;
                m[k] = *reinterpret_cast<const float4 *>(m_emb + at);
                v[k] = *reinterpret_cast<const float4 *>(v_emb + at);
                x[k] = *reinterpret_cast<const float4 *>(emb + at);
                a0[k] = __ldg(reinterpret_cast<const double2 *>(acc_emb + at));
                a1[k] = __ldg(reinterpret_cast<const double2 *>(acc_emb + at + 2));
            }
        }
#pragma unroll
        for (int k = 0; k < UNR; ++k) {
            if (e4[k] < 0) continue;
            const size_t at = (size_t)e4[k] << 2;
            float4 g;
            g.x = GG_DENSE_G(a0[k].x, x[k].x); g.y = GG_DENSE_G(a0[k].y, x[k].y);
            g.z = GG_DENSE_G(a1[k].x, x[k].z); g.w = GG_DENSE_G(a1[k].y, x[k].w);
            GG_ADAM1(x) GG_ADAM1(y) GG_ADAM1(z) GG_ADAM1(w)
            *reinterpret_cast<float4 *>(m_emb + at) = m[k];
            *reinterpret_cast<float4 *>(v_emb + at) = v[k];
            *reinterpret_cast<float4 *>(emb + at) = x[k];
            if ((e4[k] & (q - 1)) == 0) {          // this lane holds the row's first columns: the bias
                const long long row = e4[k] >> qs;
                const float xb = bias[row];
                const float gb = __double2float_rn(__dadd_rn(__dmul_rn(scale, __ldg(acc_bias + row)), __dmul_rn(lb, (double)xb)));
                const float mm = __fadd_rn(__fmul_rn(m_bias[row], b1), __fmul_rn(omb1, gb));
                const float vv = __fadd_rn(__fmul_rn(v_bias[row], b2), __fmul_rn(__fmul_rn(gb, gb), omb2));
                m_bias[row] = mm; v_bias[row] = vv;
                bias[row] = __fsub_rn(xb, __fdiv_rn(__fmul_rn(lr_t, mm), __fadd_rn(__fsqrt_rn(vv), eps)));
            }
        }
    }
#undef GG_ADAM1
#undef GG_DENSE_G
}

__global__ void __launch_bounds__(256, 4) adam_dense_kernel(long long n_node, int ld, float *__restrict__ emb,
                                                         float *__restrict__ m_emb, float *__restrict__ v_emb,
                                                         float *__restrict__ bias, float *__restrict__ m_bias,
                                                         float *__restrict__ v_bias, const double *__restrict__ acc_emb,
                                                         const double *__restrict__ acc_bias, double scale, float lam_e,
                                                         float lam_b, float lr_t, float b1, float b2, float eps) {
    adam_dense_rows<2>(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, acc_emb, acc_bias, scale, lam_e, lam_b, lr_t,
                       b1, b2, eps);
}

// ld = 512 as adam_wide_kernel: a warp keeps four segments -- one whole row -- in flight, at 2 CTAs per SM.
__global__ void __launch_bounds__(256, 2) adam_dense_wide_kernel(long long n_node, int ld, float *__restrict__ emb,
                                                              float *__restrict__ m_emb, float *__restrict__ v_emb,
                                                              float *__restrict__ bias, float *__restrict__ m_bias,
                                                              float *__restrict__ v_bias,
                                                              const double *__restrict__ acc_emb,
                                                              const double *__restrict__ acc_bias, double scale,
                                                              float lam_e, float lam_b, float lr_t, float b1, float b2,
                                                              float eps) {
    adam_dense_rows<ADAM_WIDE_UNR>(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, acc_emb, acc_bias, scale, lam_e,
                                   lam_b, lr_t, b1, b2, eps);
}

// which sweep gg_adam_apply launches: 0 = per-thread loads (default: fastest measured), 1..3 = CTA-barrier TMA pipeline
// (512x2, 256x2, 512x3 threads x CTAs per SM), 4 / 5 = warp-specialised TMA pipeline with 16 / 8 consumer warps
int g_adam_path = -1;
int adam_path_from_name(const char *e) {
    if (!e) return 0;
    if (strcmp(e, "tma") == 0) return 1;
    if (strcmp(e, "tma256x2") == 0) return 2;
    if (strcmp(e, "tma512x3") == 0) return 3;
    if (strcmp(e, "ws16") == 0) return 4;
    if (strcmp(e, "ws8") == 0) return 5;
    return 0;
}

}  // namespace
}  // namespace gg

extern "C" int gg_set_adam_path(const char *name) {
    gg::g_adam_path = gg::adam_path_from_name(name);
    return 0;
}

extern "C" int gg_adam_apply(int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
                             float *m_bias, float *v_bias, const int32_t *n_unique, const int32_t *uniq_ids,
                             const float *grad_rows, const float *grad_bias, int32_t *row_slot, float lr_t, float beta1,
                             float beta2, float eps, void *stream) {
    (void)n_unique; (void)uniq_ids;
    if (gg::g_adam_path < 0) gg::g_adam_path = gg::adam_path_from_name(getenv("GG_ADAM_PATH"));
    const int use_tma = gg::g_adam_path;
    GG_REQUIRE(emb && m_emb && v_emb && bias && m_bias && v_bias && grad_rows && grad_bias && row_slot, "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    if (n_node == 0) return 0;
    if (use_tma) {
        const long long n_tiles = (n_node * (long long)ld + gg::ADAM_TILE - 1) / gg::ADAM_TILE;
        cudaStream_t st = (cudaStream_t)stream;
#define GG_ADAM_TMA(NT, MINB)                                                                                                   \
    do {                                                                                                                        \
        long long blocks = (long long)gg::sm_count() * MINB;                                                                    \
        if (blocks > n_tiles) blocks = n_tiles;                                                                                 \
        GG_CHECK(cudaFuncSetAttribute(gg::adam_tma_kernel<NT, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize,               \
                                      (int)gg::ADAM_TMA_SMEM));                                                                 \
        gg::adam_tma_kernel<NT, MINB><<<(unsigned)blocks, NT, gg::ADAM_TMA_SMEM, st>>>(                                         \
            n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, grad_rows, grad_bias, row_slot, lr_t, beta1, beta2, eps);      \
    } while (0)
        if (use_tma >= 4) {             // warp-specialised: 16 (or 8) consumer warps + 1 producer warp, 2 CTAs per SM
            long long blocks = (long long)gg::sm_count() * 2;
            if (blocks > n_tiles) blocks = n_tiles;
            if (use_tma == 4) {
                GG_CHECK(cudaFuncSetAttribute(gg::adam_ws_kernel<16, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg::ADAM_TMA_SMEM));
                gg::adam_ws_kernel<16, 2><<<(unsigned)blocks, 17 * 32, gg::ADAM_TMA_SMEM, st>>>(
                    n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, grad_rows, grad_bias, row_slot, lr_t, beta1, beta2, eps);
            } else {
                GG_CHECK(cudaFuncSetAttribute(gg::adam_ws_kernel<8, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg::ADAM_TMA_SMEM));
                gg::adam_ws_kernel<8, 2><<<(unsigned)blocks, 9 * 32, gg::ADAM_TMA_SMEM, st>>>(
                    n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, grad_rows, grad_bias, row_slot, lr_t, beta1, beta2, eps);
            }
            return gg::check_cuda(cudaGetLastError(), "adam (warp-specialised TMA) kernel launch");
        }
        if (use_tma == 2) GG_ADAM_TMA(256, 2);
        else if (use_tma == 3) GG_ADAM_TMA(512, 3);
        else GG_ADAM_TMA(512, 2);
#undef GG_ADAM_TMA
        return gg::check_cuda(cudaGetLastError(), "adam (TMA) kernel launch");
    }
    const int q = ld / 4;                                                       // float4 per row
    const long long nseg = q >= 32 ? n_node * (q / 32) : (n_node + 32 / q - 1) / (32 / q);   // 512-byte segments
    if (ld == gg::LD_MAX) {                                                     // 8 warps x 4 segments (one row each)
        long long blocks = (nseg + 4 * 8 - 1) / (4 * 8);
        const long long cap = (long long)gg::sm_count() * 16;
        if (blocks > cap) blocks = cap;
        gg::adam_wide_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n_node, ld, emb, m_emb, v_emb, bias, m_bias,
                                                                                 v_bias, grad_rows, grad_bias, row_slot, lr_t,
                                                                                 beta1, beta2, eps);
        return gg::check_cuda(cudaGetLastError(), "adam kernel launch");
    }
    long long blocks = (nseg + 2 * 8 - 1) / (2 * 8);                            // 8 warps x 2 segments in flight
    const long long cap = (long long)gg::sm_count() * 16;
    if (blocks > cap) blocks = cap;
    gg::adam_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n_node, ld, emb, m_emb, v_emb, bias, m_bias,
                                                                        v_bias, grad_rows, grad_bias, row_slot, lr_t,
                                                                        beta1, beta2, eps);
    return gg::check_cuda(cudaGetLastError(), "adam kernel launch");
}

extern "C" int gg_adam_apply_dense(int64_t n_node, int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias,
                                   float *m_bias, float *v_bias, const double *acc_emb, const double *acc_bias,
                                   double scale, float lambda_emb, float lambda_bias, float lr_t, float beta1,
                                   float beta2, float eps, void *stream) {
    GG_REQUIRE(emb && m_emb && v_emb && bias && m_bias && v_bias && acc_emb && acc_bias, "null pointer");
    GG_REQUIRE(n_node > 0, "n_node must be positive");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(isfinite(scale), "scale must be finite");
    const long long nseg = (n_node * (ld / 4) + 31) / 32;                      // 512-byte segments
    const int unr = ld == gg::LD_MAX ? gg::ADAM_WIDE_UNR : 2;
    long long blocks = (nseg + unr * 8 - 1) / (unr * 8);                         // 8 warps x unr segments in flight
    const long long cap = (long long)gg::sm_count() * 16;
    if (blocks > cap) blocks = cap;
    if (ld == gg::LD_MAX)
        gg::adam_dense_wide_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
            n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, acc_emb, acc_bias, scale, lambda_emb, lambda_bias, lr_t,
            beta1, beta2, eps);
    else
        gg::adam_dense_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
            n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, acc_emb, acc_bias, scale, lambda_emb, lambda_bias, lr_t,
            beta1, beta2, eps);
    return gg::check_cuda(cudaGetLastError(), "adam (dense gradient) kernel launch");
}
