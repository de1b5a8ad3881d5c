// steps.cu -- the reference's per-batch loop (graph_gan.py:149-157, 168-176) driven from C.
//
// One 64-pair step is two tiny launches (K2 pair_grad, K3 adam); at config C1 an epoch is ~230 k of them, so
// the host-language overhead per step (argument marshalling, tensor slicing) would dominate.  This entry point
// walks the caller's shuffled start list and enqueues every step on the stream; nothing synchronises.
#include <math.h>
#include <string.h>

#include "update_dev.cuh"

extern "C" int gg_train_steps(int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts, int32_t batch_size,
                              const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node,
                              int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias,
                              float lambda, int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias,
                              int32_t *row_slot, float lr, float beta1, float beta2, float eps, float *beta1_power,
                              float *beta2_power, void *stream) {
    GG_REQUIRE(batch_size > 0 && batch_size <= GG_MAX_BATCH, "batch size out of range");
    return gg_train_steps_ex(mode, n_rows, start_list, n_starts, batch_size, node_id, node_neighbor_id, aux, n_node, ld, emb,
                             m_emb, v_emb, bias, m_bias, v_bias, lambda, n_unique, uniq_ids, grad_rows, grad_bias, row_slot, lr,
                             beta1, beta2, eps, beta1_power, beta2_power, nullptr, 0, stream);
}

extern "C" int gg_train_steps_ex(int32_t mode, int64_t n_rows, const int64_t *start_list, int64_t n_starts, int32_t batch_size,
                                 const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node,
                                 int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias,
                                 float lambda, int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias,
                                 int32_t *row_slot, float lr, float beta1, float beta2, float eps, float *beta1_power,
                                 float *beta2_power, void *scratch, int64_t scratch_bytes, void *stream) {
    GG_REQUIRE(start_list && beta1_power && beta2_power, "null host pointer");
    GG_REQUIRE(batch_size > 0, "batch size out of range");
    for (int64_t s = 0; s < n_starts; ++s) {
        const int64_t start = start_list[s];
        GG_REQUIRE(start >= 0 && start < n_rows, "start out of range");
        const int64_t end = start + batch_size < n_rows ? start + batch_size : n_rows;
        int rc = gg_pair_grad_ex(mode, (int32_t)(end - start), 0, node_id + start, node_neighbor_id + start, aux + start, emb,
                                 bias, ld, lambda, n_unique, uniq_ids, grad_rows, grad_bias, row_slot, scratch, scratch_bytes, 0,
                                 stream);
        if (rc) return rc;
        // lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t), fp32 step by step like the TF graph (and model.py)
        volatile float one_m_b2 = 1.0f - *beta2_power;
        volatile float root = sqrtf(one_m_b2);
        volatile float num = lr * root;
        volatile float den = 1.0f - *beta1_power;
        const float lr_t = num / den;
        rc = gg_adam_apply(n_node, ld, emb, m_emb, v_emb, bias, m_bias, v_bias, n_unique, uniq_ids, grad_rows, grad_bias,
                           row_slot, lr_t, beta1, beta2, eps, stream);
        if (rc) return rc;
        volatile float p1 = *beta1_power * beta1, p2 = *beta2_power * beta2;
        *beta1_power = p1;
        *beta2_power = p2;
    }
    return 0;
}

// ---------------------------------------------------------------- persistent step loop (f3)
// The same steps as above in ONE cooperative launch (co-residency is what the cooperative launch buys; the
// barriers are hand-rolled because the dependence is one-to-all then all-to-one, not all-to-all):
//   CTA 0 computes the mini-batch gradient (K2 body) and publishes `ready = s+1` (release store);
//   every CTA waits for that flag (acquire load), runs its share of the dense Adam sweep (K3 body) and
//   adds 1 to `done` (release add);  CTA 0 alone waits for done == gridDim.x*(s+1) before the next gradient.
// Parameters written in one step are read in the next by another SM, so cross-SM reads go through L2 (the
// COH = true bodies); a row of m/v/emb is always swept by the same warp.  Bit-identical to gg_train_steps.
namespace gg {
namespace {

struct LoopArgs {
    int mode, batch_size, ld;
    long long n_rows, n_starts, n_node;
    const long long *starts;
    const int *node_id, *node_neighbor_id;
    const float *aux;
    float *emb, *m_emb, *v_emb, *bias, *m_bias, *v_bias;
    float *emb2, *bias2;               // fused loop only: the second parameter buffers of the ping-pong
    float lambda;
    int *n_unique, *uniq_ids;
    float *grad_rows, *grad_bias;
    int *row_slot;
    float lr, beta1, beta2, eps, beta1_power, beta2_power;
    unsigned long long *sync_words;    // [0] ready (steps whose gradient is published), [1] done (CTA arrivals),
                                       // [2..5] CTA 0's cycles in gradient / sweep / wait and the step count (diagnostic)
};

__device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void add_release(unsigned long long *p, unsigned long long v) {
    asm volatile("red.release.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// SWEEP_UNR: segments per warp of the sweep (adam_rows); ld = 512 needs ADAM_WIDE_UNR (the warp clears the rows' slots)
template <int NT, int SWEEP_UNR>
__device__ __forceinline__ void train_loop_body(const LoopArgs &a) {
    extern __shared__ int smem[];
    unsigned long long *ready = a.sync_words, *done = a.sync_words + 1;
    float b1p = a.beta1_power, b2p = a.beta2_power;
    const bool clk = blockIdx.x == 0 && threadIdx.x == 0;     // CTA 0 keeps a cycle breakdown (diagnostic)
    long long c_grad = 0, c_sweep = 0, c_wait = 0;
    for (long long s = 0; s < a.n_starts; ++s) {
        const long long t0 = clk ? clock64() : 0;
        if (blockIdx.x == 0) {
            const long long start = a.starts[s];
            const long long end = start + a.batch_size < a.n_rows ? start + a.batch_size : a.n_rows;
            pair_grad_body<true, NT>(smem, a.mode, (int)(end - start), (int)(end - start), a.node_id + start, a.node_neighbor_id + start,
                                     a.aux + start, a.emb, a.bias, a.ld, a.lambda, a.n_unique, a.uniq_ids, a.grad_rows, a.grad_bias,
                                     a.row_slot);
            __syncthreads();
            if (threadIdx.x == 0) st_release(ready, (unsigned long long)(s + 1));
        } else {
            if (threadIdx.x == 0) while (ld_acquire(ready) < (unsigned long long)(s + 1)) {}
            __syncthreads();
        }
        const long long t1 = clk ? clock64() : 0;
        // lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t): the same fp32 operation sequence as the host loop
        const float lr_t = __fdiv_rn(__fmul_rn(a.lr, __fsqrt_rn(__fsub_rn(1.0f, b2p))), __fsub_rn(1.0f, b1p));
        adam_rows<true, SWEEP_UNR, false>(a.n_node, a.ld, a.emb, a.m_emb, a.v_emb, a.bias, a.m_bias, a.v_bias, a.grad_rows, a.grad_bias,
                                  a.row_slot, lr_t, a.beta1, a.beta2, a.eps);
        b1p = __fmul_rn(b1p, a.beta1);
        b2p = __fmul_rn(b2p, a.beta2);
        __syncthreads();
        const long long t2 = clk ? clock64() : 0;
        if (threadIdx.x == 0) {
            add_release(done, 1ull);
            if (blockIdx.x == 0) while (ld_acquire(done) < (unsigned long long)gridDim.x * (unsigned long long)(s + 1)) {}
        }
        if (blockIdx.x == 0) __syncthreads();
        if (clk) { c_grad += t1 - t0; c_sweep += t2 - t1; c_wait += clock64() - t2; }
    }
    if (clk) {
        a.sync_words[2] = (unsigned long long)c_grad; a.sync_words[3] = (unsigned long long)c_sweep;
        a.sync_words[4] = (unsigned long long)c_wait; a.sync_words[5] = (unsigned long long)a.n_starts;
    }
}
template <int NT>
__global__ void __launch_bounds__(NT, 1) train_loop_kernel(const __grid_constant__ LoopArgs a) { train_loop_body<NT, 2>(a); }
template <int NT>
__global__ void __launch_bounds__(NT, 1) train_loop_wide_kernel(const __grid_constant__ LoopArgs a) {
    train_loop_body<NT, ADAM_WIDE_UNR>(a);
}

// ---------------------------------------------------------------- fused step loop
// One barrier per step instead of two.  EVERY CTA runs the forward pass and the unique/list construction of the
// mini-batch redundantly (64 pairs: ~32 KB of rows from L2, identical results everywhere), then sweeps the rows it
// owns; for an owned row with a gradient the sweeping lane accumulates its own columns of the segment sum from
// the entry list (the same additions in the same order as pair_sums) and applies Adam at once.  Nothing is
// published between CTAs except the parameters themselves, which ping-pong between two buffers: step s reads
// (emb, bias) of parity s and writes parity s+1 -- the sweep writes every row, and a CTA that is already sweeping
// cannot disturb a CTA that is still in its forward pass.  The barrier at the end of the step is the only
// inter-CTA synchronisation.  m / v are updated in place (only their owner touches them).
template <int NT, int UNR>
__global__ void __launch_bounds__(NT, 1) train_fused_kernel(const __grid_constant__ LoopArgs a) {
    extern __shared__ int smem[];
    static_assert(UNR % 2 == 0, "both halves of a 256-wide row must be in flight in the same warp");
    constexpr int W = NT / 32;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    int *lslot = smem + 11 * a.batch_size + 8;   // [iters * RPC] owned row (local index) -> slot of this step, or -1
    const int ld = a.ld, q = ld >> 2;
    const int rps = q >= 32 ? 1 : 32 / q, halves = q > 32 ? q / 32 : 1;
    const long long nseg = ((a.n_node + rps - 1) / rps) * halves;
    const int sub = q >= 32 ? 0 : lane / q;
    const int col = q >= 32 ? 4 * lane : 4 * (lane % q);
    const int G = gridDim.x;
    const int RPC = W * UNR * rps / halves;                    // rows of one (CTA, iteration) chunk
    const long long seg_round = (long long)G * W * UNR;
    const int iters = (int)((nseg + seg_round - 1) / seg_round);
    const int tab_n = iters * RPC;
    unsigned long long *done = a.sync_words + 1;
    float b1p = a.beta1_power, b2p = a.beta2_power;
    const float b1 = a.beta1, b2 = a.beta2, omb1 = 1.0f - b1, omb2 = 1.0f - b2, eps = a.eps, lambda = a.lambda;
    const bool clk = blockIdx.x == 0 && tid == 0;
    long long c_grad = 0, c_sweep = 0, c_wait = 0;
    for (long long s = 0; s < a.n_starts; ++s) {
        const long long t0 = clk ? clock64() : 0;
        const float *E_old = (s & 1) ? a.emb2 : a.emb, *b_old = (s & 1) ? a.bias2 : a.bias;
        float *E_new = (s & 1) ? a.emb : a.emb2, *b_new = (s & 1) ? a.bias : a.bias2;
        const long long start = a.starts[s];
        const int B = (int)((start + a.batch_size < a.n_rows ? start + a.batch_size : a.n_rows) - start);
        for (int i = tid; i < tab_n; i += NT) lslot[i] = -1;
        pair_lists<true, NT>(smem, a.mode, B, B, a.node_id + start, a.node_neighbor_id + start, a.aux + start, E_old, b_old, ld,
                             nullptr, nullptr, nullptr);
        const PairSmem ps = pair_smem(smem, B);
        for (int t = tid; t < 2 * B; t += NT)
            if (ps.rnk[t] == 0) {                              // first occurrence of its row
                const int row = ps.ids[t];
                const long long chunk = row / RPC;
                if ((int)(chunk % G) == (int)blockIdx.x) lslot[(int)(chunk / G) * RPC + row % RPC] = ps.slot[t];
            }
        __syncthreads();
        const long long t1 = clk ? clock64() : 0;
        // lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t): the same fp32 operation sequence as the host loop
        const float lr_t = __fdiv_rn(__fmul_rn(a.lr, __fsqrt_rn(__fsub_rn(1.0f, b2p))), __fsub_rn(1.0f, b1p));
#define GG_ADAM1(f)                                                                                   \
    m[k].f = __fadd_rn(__fmul_rn(m[k].f, b1), __fmul_rn(omb1, g.f));                                  \
    v[k].f = __fadd_rn(__fmul_rn(v[k].f, b2), __fmul_rn(__fmul_rn(g.f, g.f), omb2));                  \
    x[k].f = __fsub_rn(x[k].f, __fdiv_rn(__fmul_rn(lr_t, m[k].f), __fadd_rn(__fsqrt_rn(v[k].f), eps)));
#define GG_ACC(f) g.f = __fadd_rn(g.f, __fadd_rn(__fmul_rn(dd[e], o[e].f), __fmul_rn(lambda, x[k].f)))
        for (int it = 0; it < iters; ++it) {
            const long long s0 = ((long long)it * G + blockIdx.x) * (W * UNR) + (long long)wid * UNR;
            int row[UNR], cc[UNR], slot[UNR];
            float4 m[UNR], v[UNR], x[UNR];
            float xb[UNR], mb[UNR], vb[UNR];
            // every load that does not depend on another load is issued here: parameters, Adam slots, the bias triple
#pragma unroll
            for (int k = 0; k < UNR; ++k) {
                const long long seg = s0 + k;
                const long long r = (seg / halves) * rps + sub;
                cc[k] = col + 128 * (int)(seg % halves);
                row[k] = (seg < nseg && r < a.n_node) ? (int)r : -1;
                slot[k] = -1;
                xb[k] = mb[k] = vb[k] = 0.0f;
                if (row[k] >= 0) {
                    const size_t at = (size_t)r * ld + cc[k];
                    slot[k] = lslot[it * RPC + (int)(r % RPC)];
                    m[k] = *reinterpret_cast<const float4 *>(a.m_emb + at);
                    v[k] = *reinterpret_cast<const float4 *>(a.v_emb + at);
                    x[k] = __ldcg(reinterpret_cast<const float4 *>(E_old + at));
                    if (cc[k] == 0) { xb[k] = __ldcg(b_old + r); mb[k] = a.m_bias[r]; vb[k] = a.v_bias[r]; }
                }
            }
#pragma unroll
            for (int k = 0; k < UNR; ++k) {
                if (row[k] < 0) continue;
                const size_t at = (size_t)row[k] * ld + cc[k];
                float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
                int lo = 0, n = 0;
                if (slot[k] >= 0) { lo = ps.off[slot[k]]; n = ps.off[slot[k] + 1] - lo; }
                for (int r2 = 0; r2 < n; r2 += 4) {            // pair_sums' additions for this lane's columns
                    float4 o[4];
                    float dd[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const bool in = r2 + e < n;
                        const int t = in ? ps.lst[lo + r2 + e] : 0;
                        o[e] = in ? __ldcg(reinterpret_cast<const float4 *>(E_old + (size_t)ps.ids[t < B ? t + B : t - B] * ld + cc[k]))
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
                        dd[e] = ps.delta[t < B ? t : t - B];
                    }
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        if (r2 + e >= n) break;
                        GG_ACC(x); GG_ACC(y); GG_ACC(z); GG_ACC(w);
                    }
                }
                float gb = 0.0f;
                if (cc[k] == 0) {                               // this lane also owns the row's bias
                    for (int r2 = 0; r2 < n; ++r2) {            // j-side entries only; generator.py:28-29 has no bias l2
                        const int t = ps.lst[lo + r2];
                        if (t < B) continue;
                        const float d = ps.delta[t - B];
                        gb = __fadd_rn(gb, a.mode == 0 ? __fadd_rn(d, __fmul_rn(lambda, xb[k])) : d);
                    }
                }
                GG_ADAM1(x) GG_ADAM1(y) GG_ADAM1(z) GG_ADAM1(w)
                *reinterpret_cast<float4 *>(a.m_emb + at) = m[k];
                *reinterpret_cast<float4 *>(a.v_emb + at) = v[k];
                *reinterpret_cast<float4 *>(E_new + at) = x[k];
                if (cc[k] == 0) {
                    const float mm = __fadd_rn(__fmul_rn(mb[k], b1), __fmul_rn(omb1, gb));
                    const float vv = __fadd_rn(__fmul_rn(vb[k], b2), __fmul_rn(__fmul_rn(gb, gb), omb2));
                    a.m_bias[row[k]] = mm; a.v_bias[row[k]] = vv;
                    b_new[row[k]] = __fsub_rn(xb[k], __fdiv_rn(__fmul_rn(lr_t, mm), __fadd_rn(__fsqrt_rn(vv), eps)));
                }
            }
        }
#undef GG_ACC
#undef GG_ADAM1
        b1p = __fmul_rn(b1p, b1);
        b2p = __fmul_rn(b2p, b2);
        __syncthreads();
        const long long t2 = clk ? clock64() : 0;
        if (tid == 0) {
            add_release(done, 1ull);
            while (ld_acquire(done) < (unsigned long long)G * (unsigned long long)(s + 1)) {}
        }
        __syncthreads();
        if (clk) { c_grad += t1 - t0; c_sweep += t2 - t1; c_wait += clock64() - t2; }
    }
    if (clk) {
        a.sync_words[2] = (unsigned long long)c_grad; a.sync_words[3] = (unsigned long long)c_sweep;
        a.sync_words[4] = (unsigned long long)c_wait; a.sync_words[5] = (unsigned long long)a.n_starts;
    }
}
}  // namespace
}  // namespace gg

extern "C" int gg_train_loop(int32_t mode, int64_t n_rows, const int64_t *start_list_dev, int64_t n_starts, int32_t batch_size,
                             const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node,
                             int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias,
                             float lambda, int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias,
                             int32_t *row_slot, float lr, float beta1, float beta2, float eps, float *beta1_power,
                             float *beta2_power, uint64_t *sync_words, void *stream) {
    GG_REQUIRE(start_list_dev && beta1_power && beta2_power && sync_words, "null pointer");
    GG_REQUIRE(batch_size > 0 && batch_size <= GG_MAX_BATCH, "batch size out of range");
    GG_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (discriminator) or 1 (generator)");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    if (n_starts == 0) return 0;
    int dev = 0, coop = 0, per_sm = 0;
    GG_CHECK(cudaGetDevice(&dev));
    GG_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    GG_REQUIRE(coop, "device does not support cooperative launches");
    const size_t smem = gg::pair_grad_smem_bytes(batch_size);
    // 512 threads: the 64-register ceiling of a 1024-thread CTA makes the fused body spill (measured 18.7 vs 13.5 us/step)
    constexpr int NT = 512;
    const bool wide = ld == gg::LD_MAX;
    const void *kern = wide ? (const void *)gg::train_loop_wide_kernel<NT> : (const void *)gg::train_loop_kernel<NT>;
    GG_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, NT, smem));
    GG_REQUIRE(per_sm >= 1, "step loop kernel does not fit on an SM");
    // one sweep iteration per warp (2 segments of 512 B in flight), at most one CTA per SM
    long long ctas = (n_node + 63) / 64;
    if (ctas > gg::sm_count()) ctas = gg::sm_count();
    if (ctas < 1) ctas = 1;
    gg::LoopArgs a;
    a.mode = mode; a.batch_size = batch_size; a.ld = ld; a.n_rows = n_rows; a.n_starts = n_starts; a.n_node = n_node;
    a.starts = (const long long *)start_list_dev; a.node_id = node_id; a.node_neighbor_id = node_neighbor_id; a.aux = aux;
    a.emb = emb; a.m_emb = m_emb; a.v_emb = v_emb; a.bias = bias; a.m_bias = m_bias; a.v_bias = v_bias; a.lambda = lambda;
    a.n_unique = n_unique; a.uniq_ids = uniq_ids; a.grad_rows = grad_rows; a.grad_bias = grad_bias; a.row_slot = row_slot;
    a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.beta1_power = *beta1_power; a.beta2_power = *beta2_power;
    a.sync_words = (unsigned long long *)sync_words;
    GG_CHECK(cudaMemsetAsync(sync_words, 0, 8 * sizeof(uint64_t), (cudaStream_t)stream));
    void *args[] = {&a};
    GG_CHECK(cudaLaunchCooperativeKernel(kern, dim3((unsigned)ctas), dim3(NT), args,
                                         smem, (cudaStream_t)stream));
    // the accumulators advance deterministically: replay the fp32 products on the host
    for (int64_t s = 0; s < n_starts; ++s) {
        volatile float p1 = *beta1_power * beta1, p2 = *beta2_power * beta2;
        *beta1_power = p1;
        *beta2_power = p2;
    }
    return 0;
}

extern "C" int gg_train_fused(int32_t mode, int64_t n_rows, const int64_t *start_list_dev, int64_t n_starts, int32_t batch_size,
                              const int32_t *node_id, const int32_t *node_neighbor_id, const float *aux, int64_t n_node,
                              int32_t ld, float *emb, float *m_emb, float *v_emb, float *bias, float *m_bias, float *v_bias,
                              float *emb2, float *bias2, float lambda, float lr, float beta1, float beta2, float eps,
                              float *beta1_power, float *beta2_power, uint64_t *sync_words, void *stream) {
    GG_REQUIRE(start_list_dev && beta1_power && beta2_power && sync_words && emb2 && bias2, "null pointer");
    GG_REQUIRE(emb && m_emb && v_emb && bias && m_bias && v_bias && node_id && node_neighbor_id && aux, "null pointer");
    GG_REQUIRE(batch_size > 0 && batch_size <= GG_MAX_BATCH, "batch size out of range");
    GG_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (discriminator) or 1 (generator)");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    if (n_starts == 0) return 0;
    constexpr int NT = 512, UNR = 2, W = NT / 32;
    int dev = 0, coop = 0, per_sm = 0;
    GG_CHECK(cudaGetDevice(&dev));
    GG_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    GG_REQUIRE(coop, "device does not support cooperative launches");
    const int q = ld / 4, rps = q >= 32 ? 1 : 32 / q, halves = q > 32 ? q / 32 : 1;
    const long long nseg = ((n_node + rps - 1) / rps) * halves;
    long long ctas = (nseg + W * UNR - 1) / (W * UNR);          // one sweep iteration per warp when the graph is small
    if (ctas > gg::sm_count()) ctas = gg::sm_count();
    if (ctas < 1) ctas = 1;
    const long long seg_round = ctas * W * UNR;
    const long long iters = (nseg + seg_round - 1) / seg_round;
    const long long tab_n = iters * (W * UNR * rps / halves);
    const size_t smem = gg::pair_grad_smem_bytes(batch_size) + (size_t)tab_n * 4;
    GG_REQUIRE(smem <= 200 * 1024, "graph too large for the fused step loop (use gg_train_steps)");
    const void *kern = (const void *)gg::train_fused_kernel<NT, UNR>;
    if (smem > 48 * 1024) GG_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GG_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gg::train_fused_kernel<NT, UNR>, NT, smem));
    GG_REQUIRE(per_sm >= 1, "fused step loop kernel does not fit on an SM");
    gg::LoopArgs a;
    memset(&a, 0, sizeof(a));
    a.mode = mode; a.batch_size = batch_size; a.ld = ld; a.n_rows = n_rows; a.n_starts = n_starts; a.n_node = n_node;
    a.starts = (const long long *)start_list_dev; a.node_id = node_id; a.node_neighbor_id = node_neighbor_id; a.aux = aux;
    a.emb = emb; a.m_emb = m_emb; a.v_emb = v_emb; a.bias = bias; a.m_bias = m_bias; a.v_bias = v_bias;
    a.emb2 = emb2; a.bias2 = bias2; a.lambda = lambda;
    a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.beta1_power = *beta1_power; a.beta2_power = *beta2_power;
    a.sync_words = (unsigned long long *)sync_words;
    cudaStream_t st = (cudaStream_t)stream;
    GG_CHECK(cudaMemsetAsync(sync_words, 0, 8 * sizeof(uint64_t), st));
    void *args[] = {&a};
    GG_CHECK(cudaLaunchCooperativeKernel(kern, dim3((unsigned)ctas), dim3(NT), args, smem, st));
    if (n_starts & 1) {   // an odd number of steps leaves the parameters in the second buffers
        GG_CHECK(cudaMemcpyAsync(emb, emb2, sizeof(float) * (size_t)n_node * ld, cudaMemcpyDeviceToDevice, st));
        GG_CHECK(cudaMemcpyAsync(bias, bias2, sizeof(float) * (size_t)n_node, cudaMemcpyDeviceToDevice, st));
    }
    for (int64_t s = 0; s < n_starts; ++s) {   // the accumulators advance deterministically: replay them on the host
        volatile float p1 = *beta1_power * beta1, p2 = *beta2_power * beta2;
        *beta1_power = p1;
        *beta2_power = p2;
    }
    return 0;
}
