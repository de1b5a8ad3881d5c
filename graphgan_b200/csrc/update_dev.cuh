// update_dev.cuh -- device bodies of K2 (mini-batch gradient) and K3 (TF1.8 dense Adam sweep), shared by the
// stand-alone kernels (pairs.cu, adam.cu) and the persistent step loop (steps.cu).  See pairs.cu / adam.cu for
// the reference semantics each one restates.
#pragma once
#include "gg_common.cuh"

namespace gg {

// ---------------------------------------------------------------- mini-batch gradient (1 CTA)
constexpr int GRAD_THREADS = 512;     // 128 registers per thread: the fused bodies do not spill (they do at 1024 / 64)
constexpr int MERGE_THREADS = 1024;   // grad_merge_kernel (pairs.cu)

// COH = true: the parameters may have been written earlier in the SAME kernel by other SMs (persistent step
// loop): read them through L2 (ld.global.cg) instead of the non-coherent read-only path.
template <bool COH> __device__ __forceinline__ float4 row4(const float *p) {
    if constexpr (COH) return __ldcg(reinterpret_cast<const float4 *>(p));
    else return ldg4(p);
}
template <bool COH> __device__ __forceinline__ float ldf(const float *p) {
    if constexpr (COH) return __ldcg(p);
    else return __ldg(p);
}
template <bool COH>
__device__ __forceinline__ float group_dot_t(const float *a, const float *b, int ld, int g) {
    float s = 0.0f;
    for (int c = 4 * g; c < ld; c += 32) s = fma4(row4<COH>(a + c), row4<COH>(b + c), s);
    return group8_sum(s);
}

// dL/dscore of the pair (i, j) with label / reward a_k, computed by the 8-lane group that holds it (lane g of the
// group; every lane returns the same value): the canonical group dot, + bias[j], the sigmoid in fp64, the D or G
// formula.  The one-CTA gradient (pair_lists) and the multi-CTA gradient (grad_multi.cu) both call it.
template <bool COH>
__device__ __forceinline__ float pair_delta(int mode, int batch_total, int i, int j, float a_k, const float *emb,
                                            const float *bias, int ld, int g) {
    const float bj = ldf<COH>(bias + j);
    float s = group_dot_t<COH>(emb + (size_t)i * ld, emb + (size_t)j * ld, ld, g);
    s = __fadd_rn(s, bj);
    const float p = (float)(1.0 / (1.0 + exp(-(double)s)));   // sigmoid (B values: fp64 costs nothing)
    if (mode == 0) return p - a_k;                              // d/ds sigmoid_xent(label, s) = sigmoid(s) - label
    // d/ds [-(1/B) r log(clip(p,1e-5,1))] = -(r/B)(1-p) where the clip passes (p >= 1e-5)
    return (p >= 1e-5f) ? -(a_k / (float)batch_total) * (1.0f - p) : 0.0f;
}

// Shared memory of one mini-batch gradient: ids, slot, rank, list (2B ints each), offsets (2B + 2), delta (B).
__host__ __device__ inline size_t pair_grad_smem_bytes(int B) { return (size_t)(11 * B + 8) * 4; }

// The shared-memory arrays of one mini-batch (carved from pair_grad_smem_bytes(B) bytes).
struct PairSmem {
    int *ids;      // [E]  entry -> row id (i-side entries first, then j-side);  E = 2B
    int *slot;     // [E]  entry -> unique slot
    int *rnk;      // [E]  entry -> number of earlier entries with the same id
    int *lst;      // [E]  entries grouped by slot, entry order inside a slot
    int *off;      // [E + 2] slot -> start of its list
    float *delta;  // [B]  dL/dscore_k
};
__device__ __forceinline__ PairSmem pair_smem(int *smem, int B) {
    const int E = 2 * B;
    PairSmem p;
    p.ids = smem; p.slot = p.ids + E; p.rnk = p.slot + E; p.lst = p.rnk + E; p.off = p.lst + E;
    p.delta = reinterpret_cast<float *>(p.off + E + 2);
    return p;
}

// forward + unique + lists (see pair_grad_body).  Returns the number of unique rows U; uniq_ids / row_slot /
// n_unique (global) are written only when uniq_ids is not null.
template <bool COH, int NT>
__device__ __forceinline__ int pair_lists(int *smem, int mode, int B, int batch_total, const int *__restrict__ ni,
                                          const int *__restrict__ nj, const float *__restrict__ aux, const float *emb,
                                          const float *bias, int ld, int *n_unique, int *uniq_ids, int *row_slot) {
    const int E = 2 * B;
    const PairSmem ps = pair_smem(smem, B);
    int *ids = ps.ids, *slot = ps.slot, *rnk = ps.rnk, *lst = ps.lst, *off = ps.off;
    float *delta = ps.delta;
    __shared__ int s_warp[32];
    __shared__ int s_total;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, grp = lane >> 3, g = lane & 7;
    for (int t = tid; t < E; t += NT) { ids[t] = (t < B) ? ni[t] : nj[t - B]; off[t] = 0; }
    if (tid < 2) off[E + tid] = 0;
    // ---- forward: score and dL/dscore
    for (int k0 = wid * 4; k0 < B; k0 += (NT / 32) * 4) {
        const int k = k0 + grp;
        const bool valid = k < B;
        const int i = valid ? ni[k] : 0, j = valid ? nj[k] : 0;
        const float a_k = valid ? aux[k] : 0.0f;
        const float d = pair_delta<COH>(mode, batch_total, i, j, a_k, emb, bias, ld, g);
        if (valid && g == 0) delta[k] = d;
    }
    __syncthreads();
    // ---- unique, phase A: 8 lanes per entry scan the earlier entries (strided) for equal ids
    for (int t0 = 0; t0 < E; t0 += NT / 8) {
        const int t = t0 + (tid >> 3);
        int f = E, r = 0;
        if (t < E) {
            const int id = ids[t];
            for (int q = g; q < t; q += 8)
                if (ids[q] == id) { f = min(f, q); ++r; }
        }
#pragma unroll
        for (int o = 4; o >= 1; o >>= 1) {
            f = min(f, __shfl_xor_sync(FULL, f, o));
            r += __shfl_xor_sync(FULL, r, o);
        }
        if (t < E && g == 0) { slot[t] = min(f, t); rnk[t] = r; }
    }
    __syncthreads();
    // ---- phase B: exclusive scan of the first-occurrence flags (one entry per thread per round)
    int base_total = 0;
    for (int t0 = 0; t0 < E; t0 += NT) {
        const int t = t0 + tid;
        int is_first = 0, first_t = t;
        if (t < E) { first_t = slot[t]; is_first = (first_t == t); }   // (each thread rewrites only its own slot[t])
        int x = is_first;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(FULL, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            int v = lane < NT / 32 ? s_warp[lane] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(FULL, v, o);
                if (lane >= o) v += y;
            }
            s_warp[lane] = v;
        }
        __syncthreads();
        const int excl = base_total + (wid ? s_warp[wid - 1] : 0) + x - is_first;
        if (t < E) slot[t] = is_first ? excl : -1 - first_t;  // non-first: remember where the first is
        if (t < E && is_first && uniq_ids) { uniq_ids[excl] = ids[t]; row_slot[ids[t]] = excl; }
        base_total += s_warp[31];
        __syncthreads();
    }
    if (tid == 0) { s_total = base_total; if (uniq_ids) *n_unique = base_total; }
    // non-first entries take the slot of their first occurrence (which is >= 0 and final); count the list lengths
    for (int t = tid; t < E; t += NT) {
        int sl = slot[t];
        if (sl < 0) { sl = slot[-1 - sl]; slot[t] = sl; }
        atomicAdd(&off[sl + 1], 1);
    }
    __syncthreads();
    const int U = s_total;
    // ---- offsets: inclusive scan of the counts in off[1 .. U] (two per thread per round)
    int run = 0;
    for (int u0 = 0; u0 < U; u0 += 2 * NT) {
        const int ia = u0 + 2 * tid, ib = ia + 1;
        const int ca = (ia < U) ? off[ia + 1] : 0, cb = (ib < U) ? off[ib + 1] : 0;
        int x = ca + cb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(FULL, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            int v = lane < NT / 32 ? s_warp[lane] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(FULL, v, o);
                if (lane >= o) v += y;
            }
            s_warp[lane] = v;
        }
        __syncthreads();
        const int incl = run + (wid ? s_warp[wid - 1] : 0) + x;     // through ib
        if (ia < U) off[ia + 1] = incl - cb;
        if (ib < U) off[ib + 1] = incl;
        run += s_warp[31];
        __syncthreads();
    }
    for (int t = tid; t < E; t += NT) lst[off[slot[t]] + rnk[t]] = t;
    __syncthreads();
    return U;
}

// segment sums of the lists built by pair_lists -> grad_rows [U, ld], grad_bias [U]
template <bool COH, int NT>
__device__ __forceinline__ void pair_sums(int *smem, int mode, int B, int U, const float *emb, const float *bias, int ld,
                                          float lambda, float *grad_rows, float *grad_bias) {
    const PairSmem ps = pair_smem(smem, B);
    const int *ids = ps.ids, *lst = ps.lst, *off = ps.off;
    const float *delta = ps.delta;
    const int tid = threadIdx.x, g = tid & 7;
    // ---- segment sums: 8 lanes per slot, columns in passes of 64 (one float4 at c and one at c + 32 per lane)
    for (int u0 = 0; u0 < U; u0 += NT / 8) {
        const int u = u0 + (tid >> 3);
        if (u >= U) continue;           // whole 8-lane groups drop out together; only group shuffles are not used below
        const int lo = off[u], n = off[u + 1] - lo;
        const int row = ids[lst[lo]];
        const float *erow = emb + (size_t)row * ld;
        for (int c0 = 0; c0 < ld; c0 += 64) {
            const int c = c0 + 4 * g;
            const bool two = c + 32 < ld;
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            float4 acc0 = z, acc1 = z;
            const float4 self0 = row4<COH>(erow + c), self1 = two ? row4<COH>(erow + c + 32) : z;
            // d(score)/d(this row) = other row;  l2 term: lambda * this row, once per occurrence.
            // Explicit mul/mul/add/add (no fma contraction): the same op sequence as the IndexedSlices
            // sum of the numpy oracle, so cancellation noise in near-zero coordinates stays comparable.
#define GG_ACC(acc, o, self, f) acc.f = __fadd_rn(acc.f, __fadd_rn(__fmul_rn(d, o.f), __fmul_rn(lambda, self.f)))
#define GG_ACC4(acc, o, self) GG_ACC(acc, o, self, x); GG_ACC(acc, o, self, y); GG_ACC(acc, o, self, z); GG_ACC(acc, o, self, w)
            // four entries' rows in flight, added in entry order (a centre node repeated through a whole batch gives
            // one slot a list of ~B entries: the loads must not be serialised behind the adds)
            for (int r = 0; r < n; r += 4) {
                float4 o0[4], o1[4];
                float dd[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const bool in = r + e < n;
                    const int t = in ? lst[lo + r + e] : 0;
                    const float *op = emb + (size_t)ids[t < B ? t + B : t - B] * ld + c;
                    o0[e] = in ? row4<COH>(op) : z;
                    o1[e] = (in && two) ? row4<COH>(op + 32) : z;
                    dd[e] = delta[t < B ? t : t - B];
                }
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (r + e >= n) break;
                    const float d = dd[e];
                    GG_ACC4(acc0, o0[e], self0); GG_ACC4(acc1, o1[e], self1);
                }
            }
#undef GG_ACC4
#undef GG_ACC
            *reinterpret_cast<float4 *>(grad_rows + (size_t)u * ld + c) = acc0;
            if (two) *reinterpret_cast<float4 *>(grad_rows + (size_t)u * ld + c + 32) = acc1;
        }
        if (g == 0) {   // bias gradient: j-side entries only; generator.py:28-29 has no bias l2
            const float bself = ldf<COH>(bias + row);
            float gb = 0.0f;
            for (int r = 0; r < n; ++r) {
                const int t = lst[lo + r];
                if (t < B) continue;
                const float d = delta[t - B];
                gb = __fadd_rn(gb, mode == 0 ? __fadd_rn(d, __fmul_rn(lambda, bself)) : d);
            }
            grad_bias[u] = gb;
        }
    }
}


// One mini-batch gradient, executed by one CTA of NT threads (a multiple of 32, at most 1024); smem: pair_grad_smem_bytes(B).
//   forward     4 pairs per warp (8 lanes per dot, the canonical group dot), sigmoid in fp64
//   unique      8 lanes per entry count the earlier equal ids (-> first occurrence and rank within the row's
//               entries); a block scan numbers the first occurrences in entry order (TF's unique() order)
//   lists       per-slot entry lists in entry order (CSR in shared memory: offsets by a second block scan)
//   sums        8 lanes per slot walk the slot's list; two entries' rows are in flight per iteration and are
//               added in entry order, so the sum is the same op sequence as a sequential IndexedSlices sum
template <bool COH, int NT = GRAD_THREADS>
__device__ __forceinline__ void pair_grad_body(int *smem, int mode, int B, int batch_total, const int *__restrict__ ni,
                                               const int *__restrict__ nj, const float *__restrict__ aux,
                                               const float *emb, const float *bias, int ld, float lambda, int *n_unique,
                                               int *uniq_ids, float *grad_rows, float *grad_bias, int *row_slot) {
    const int U = pair_lists<COH, NT>(smem, mode, B, batch_total, ni, nj, aux, emb, bias, ld, n_unique, uniq_ids, row_slot);
    pair_sums<COH, NT>(smem, mode, B, U, emb, bias, ld, lambda, grad_rows, grad_bias);
}


// The dense Adam sweep over all rows, executed by the whole grid.  A warp owns segments of 32 float4 (= 128/ld
// rows, or half a row at ld = 256) and keeps UNR segments in flight: the row -> slot probes and the m / v / var
// loads of all of them are issued before the first use; only the rare rows with a gradient add a dependent load.
// The lane owning a row's first columns also updates the row's bias and clears its slot (after the warp has read
// it; PRE = its bias loads are issued with the others, which costs registers).  COH: the gradient slots were written earlier in the same kernel by another SM -> read them through L2.
// At ld = 512 (four segments per row) UNR must be a multiple of 4 (ADAM_WIDE_UNR): the whole row in one warp.
constexpr int ADAM_WIDE_UNR = 4;
template <bool COH, int UNR, bool PRE = true>
__device__ __forceinline__ void adam_rows(long long n_node, int ld, float *emb, float *m_emb, float *v_emb, float *bias,
                                          float *m_bias, float *v_bias, const float *grad_rows, const float *grad_bias,
                                          int *row_slot, float lr_t, float b1, float b2, float eps) {
    static_assert(UNR % 2 == 0, "both halves of a 256-wide row must be in flight in the same warp");
    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const float omb1 = 1.0f - b1, omb2 = 1.0f - b2;
    const int q = ld >> 2;                        // float4 per row: 8, 16, 32 or 64
    const int rows_per_seg = q >= 32 ? 1 : 32 / q;
    const int halves = q > 32 ? q / 32 : 1;       // segments per row (2 at ld = 256)
    const long long nseg = ((n_node + rows_per_seg - 1) / rows_per_seg) * halves;
    const int sub = q >= 32 ? 0 : lane / q;       // which of the segment's rows this lane is in
    const int col = q >= 32 ? 4 * lane : 4 * (lane % q);
// TF1.8 op order (assign m*b1; scatter_add (1-b1)*g; ... var -= lr*m/(sqrt(v)+eps)), no contraction
#define GG_ADAM1(f)                                                                                   \
    m[k].f = __fadd_rn(__fmul_rn(m[k].f, b1), __fmul_rn(omb1, g.f));                                  \
    v[k].f = __fadd_rn(__fmul_rn(v[k].f, b2), __fmul_rn(__fmul_rn(g.f, g.f), omb2));                  \
    x[k].f = __fsub_rn(x[k].f, __fdiv_rn(__fmul_rn(lr_t, m[k].f), __fadd_rn(__fsqrt_rn(v[k].f), eps)));
    for (long long s0 = warp * UNR; s0 < nseg; s0 += nwarps * UNR) {
        int row[UNR], cc[UNR], slot[UNR];      // row < 0: nothing to do for this lane
        float4 m[UNR], v[UNR], x[UNR];
        float mb[UNR], vb[UNR], xb[UNR];
#pragma unroll
        for (int k = 0; k < UNR; ++k) {
            const long long seg = s0 + k;
            const long long r = (seg / halves) * rows_per_seg + sub;
            cc[k] = col + 128 * (int)(seg % halves);
            row[k] = (seg < nseg && r < n_node) ? (int)r : -1;
            slot[k] = -1;
            if (row[k] >= 0) {
                const size_t at = (size_t)r * ld + cc[k];
                slot[k] = COH ? __ldcg(row_slot + r) : row_slot[r];
                m[k] = *reinterpret_cast<const float4 *>(m_emb + at);
                v[k] = *reinterpret_cast<const float4 *>(v_emb + at);
                x[k] = *reinterpret_cast<const float4 *>(emb + at);
                if (PRE && cc[k] == 0) { mb[k] = m_bias[r]; vb[k] = v_bias[r]; xb[k] = bias[r]; }
            }
        }
        __syncwarp();      // every lane has read its rows' slots before a leader clears them
#pragma unroll
        for (int k = 0; k < UNR; ++k) {
            if (row[k] < 0) continue;
            const size_t at = (size_t)row[k] * ld + cc[k];
            float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
            if (slot[k] >= 0) {
                const float *gp = grad_rows + (size_t)slot[k] * ld + cc[k];
                g = COH ? __ldcg(reinterpret_cast<const float4 *>(gp)) : *reinterpret_cast<const float4 *>(gp);
            }
            GG_ADAM1(x) GG_ADAM1(y) GG_ADAM1(z) GG_ADAM1(w)
            *reinterpret_cast<float4 *>(m_emb + at) = m[k];
            *reinterpret_cast<float4 *>(v_emb + at) = v[k];
            *reinterpret_cast<float4 *>(emb + at) = x[k];
            if (cc[k] == 0) {
                if (!PRE) { mb[k] = m_bias[row[k]]; vb[k] = v_bias[row[k]]; xb[k] = bias[row[k]]; }
                const float gb = slot[k] >= 0 ? (COH ? __ldcg(grad_bias + slot[k]) : grad_bias[slot[k]]) : 0.0f;
                const float mm = __fadd_rn(__fmul_rn(mb[k], b1), __fmul_rn(omb1, gb));
                const float vv = __fadd_rn(__fmul_rn(vb[k], b2), __fmul_rn(__fmul_rn(gb, gb), omb2));
                m_bias[row[k]] = mm; v_bias[row[k]] = vv;
                bias[row[k]] = __fsub_rn(xb[k], __fdiv_rn(__fmul_rn(lr_t, mm), __fadd_rn(__fsqrt_rn(vv), eps)));
                if (slot[k] >= 0) row_slot[row[k]] = -1;
            }
        }
    }
#undef GG_ADAM1
}


// ---------------------------------------------------------------- data-parallel merge (1 CTA of MERGE_THREADS)
// Entry (r, s) = slot s of rank r's compact gradient.  Same unique + ordered segment-sum as the mini-batch gradient, on
// ready-made row vectors; entry order is rank-major, so all ranks reduce in the same order.  smem: 2 * world * cap ints.
__device__ __forceinline__ void grad_merge_body(int *smem, int world, int cap, int ld, const float *gathered,
                                                int *__restrict__ n_unique, int *__restrict__ uniq_ids,
                                                float *__restrict__ grad_rows, float *__restrict__ grad_bias,
                                                int *__restrict__ row_slot) {
    const int E = world * cap;
    int *ids = smem;          // [E] row id or -1
    int *slot = ids + E;      // [E]
    __shared__ int s_warp[32];
    __shared__ int s_total;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const size_t stride = (size_t)cap * ld + 2 * (size_t)cap + 4;   // == gg_grad_buf_floats
    for (int t = tid; t < E; t += MERGE_THREADS) {
        const int r = t / cap, sidx = t % cap;
        const float *buf = gathered + (size_t)r * stride;
        const int nu = __float_as_int(buf[(size_t)cap * ld + 2 * (size_t)cap]);
        const int id = (sidx < nu) ? __float_as_int(buf[(size_t)cap * ld + cap + sidx]) : -1;
        ids[t] = id;
        if (id >= 0) row_slot[id] = -1;   // forget the slots of the local (pre-merge) gradient
    }
    __syncthreads();
    int base_total = 0;
    for (int t0 = 0; t0 < E; t0 += MERGE_THREADS) {
        const int t = t0 + tid;
        int is_first = 0, first_t = t;
        if (t < E && ids[t] >= 0) {
            const int id = ids[t];
            int f = t;
            for (int q = 0; q < t; ++q) if (ids[q] == id) { f = q; break; }
            first_t = f; is_first = (f == t);
        }
        int x = is_first;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int y = __shfl_up_sync(FULL, x, off);
            if (lane >= off) x += y;
        }
        if (lane == 31) s_warp[wid] = x;
        __syncthreads();
        if (wid == 0) {
            int v = s_warp[lane];
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const int y = __shfl_up_sync(FULL, v, off);
                if (lane >= off) v += y;
            }
            s_warp[lane] = v;
        }
        __syncthreads();
        const int excl = base_total + (wid ? s_warp[wid - 1] : 0) + x - is_first;
        if (t < E) slot[t] = (ids[t] < 0) ? -(E + 1) : (is_first ? excl : -1 - first_t);
        if (t < E && is_first) { uniq_ids[excl] = ids[t]; row_slot[ids[t]] = excl; }
        base_total += s_warp[31];
        __syncthreads();
    }
    if (tid == 0) { s_total = base_total; *n_unique = base_total; }
    __syncthreads();
    for (int t = tid; t < E; t += MERGE_THREADS)
        if (slot[t] < 0 && slot[t] != -(E + 1)) slot[t] = slot[-1 - slot[t]];
    __syncthreads();
    const int U = s_total;
    for (int u = wid; u < U; u += MERGE_THREADS / 32) {
        for (int c = 4 * lane; c < ld; c += 128) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int t = 0; t < E; ++t) {
                if (slot[t] != u) continue;
                const float4 o = *reinterpret_cast<const float4 *>(gathered + (size_t)(t / cap) * stride + (size_t)(t % cap) * ld + c);
                acc.x = __fadd_rn(acc.x, o.x); acc.y = __fadd_rn(acc.y, o.y);
                acc.z = __fadd_rn(acc.z, o.z); acc.w = __fadd_rn(acc.w, o.w);
            }
            *reinterpret_cast<float4 *>(grad_rows + (size_t)u * ld + c) = acc;
        }
        if (lane == 0) {
            float gb = 0.0f;
            for (int t = 0; t < E; ++t)
                if (slot[t] == u) gb = __fadd_rn(gb, gathered[(size_t)(t / cap) * stride + (size_t)cap * ld + (t % cap)]);
            grad_bias[u] = gb;
        }
    }
}

}  // namespace gg
