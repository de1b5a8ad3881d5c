// pairs.cu -- K2: pairwise scoring, reward, sparse gradients; window-pair expansion (sm_90a).
//
//   score_k = e[i_k] . e[j_k] + b[j_k]      discriminator.py:21-24 / generator.py:22-25
//   reward  = log(1 + exp(clip(score,-10,10)))  discriminator.py:33-34 (fetched at graph_gan.py:220-222)
//   D loss  = sum_k sigmoid_xent(label_k, score_k) + lambda (l2(e_j) + l2(e_i) + l2(b_j))   discriminator.py:26-30
//   G loss  = -mean_k(log(clip(sigmoid(score_k),1e-5,1)) * reward_k) + lambda (l2(e_j) + l2(e_i))  generator.py:26-29
//
// Gradients are produced in TF1.8's IndexedSlices form after _apply_sparse_duplicate_indices:
// unique row ids + per-row sums (entries accumulated in (i-side 0..B-1, j-side 0..B-1) order,
// deterministic).  The reference's mini-batch is small (config.batch_size_* = 64), so one CTA does
// up to GG_MAX_BATCH = 1024 pairs here; the expensive part of such a step is K3's dense sweep
// (adam.cu).  Larger batches go to the multi-CTA gradient of grad_multi.cu (gg_pair_grad_ex), which
// computes the same bits: slots in first-occurrence order, and per slot one +0-started __fadd_rn
// chain per coordinate over the slot's entries in entry order (bias: j-side entries only).  Such a
// chain is serial, so the batch's longest slot is the floor of that path.  Gather-bound, fp32, no
// tensor cores.
#include "update_dev.cuh"

namespace gg {
namespace {

// 8-lane group dot over a padded row pair; all 8 lanes return the sum.
__device__ __forceinline__ float group_dot(const float *a, const float *b, int ld, int g) {
    float s = 0.0f;
    for (int c = 4 * g; c < ld; c += 32) s = fma4(ldg4(a + c), ldg4(b + c), s);
    return group8_sum(s);
}

__global__ void __launch_bounds__(256) reward_kernel(long long n_pairs, const int *__restrict__ ni,
                                                     const int *__restrict__ nj, const float *__restrict__ emb,
                                                     const float *__restrict__ bias, int ld, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, grp = lane >> 3, g = lane & 7;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long p0 = warp * 4; p0 < n_pairs; p0 += nwarps * 4) {
        const long long p = p0 + grp;
        const bool valid = p < n_pairs;
        const int i = valid ? ni[p] : 0, j = valid ? nj[p] : 0;
        float s = group_dot(emb + (size_t)i * ld, emb + (size_t)j * ld, ld, g);
        if (valid && g == 0) {
            s = __fadd_rn(s, bias[j]);
            s = fminf(fmaxf(s, -10.0f), 10.0f);        // tf.clip_by_value (discriminator.py:33)
            out[p] = logf(1.0f + expf(s));             // tf.log(1 + tf.exp(score)) (discriminator.py:34)
        }
    }
}

__global__ void __launch_bounds__(256) all_score_kernel(long long n, const float *__restrict__ emb,
                                                        const float *__restrict__ bias, int ld, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, grp = lane >> 3, g = lane & 7;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    const long long total = n * n;
    for (long long p0 = warp * 4; p0 < total; p0 += nwarps * 4) {
        const long long p = p0 + grp;
        const bool valid = p < total;
        const long long i = valid ? p / n : 0, j = valid ? p % n : 0;
        const float s = group_dot(emb + (size_t)i * ld, emb + (size_t)j * ld, ld, g);
        if (valid && g == 0) out[p] = __fadd_rn(s, bias[j]);  // generator.py:21: E.E^T + b (b broadcast over columns)
    }
}

// ---------------------------------------------------------------- mini-batch gradient (1 CTA)
__global__ void __launch_bounds__(GRAD_THREADS, 1)
pair_grad_kernel(int mode, int B, int batch_total, const int *__restrict__ ni, const int *__restrict__ nj, const float *__restrict__ aux,
                 const float *__restrict__ emb, const float *__restrict__ bias, int ld, float lambda,
                 int *__restrict__ n_unique, int *__restrict__ uniq_ids, float *__restrict__ grad_rows,
                 float *__restrict__ grad_bias, int *__restrict__ row_slot) {
    extern __shared__ int smem[];
    pair_grad_body<false>(smem, mode, B, batch_total, ni, nj, aux, emb, bias, ld, lambda, n_unique, uniq_ids, grad_rows, grad_bias,
                          row_slot);
}

// ---------------------------------------------------------------- data-parallel merge (1 CTA)
// Entry (r, s) = slot s of rank r's compact gradient.  Same unique + ordered segment-sum as above, on
// ready-made row vectors; entry order is rank-major, so all ranks reduce in the same order.
__global__ void __launch_bounds__(MERGE_THREADS, 1)
grad_merge_kernel(int world, int cap, int ld, const float *__restrict__ gathered, int *__restrict__ n_unique,
                  int *__restrict__ uniq_ids, float *__restrict__ grad_rows, float *__restrict__ grad_bias,
                  int *__restrict__ row_slot) {
    extern __shared__ int smem[];
    grad_merge_body(smem, world, cap, ld, gathered, n_unique, uniq_ids, grad_rows, grad_bias, row_slot);
}

// ---------------------------------------------------------------- window pairs (graph_gan.py:272-291)
__device__ __forceinline__ int pairs_of(int body, int w) {
    int c = 0;
    for (int i = 0; i < body; ++i) {
        const int lo = i - w < 0 ? 0 : i - w, hi = i + w + 1 > body ? body : i + w + 1;
        c += hi - lo - 1;
    }
    return c;
}

__global__ void window_count_kernel(long long n_walks, const int *__restrict__ path_len, int max_path, int window,
                                    long long *__restrict__ pair_ptr) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_walks) return;
    int L = path_len[w];
    if (L > max_path) L = max_path;
    const int body = L - 1;  // path[:-1]
    pair_ptr[w] = body > 0 ? pairs_of(body, window) : 0;
}

__global__ void window_emit_kernel(long long n_walks, const int *__restrict__ paths, const int *__restrict__ path_len,
                                   int max_path, int window, const long long *__restrict__ pair_ptr,
                                   int *__restrict__ n1, int *__restrict__ n2, long long capacity) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_walks) return;
    int L = path_len[w];
    if (L > max_path) L = max_path;
    const int body = L - 1;
    long long o = pair_ptr[w];
    const int *p = paths + (size_t)w * max_path;
    for (int i = 0; i < body; ++i) {
        const int lo = i - window < 0 ? 0 : i - window, hi = i + window + 1 > body ? body : i + window + 1;
        const int c = p[i];
        for (int j = lo; j < hi; ++j) {
            if (j == i) continue;
            if (o < capacity) { n1[o] = c; n2[o] = p[j]; }
            ++o;
        }
    }
}

}  // namespace
}  // namespace gg

extern "C" int gg_pair_reward(int64_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id, const float *emb,
                              const float *bias, int32_t ld, float *reward, void *stream) {
    if (n_pairs == 0) return 0;
    GG_REQUIRE(node_id && node_neighbor_id && emb && bias && reward, "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    long long blocks = (n_pairs + 31) / 32;  // 8 warps x 4 pairs per pass
    const long long cap = (long long)gg::sm_count() * 8;
    if (blocks > cap) blocks = cap;
    gg::reward_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n_pairs, node_id, node_neighbor_id, emb, bias,
                                                                          ld, reward);
    return gg::check_cuda(cudaGetLastError(), "reward kernel launch");
}

extern "C" int gg_all_score(int64_t n_node, const float *emb, const float *bias, int32_t ld, float *out, void *stream) {
    if (n_node == 0) return 0;
    GG_REQUIRE(emb && bias && out, "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    GG_REQUIRE(n_node <= 46340, "all_score is only materialised for small graphs (N*N must fit int32 range of tests)");
    gg::all_score_kernel<<<gg::sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(n_node, emb, bias, ld, out);
    return gg::check_cuda(cudaGetLastError(), "all_score kernel launch");
}

extern "C" int gg_pair_grad(int32_t mode, int32_t n_pairs, int32_t batch_total, const int32_t *node_id, const int32_t *node_neighbor_id,
                            const float *aux, const float *emb, const float *bias, int32_t ld, float lambda,
                            int32_t *n_unique, int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot,
                            void *stream) {
    GG_REQUIRE(mode == 0 || mode == 1, "mode must be 0 (discriminator) or 1 (generator)");
    GG_REQUIRE(n_pairs > 0 && n_pairs <= GG_MAX_BATCH, "batch size out of range");
    GG_REQUIRE(node_id && node_neighbor_id && aux && emb && bias && n_unique && uniq_ids && grad_rows && grad_bias && row_slot,
               "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    const size_t smem = gg::pair_grad_smem_bytes(n_pairs);
    gg::pair_grad_kernel<<<1, gg::GRAD_THREADS, smem, (cudaStream_t)stream>>>(
        mode, n_pairs, batch_total > 0 ? batch_total : n_pairs, node_id, node_neighbor_id, aux, emb, bias, ld, lambda,
        n_unique, uniq_ids, grad_rows, grad_bias, row_slot);
    return gg::check_cuda(cudaGetLastError(), "pair_grad kernel launch");
}

extern "C" int64_t gg_grad_buf_floats(int32_t cap, int32_t ld) { return (int64_t)cap * ld + 2 * (int64_t)cap + 4; }

extern "C" int gg_grad_merge(int32_t world, int32_t cap, int32_t ld, const float *gathered, int32_t *n_unique,
                             int32_t *uniq_ids, float *grad_rows, float *grad_bias, int32_t *row_slot, void *stream) {
    GG_REQUIRE(world > 0 && cap > 0 && (int64_t)world * cap <= 2 * GG_MAX_BATCH * 8, "too many entries to merge");
    GG_REQUIRE(gathered && n_unique && uniq_ids && grad_rows && grad_bias && row_slot, "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    const size_t smem = (size_t)world * cap * 2 * 4;
    GG_REQUIRE(smem <= 200 * 1024, "merge exceeds shared memory");
    if (smem > 48 * 1024)
        GG_CHECK(cudaFuncSetAttribute(gg::grad_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gg::grad_merge_kernel<<<1, gg::MERGE_THREADS, smem, (cudaStream_t)stream>>>(world, cap, ld, gathered, n_unique, uniq_ids,
                                                                             grad_rows, grad_bias, row_slot);
    return gg::check_cuda(cudaGetLastError(), "grad merge launch");
}

extern "C" int gg_window_pairs(int64_t n_walks, const int32_t *paths, const int32_t *path_len, int32_t max_path,
                               int32_t window, int64_t *pair_ptr, int32_t *node_1, int32_t *node_2, int64_t *n_pairs_out,
                               int64_t capacity, void *stream) {
    GG_REQUIRE(pair_ptr && n_pairs_out, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int threads = 256;
    const unsigned blocks = (unsigned)((n_walks + threads - 1) / threads);
    if (n_walks > 0) {
        GG_REQUIRE(paths && path_len && max_path > 0 && window >= 0, "bad path arguments");
        gg::window_count_kernel<<<blocks, threads, 0, st>>>(n_walks, path_len, max_path, window, (long long *)pair_ptr);
        GG_CHECK(cudaGetLastError());
    }
    int rc = gg::launch_exclusive_scan_i64((long long *)pair_ptr, n_walks, (long long *)n_pairs_out, st);
    if (rc) return rc;
    if (n_walks == 0 || capacity == 0) return 0;
    GG_REQUIRE(node_1 && node_2, "null output pointer");
    gg::window_emit_kernel<<<blocks, threads, 0, st>>>(n_walks, paths, path_len, max_path, window,
                                                       (const long long *)pair_ptr, node_1, node_2, capacity);
    return gg::check_cuda(cudaGetLastError(), "window emit launch");
}
