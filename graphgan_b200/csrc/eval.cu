// eval.cu -- the end-of-epoch quality line and embedding dump on the device (sm_90a; SURVEY.md section 8 row f4).
//
// Reference: GraphGAN.write_embeddings_to_file (graph_gan.py:293-306) writes both embedding matrices as text and
// GraphGAN.evaluation (:308-319) -> LinkPredictEval.eval_link_prediction (src/evaluation/link_prediction.py:19-38)
// reads the text back (utils.py:57-67), scores the test positives then negatives by np.dot (float64), thresholds at
// np.median and reports sklearn accuracy against [1]*half + [0]*half.  At N = 1M the text round trip is minutes per
// epoch.  Here:
//   gg_pair_dot_f64  : float64 dot of two embedding rows per test edge (the text round trip of an fp32 value is exact,
//                      so these are the reference's operands; products of fp32 values are exact in fp64)
//   gg_link_pred_acc : np.median (mean of the two middle order statistics for even counts) by an MSB-first radix
//                      select over order-preserving 64-bit keys, then the accuracy count -- one CTA, no sort; a NaN
//                      score gives np.median's NaN (and so no positive prediction), as the reference reports it
//   gg_unpad_rows    : [N, ld] padded rows -> dense [N, n_emb] fp32, the binary dump's payload
// Gather-bound / tiny; no tensor cores.
#include "gg_common.cuh"

namespace gg {
namespace {

__global__ void __launch_bounds__(256) pair_dot_f64_kernel(long long n_pairs, const int *__restrict__ ni,
                                                           const int *__restrict__ nj, const float *__restrict__ emb,
                                                           int ld, double *__restrict__ out) {
    const int lane = threadIdx.x & 31, grp = lane >> 3, g = lane & 7;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long p0 = warp * 4; p0 < n_pairs; p0 += nwarps * 4) {
        const long long p = p0 + grp;
        const bool valid = p < n_pairs;
        const float *a = emb + (size_t)(valid ? ni[p] : 0) * ld, *b = emb + (size_t)(valid ? nj[p] : 0) * ld;
        double s = 0.0;
        for (int c = 4 * g; c < ld; c += 32) {
            const float4 x = ldg4(a + c), y = ldg4(b + c);
            s += (double)x.x * (double)y.x;
            s += (double)x.y * (double)y.y;
            s += (double)x.z * (double)y.z;
            s += (double)x.w * (double)y.w;
        }
        s += __shfl_xor_sync(FULL, s, 4);
        s += __shfl_xor_sync(FULL, s, 2);
        s += __shfl_xor_sync(FULL, s, 1);
        if (valid && g == 0) out[p] = s;
    }
}

__device__ __forceinline__ unsigned long long order_key(double x) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);      // unsigned order == numeric order
}
__device__ __forceinline__ double key_value(unsigned long long k) {
    const unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)u);
}

// k-th smallest (0-based) key of score[0..n): 8 passes of an 8-bit histogram over the keys that match the prefix
__device__ unsigned long long radix_select(const double *score, long long n, long long k, unsigned *hist,
                                           unsigned long long *s_prefix, long long *s_k) {
    unsigned long long prefix = 0, mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
        __syncthreads();
        for (long long i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long key = order_key(score[i]);
            if ((key & mask) == prefix) atomicAdd(hist + (unsigned)((key >> shift) & 0xff), 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long kk = k;
            int b = 0;
            for (; b < 255; ++b) {
                if (kk < (long long)hist[b]) break;
                kk -= hist[b];
            }
            *s_prefix = prefix | ((unsigned long long)b << shift);
            *s_k = kk;
        }
        __syncthreads();
        prefix = *s_prefix; k = *s_k;
        mask |= 0xffull << shift;
        __syncthreads();
    }
    return prefix;
}

__global__ void __launch_bounds__(1024, 1) link_pred_kernel(long long n, const double *__restrict__ score, double *out) {
    __shared__ unsigned hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ long long s_k;
    __shared__ unsigned long long s_hits, s_nans;
    // np.median: middle element (odd n) or the mean of the two middle elements (even n)
    const double hi = key_value(radix_select(score, n, n / 2, hist, &s_prefix, &s_k));
    const double lo = (n % 2) ? hi : key_value(radix_select(score, n, n / 2 - 1, hist, &s_prefix, &s_k));
    const double med = (n % 2) ? hi : (lo + hi) / 2.0;
    if (threadIdx.x == 0) { s_hits = 0ull; s_nans = 0ull; }
    __syncthreads();
    const long long half = n / 2;                 // true_label[0 : len // 2] = 1 (link_prediction.py:34-35)
    unsigned long long hits = 0, nans = 0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const double x = score[i];
        const bool pred = x >= med;               // index_pos = test_label >= median (:30)
        hits += (pred == (i < half)) ? 1ull : 0ull;
        nans += isnan(x) ? 1ull : 0ull;
    }
    atomicAdd(&s_hits, hits);
    atomicAdd(&s_nans, nans);
    __syncthreads();
    // any NaN makes np.median NaN (order_key sorts NaN to an end instead), so no score is >= it: every prediction is 0
    if (threadIdx.x == 0) {
        out[0] = s_nans ? (double)(n - half) / (double)n : (double)s_hits / (double)n;
        out[1] = s_nans ? __longlong_as_double(0x7ff8000000000000ll) : med;
    }
}

__global__ void unpad_rows_kernel(long long n_node, int ld, int d, const float *__restrict__ emb, float *__restrict__ out) {
    const long long total = n_node * (long long)d;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long r = t / d;
        out[t] = emb[(size_t)r * ld + (t - r * d)];
    }
}

}  // namespace
}  // namespace gg

extern "C" int gg_pair_dot_f64(int64_t n_pairs, const int32_t *node_id, const int32_t *node_neighbor_id, const float *emb,
                               int32_t ld, double *out, void *stream) {
    if (n_pairs == 0) return 0;
    GG_REQUIRE(node_id && node_neighbor_id && emb && out, "null pointer");
    GG_REQUIRE(gg::ld_supported(ld), GG_LD_MESSAGE);
    long long blocks = (n_pairs + 31) / 32;
    const long long cap = (long long)gg::sm_count() * 16;
    if (blocks > cap) blocks = cap;
    gg::pair_dot_f64_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n_pairs, node_id, node_neighbor_id, emb, ld, out);
    return gg::check_cuda(cudaGetLastError(), "pair dot kernel launch");
}

extern "C" int gg_link_pred_acc(int64_t n, const double *score, double *out2, void *stream) {
    GG_REQUIRE(score && out2 && n > 0, "bad arguments");
    gg::link_pred_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(n, score, out2);
    return gg::check_cuda(cudaGetLastError(), "link prediction kernel launch");
}

extern "C" int gg_unpad_rows(int64_t n_node, int32_t ld, int32_t n_emb, const float *emb, float *out, void *stream) {
    if (n_node == 0) return 0;
    GG_REQUIRE(emb && out && n_emb > 0 && n_emb <= ld, "bad arguments");
    long long blocks = (n_node * n_emb + 255) / 256;
    const long long cap = (long long)gg::sm_count() * 32;
    if (blocks > cap) blocks = cap;
    gg::unpad_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n_node, ld, n_emb, emb, out);
    return gg::check_cuda(cudaGetLastError(), "unpad kernel launch");
}
