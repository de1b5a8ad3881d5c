// value_grad.cuh -- what the exact gradients of the game value (value_grad.cu and value_dgrad.cu, DESIGN.md sections 5.3
// and 5.4) take from the generator distribution (gdist.cu) and the game value (value.cu).
#pragma once
#include "gg_common.cuh"

namespace gg {

// Per (root slot, node), [n_roots, n_node] row-major, written by the recording variant of the section 5.1 kernel for the
// nodes it reaches: pi_in (the node's probability in its father's list), pi_stop (its father's probability in its own
// list; the caller clears it to 0), father (the caller clears it to -1).  items / lev_off / n_lev live in the scratch
// (gdist_rec_layout): every level's items, level L at [lev_off[L], lev_off[L + 1]), n_lev levels.
struct GdRec {
    double *pi_in = nullptr, *pi_stop = nullptr;
    int *father = nullptr;
    int4 *items = nullptr;
    unsigned *lev_off = nullptr, *n_lev = nullptr;
};

// bytes of the recording kernel's scratch; fills rec->{items, lev_off, n_lev} when `buf` is given
size_t gdist_rec_layout(void *buf, long long n_node, long long nnz_words, long long n_roots, GdRec *rec);
// dist / root_ok with the bits of gg_generator_dist, plus the records (dist and root_ok cleared by the caller)
int gdist_rec_launch(const gg_walk_desc &d, double *dist, int *root_ok, GdRec rec, void *scratch, cudaStream_t st);
// h[k, v] = dist[k, v] * bce(s(roots[k], v), 0) (0 where dist is 0): the products the value kernel adds into neg
int value_h_launch(long long n_node, int ld, const float *emb, const float *bias, long long n_roots, const int *roots,
                   const double *dist, double *h, cudaStream_t st);
// W[k, v] = dV_{c_k} / ds(c_k, v) = mult[k, v] sigma(-s) / |graph[c_k]| - dist[k, v] sigma(s), 0 for roots with ok_k = 0
// (the discriminator gradient, value_dgrad.cu, DESIGN.md section 5.4); mult: v's count in graph[c_k]
int value_w_launch(long long n_node, int ld, const float *emb, const float *bias, const long long *raw_indptr,
                   long long n_roots, const int *roots, const double *dist, const int *root_ok, const int *mult, double *W,
                   cudaStream_t st);
// W_ref[k, v] = fl(fl(|graph[c_k]| accept[k]) dgrad_w(mult, |graph[c_k]|, Q, s)), Q = dist_d[k, v] / (1 - p_void[k]):
// the expected reference D step per (root, node) (value_dgrad.cu, DESIGN.md section 5.7), 0 for roots with ok_ref = 0
int value_wref_launch(long long n_node, int ld, const float *emb, const float *bias, const long long *raw_indptr,
                      long long n_roots, const int *roots, const double *dist_d, const double *p_void, const int *ok_ref,
                      const double *accept, const int *mult, double *W, cudaStream_t st);

}  // namespace gg
