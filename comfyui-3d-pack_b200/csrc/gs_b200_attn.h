/* libgs_attn.so: the attention forward behind the `flash_attn` import name (gs_attn.cu), sm_90a.
 * A companion of libgs_b200.so, built beside it by csrc/build.sh and linked against it: argument errors are reported
 * through gs_b200_last_error() (include/gs_b200.h) and launches count in gs_b200's launch counter.  Its header sits
 * with its source because include/ is libgs_b200.so's own boundary (the gs, dr and ngp families), which this library
 * leaves unchanged.  Plain pointers, extern "C", no torch types. */
#ifndef GS_B200_ATTN_H
#define GS_B200_ATTN_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- attention (flash_attn 2.x's forward entry points, head dim 64, no mask) ------------------------------------------
 * B sequences, H heads, head dim d = GS_B200_ATTN_HEAD_DIM.  q: total_q rows, element (row, head, dim) at
 * q[row * q_row_stride + head * q_head_stride + dim] (strides in elements, so packed qkv [*, 3, H, d] / kv [*, 2, H, d]
 * are read in place); k and v likewise with total_k rows.  q, k, v must be 16-byte aligned with strides that are
 * multiples of 8 elements; the last dim is contiguous.  out: contiguous [total_q, H, d], 16-byte aligned.
 * Sequence b: query rows [cu_seqlens_q[b], cu_seqlens_q[b+1]) and key rows [cu_seqlens_k[b], cu_seqlens_k[b+1])
 *   (int32, B + 1 entries each, read on the device only; every bound is clamped into [0, total], so a malformed array
 *   cannot move an access out of the tensors).  A NULL cu_seqlens_q means dense: sequence b is query rows
 *   [b * max_seqlen_q, (b+1) * max_seqlen_q) and total_q must equal B * max_seqlen_q; likewise for cu_seqlens_k.
 * max_seqlen_q only sizes the grid: a hint smaller than the longest sequence still computes every row, with the same bits.
 * out[i, h] = sum over the sequence's keys j of softmax_j(softmax_scale * q_i . k_j) v_j, every head independent; a
 *   sequence with no keys gives 0; rows of out outside every sequence are not written.
 * dtype GS_B200_ATTN_F16 / GS_B200_ATTN_BF16 (q, k, v, out alike): q.k^T and p.v are tensor-core products summed in
 *   fp32; the softmax runs in fp32 on exp2 with softmax_scale * log2(e) folded in, online over 64-key tiles; p is
 *   rounded to the dtype before p.v, the row sum is taken over the unrounded p, and out = O / l is rounded once.
 *   Every sum has a fixed order that depends only on a row's position within its sequence: every output has the same
 *   bits on every run, alone or inside any batch, for any max_seqlen_q hint and any strides.
 * No scratch, no host read; H <= 65535. */
enum { GS_B200_ATTN_F16 = 0, GS_B200_ATTN_BF16 = 1 };
#define GS_B200_ATTN_HEAD_DIM 64
int32_t gs_b200_attn_forward(int32_t dtype, int32_t B, int32_t H, int32_t d, const void* q, int64_t q_row_stride,
                             int64_t q_head_stride, const void* k, int64_t k_row_stride, int64_t k_head_stride,
                             const void* v, int64_t v_row_stride, int64_t v_head_stride, const int32_t* cu_seqlens_q,
                             const int32_t* cu_seqlens_k, int64_t max_seqlen_q, int64_t max_seqlen_k, int64_t total_q,
                             int64_t total_k, float softmax_scale, void* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GS_B200_ATTN_H */
