/* gsr_selective_adam.h — C ABI of the visibility-masked Adam step on the flat parameter buffer
 * (libgsr_selective_adam.so, csrc/gsr_adam_selective.cu).  Conventions of include/gsr_b200.h: device pointers unless
 * the name ends in _host, int status (0 = ok, a cudaError_t value, or GSR_ERR_BAD_ARG), `stream` a cudaStream_t.
 *
 * The step is gsr_adam_step restricted to the rows a view saw.  visible: uint8 [n_rows], nonzero = the row is
 * updated (the rasterizer's frustum-cull mask, `state.visible`).  `step` is the global step count: it drives the bias
 * corrections of every row, visible or not.
 *   - every element of a visible row, in every section, gets gsr_adam_step's per-element arithmetic, bit for bit;
 *   - every other row keeps p, m and v bit-unchanged, and its gradient is never read;
 *   - section padding is left unchanged (a dense step leaves it unchanged too: p, g, m, v are 0 there).
 * An all-nonzero mask therefore gives exactly gsr_adam_step.
 *
 * The sections must be the layout of gsr_flat_numel(n_rows, n_sh_rest): [xyz 3 | quaternion 4 | scale 3 | opacity 1 |
 * rgb 3 | sh 3*n_sh_rest] rows, every section 16-byte aligned, the sh section absent when n_sh_rest == 0
 * (section_end[k] = exclusive end of section k in elements, section_lr[k] its learning rate).  Rows are found from
 * 32-bit offsets, so n_rows * (widest section) must stay below 2^32 (95 M gaussians at SH degree 3).
 *
 * GSR_ERR_BAD_ARG, before any launch, for: n_rows < 0, n_sh_rest < 0, step < 1; sections that are not that layout;
 * a NULL visible or buffer pointer (n_rows > 0); and in the sharded form a bad world, self_rank or [lo, hi). */
#ifndef GSR_SELECTIVE_ADAM_H
#define GSR_SELECTIVE_ADAM_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int gsr_adam_step_selective(int64_t n_rows, int n_sh_rest, float* p, const float* g, float* m, float* v,
                            const uint8_t* visible, int n_sections, const int64_t* section_end,
                            const double* section_lr, double beta1, double beta2, double eps, int step, void* stream);

/* View-parallel form (gsr_adam_step_sharded's conventions): this rank owns elements [lo, hi) of the flat buffer of
 * n_rows gaussians, m_shard / v_shard hold that range.  peer_visible[q] is rank q's mask (peer memory, like the
 * gradients); a row is updated when ANY rank's view saw it, with the rank-ordered mean of every rank's gradient, and
 * its new parameters are stored into every rank's buffer.  Rows no rank saw are left bit-unchanged on every replica,
 * so the replicas stay bit-identical. */
int gsr_adam_step_selective_sharded(int64_t lo, int64_t hi, int world, const float* const* peer_grads,
                                    float* const* peer_params, const uint8_t* const* peer_visible, int self_rank,
                                    float* m_shard, float* v_shard, int64_t n_rows, int n_sh_rest, int n_sections,
                                    const int64_t* section_end, const double* section_lr, double beta1, double beta2,
                                    double eps, int step, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GSR_SELECTIVE_ADAM_H */
