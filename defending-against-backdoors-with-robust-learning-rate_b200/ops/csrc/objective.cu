// The local objective's instantiations of the flat optimizer kernels (flat_sgd.cuh): the norm pass that also sums g d and d^2, and the
// step that applies G = a g + beta d.  FlatSGD (ops/__init__.py) states the objective; elementwise.cu's launchers call these.
#include "flat_sgd.cuh"

namespace rlr {

void launch_sqnorm_objective(int grid, cudaStream_t st, const float* x, long long n4, double* part, const uint32_t* mask, long long n4_mask,
                             const float* w, const float* w0, long long n4_pgd) {
    if (mask) sqnorm_kernel<true, true><<<grid, 256, 0, st>>>(x, n4, part, mask, n4_mask, w, w0, n4_pgd);
    else sqnorm_kernel<false, true><<<grid, 256, 0, st>>>(x, n4, part, nullptr, 0, w, w0, n4_pgd);
}

void launch_sgd_step_objective(int grid, cudaStream_t st, float* w, const float* g, float* m, const float* w0, __nv_bfloat16* wb, long long n4,
                               float lr, float momentum, float max_grad_norm, const double* sums, double* d_part, long long n4_pgd,
                               const float* w_in, const uint32_t* mask, float obj_a, float obj_b, float obj_mu) {
    if (mask)
        sgd_step_kernel<true, true><<<grid, 256, 0, st>>>(w, g, m, w0, wb, n4, lr, momentum, max_grad_norm, sums, d_part, n4_pgd, w_in,
                                                          w_in ? 1 : 0, mask, obj_a, obj_b, obj_mu);
    else
        sgd_step_kernel<false, true><<<grid, 256, 0, st>>>(w, g, m, w0, wb, n4, lr, momentum, max_grad_norm, sums, d_part, n4_pgd, w_in,
                                                           w_in ? 1 : 0, nullptr, obj_a, obj_b, obj_mu);
}

}  // namespace rlr
