// torch.optim.Adam's float32 update of one element, shared by the training optimiser (optimizer.cu) and the PLY
// refinement step (ply_import.cu).
#pragma once

namespace ps {

struct AdamConsts {
    float w1, b2, w2, eps;   // 1 - beta1, beta2, 1 - beta2, eps
};

// exp_avg.lerp_(g, 1 - beta1); exp_avg_sq.mul_(beta2).addcmul_(g, g, 1 - beta2);
// p.addcdiv_(exp_avg, exp_avg_sq.sqrt() / bc2_sqrt + eps, -step_size), with step_size = lr_t / (1 - beta1^t) and
// bc2_sqrt = sqrt(1 - beta2^t) rounded to float32 as torch rounds its Python scalars.
__device__ __forceinline__ void adam(float &p, float g, float &m, float &v, const AdamConsts &k, float step_size,
                                     float bc2_sqrt) {
    m = fmaf(k.w1, g - m, m);
    v = fmaf(k.w2 * g, g, v * k.b2);
    p -= step_size * (m / (sqrtf(v) / bc2_sqrt + k.eps));
}

}  // namespace ps
