// Camera set-up for a batch of views in ONE launch: replaces the ~20 small torch kernels and the
// two `.item()` host syncs per view of /root/reference/src/model/decoder/cuda_splatting.py:64-87
// and :102-103 (scale-invariant rescale, get_fov, get_projection_matrix, extrinsics.inverse(),
// view @ proj).  One thread per view; everything is a handful of flops.
#include "ps_common.cuh"

namespace ps {

template <typename T>
__device__ void inverse3(const T *m, T *o) {
    const T a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
    const T A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
    const T det = a * A + b * B + c * C;
    const T r = T(1) / det;
    o[0] = A * r; o[1] = -(b * i - c * h) * r; o[2] = (b * f - c * e) * r;
    o[3] = B * r; o[4] = (a * i - c * g) * r;  o[5] = -(a * f - c * d) * r;
    o[6] = C * r; o[7] = -(a * h - b * g) * r; o[8] = (a * e - b * d) * r;
}

// General 4x4 inverse (row-major) by cofactors.
template <typename T>
__device__ void inverse4(const T *m, T *inv) {
    T t[16];
    t[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    t[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    t[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    t[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    t[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    t[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    t[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    t[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    t[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    t[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    t[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    t[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    t[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    t[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    t[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    t[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const T det = m[0] * t[0] + m[1] * t[4] + m[2] * t[8] + m[3] * t[12];
    const T r = T(1) / det;
#pragma unroll
    for (int i = 0; i < 16; ++i) inv[i] = t[i] * r;
}

__device__ float fov_of(const float *kinv, float ax, float ay, float bx, float by) {
    float a[3], b[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        a[i] = kinv[3 * i] * ax + kinv[3 * i + 1] * ay + kinv[3 * i + 2];
        b[i] = kinv[3 * i] * bx + kinv[3 * i + 1] * by + kinv[3 * i + 2];
    }
    const float na = sqrtf(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    const float nb = sqrtf(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
    const float dot = (a[0] / na) * (b[0] / nb) + (a[1] / na) * (b[1] / nb) + (a[2] / na) * (b[2] / nb);
    return acosf(dot);
}

__global__ void k_camera_setup(int n, const float *__restrict__ extr, const float *__restrict__ intr,
                               const float *__restrict__ near_, const float *__restrict__ far_,
                               int scale_invariant, float *__restrict__ view, float *__restrict__ proj,
                               float *__restrict__ campos, float *__restrict__ tanfov,
                               float *__restrict__ scene_scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float e[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) e[k] = extr[16 * i + k];
    float nr = near_[i], fr = far_[i];
    float scale = 1.0f;
    if (scale_invariant) {
        scale = 1.0f / nr;
        e[3] *= scale; e[7] *= scale; e[11] *= scale;
        nr = nr * scale; fr = fr * scale;
    }
    scene_scale[i] = scale;
    float kinv[9];
    inverse3(intr + 9 * i, kinv);
    const float fov_x = fov_of(kinv, 0.0f, 0.5f, 1.0f, 0.5f);
    const float fov_y = fov_of(kinv, 0.5f, 0.0f, 0.5f, 1.0f);
    const float tx = tanf(0.5f * fov_x), ty = tanf(0.5f * fov_y);
    tanfov[2 * i] = tx; tanfov[2 * i + 1] = ty;
    // row-major projection P (cuda_splatting.py:17-44)
    const float top = ty * nr, right = tx * nr;
    float p[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) p[k] = 0.0f;
    p[0] = 2.0f * nr / (right - (-right));
    p[5] = 2.0f * nr / (top - (-top));
    p[14] = 1.0f;                            // [3][2]
    p[10] = fr / (fr - nr);                  // [2][2]
    p[11] = -(fr * nr) / (fr - nr);          // [2][3]
    float w2c[16];
    inverse4(e, w2c);
    // outputs are the row-major storage of the TRANSPOSED matrices (= column-major originals):
    // view_t[r][c] = w2c[c][r];  full_t = view_t @ proj_t, proj_t[r][c] = p[c][r]
    float *vo = view + 16 * i, *po = proj + 16 * i;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            vo[4 * r + c] = w2c[4 * c + r];
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += w2c[4 * k + r] * p[4 * c + k];
            po[4 * r + c] = acc;
        }
    campos[3 * i] = e[3]; campos[3 * i + 1] = e[7]; campos[3 * i + 2] = e[11];
}

__device__ double fov_of_d(const double *kinv, double ax, double ay, double bx, double by) {
    double a[3], b[3];
    for (int i = 0; i < 3; ++i) {
        a[i] = kinv[3 * i] * ax + kinv[3 * i + 1] * ay + kinv[3 * i + 2];
        b[i] = kinv[3 * i] * bx + kinv[3 * i + 1] * by + kinv[3 * i + 2];
    }
    const double na = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    const double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
    return acos((a[0] * b[0] + a[1] * b[1] + a[2] * b[2]) / (na * nb));
}

// Reverse mode of fov_of (float64): adds dL/dkinv for dL/dfov, fov = acos(a^ . b^), a = kinv (ax, ay, 1).
__device__ void fov_of_backward(const double *kinv, double ax, double ay, double bx, double by, double dfov,
                                double *dkinv) {
    const double va[3] = {ax, ay, 1.0}, vb[3] = {bx, by, 1.0};
    double a[3], b[3];
    for (int i = 0; i < 3; ++i) {
        a[i] = kinv[3 * i] * va[0] + kinv[3 * i + 1] * va[1] + kinv[3 * i + 2];
        b[i] = kinv[3 * i] * vb[0] + kinv[3 * i + 1] * vb[1] + kinv[3 * i + 2];
    }
    const double na = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    const double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
    double ua[3], ub[3];
    for (int i = 0; i < 3; ++i) { ua[i] = a[i] / na; ub[i] = b[i] / nb; }
    const double dot = ua[0] * ub[0] + ua[1] * ub[1] + ua[2] * ub[2];
    const double ddot = -dfov / sqrt(1.0 - dot * dot);
    // d(v / |v|) = (dv^ - v^ (v^ . dv^)) / |v| with dv^ = ddot * (the other unit vector)
    const double pa = ddot * (ua[0] * ub[0] + ua[1] * ub[1] + ua[2] * ub[2]);
    for (int i = 0; i < 3; ++i) {
        const double da = (ddot * ub[i] - ua[i] * pa) / na, db = (ddot * ua[i] - ub[i] * pa) / nb;
        for (int j = 0; j < 3; ++j) dkinv[3 * i + j] += da * va[j] + db * vb[j];
    }
}

// One thread per view: recomputes k_camera_setup in float64 and carries the four arrays' gradients back to the
// extrinsics and intrinsics.  An inverse's gradient: Y = X^-1  =>  dL/dX = -Y^T (dL/dY) Y^T.
__global__ void k_camera_setup_backward(int n, const float *__restrict__ extr, const float *__restrict__ intr,
                                        const float *__restrict__ near_, const float *__restrict__ far_,
                                        int scale_invariant,
                                        const float *__restrict__ d_view, const float *__restrict__ d_proj,
                                        const float *__restrict__ d_campos, const float *__restrict__ d_tanfov,
                                        float *__restrict__ d_extr, float *__restrict__ d_intr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double e[16];
    for (int k = 0; k < 16; ++k) e[k] = extr[16 * i + k];
    const double scale = scale_invariant ? 1.0 / (double)near_[i] : 1.0;
    e[3] *= scale; e[7] *= scale; e[11] *= scale;
    double K[9], kinv[9];
    for (int k = 0; k < 9; ++k) K[k] = intr[9 * i + k];
    inverse3(K, kinv);
    const double tx = tan(0.5 * fov_of_d(kinv, 0.0, 0.5, 1.0, 0.5)), ty = tan(0.5 * fov_of_d(kinv, 0.5, 0.0, 0.5, 1.0));
    // row-major projection as k_camera_setup builds it: p[0][0] = 2 near / (2 tan_x near) = 1 / tan_x, p[1][1]
    // likewise; the near / far entries carry no camera input
    const double nr = (double)near_[i] * scale, fr = (double)far_[i] * scale;
    double p[16] = {0.0};
    p[0] = 1.0 / tx; p[5] = 1.0 / ty; p[14] = 1.0; p[10] = fr / (fr - nr); p[11] = -(fr * nr) / (fr - nr);
    double w2c[16];
    inverse4(e, w2c);

    // view_t[r][c] = w2c[c][r]; full_t[r][c] = sum_k w2c[k][r] p[c][k]
    double dw[16] = {0.0};
    double dp0 = 0.0, dp5 = 0.0;
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) {
            if (d_view) dw[4 * c + r] += d_view[16 * i + 4 * r + c];
            if (d_proj) {
                const double g = d_proj[16 * i + 4 * r + c];
                for (int k = 0; k < 4; ++k) dw[4 * k + r] += g * p[4 * c + k];
                if (c == 0) dp0 += g * w2c[r];          // k = 0: w2c[0][r] p[0][0]
                if (c == 1) dp5 += g * w2c[4 + r];      // k = 1: w2c[1][r] p[1][1]
            }
        }
    const double dtx = (d_tanfov ? d_tanfov[2 * i] : 0.0) - dp0 * p[0] / tx;
    const double dty = (d_tanfov ? d_tanfov[2 * i + 1] : 0.0) - dp5 * p[5] / ty;

    double de[16];
    for (int a = 0; a < 4; ++a)
        for (int b = 0; b < 4; ++b) {
            double acc = 0.0;
            for (int x = 0; x < 4; ++x)
                for (int y = 0; y < 4; ++y) acc += w2c[4 * x + a] * dw[4 * x + y] * w2c[4 * b + y];
            de[4 * a + b] = -acc;
        }
    if (d_campos) { de[3] += d_campos[3 * i]; de[7] += d_campos[3 * i + 1]; de[11] += d_campos[3 * i + 2]; }
    de[3] *= scale; de[7] *= scale; de[11] *= scale;
    for (int k = 0; k < 16; ++k) d_extr[16 * i + k] = (float)de[k];

    // tan(fov / 2): d/dfov = (1 + tan^2) / 2
    double dkinv[9] = {0.0};
    fov_of_backward(kinv, 0.0, 0.5, 1.0, 0.5, dtx * 0.5 * (1.0 + tx * tx), dkinv);
    fov_of_backward(kinv, 0.5, 0.0, 0.5, 1.0, dty * 0.5 * (1.0 + ty * ty), dkinv);
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            double acc = 0.0;
            for (int x = 0; x < 3; ++x)
                for (int y = 0; y < 3; ++y) acc += kinv[3 * x + a] * dkinv[3 * x + y] * kinv[3 * b + y];
            d_intr[9 * i + 3 * a + b] = (float)-acc;
        }
}

}  // namespace ps

extern "C" PS_API int ps_camera_setup(int32_t n_views, const float *extrinsics, const float *intrinsics,
                                      const float *near_plane, const float *far_plane,
                                      int32_t scale_invariant, float *viewmatrix, float *projmatrix,
                                      float *campos, float *tanfov, float *scene_scale, void *stream) {
    if (n_views < 1 || !extrinsics || !intrinsics || !near_plane || !far_plane || !viewmatrix ||
        !projmatrix || !campos || !tanfov || !scene_scale) {
        ps::set_error("ps_camera_setup: bad argument");
        return PS_ERR_INVALID_ARGUMENT;
    }
    ps::k_camera_setup<<<(n_views + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(
        n_views, extrinsics, intrinsics, near_plane, far_plane, scale_invariant, viewmatrix, projmatrix,
        campos, tanfov, scene_scale);
    PS_LAUNCH_CHECK("k_camera_setup");
    return PS_OK;
}

extern "C" PS_API int ps_camera_setup_backward(int32_t n_views, const float *extrinsics, const float *intrinsics,
                                               const float *near_plane, const float *far_plane,
                                               int32_t scale_invariant, const float *d_viewmatrix,
                                               const float *d_projmatrix, const float *d_campos,
                                               const float *d_tanfov, float *d_extrinsics, float *d_intrinsics,
                                               void *stream) {
    if (n_views < 1 || !extrinsics || !intrinsics || !near_plane || !far_plane || !d_extrinsics || !d_intrinsics) {
        ps::set_error("ps_camera_setup_backward: bad argument");
        return PS_ERR_INVALID_ARGUMENT;
    }
    ps::k_camera_setup_backward<<<(n_views + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(
        n_views, extrinsics, intrinsics, near_plane, far_plane, scale_invariant, d_viewmatrix, d_projmatrix,
        d_campos, d_tanfov, d_extrinsics, d_intrinsics);
    PS_LAUNCH_CHECK("k_camera_setup_backward");
    return PS_OK;
}
