// Preprocess forward: per (scene, Gaussian) thread, looping over the scene's V views.
// Frustum cull, EWA projection, conic, 3-sigma radius, tile rectangle, SH -> RGB, and the
// per-(view, tile) instance histogram (shared-memory privatised, flushed once per block).
//
// COMPILED WITH --fmad=false (see csrc/Makefile): depth bits, radii and rectangles are then
// IEEE-exact functions of the inputs and are checked bit-for-bit against oracle/.
// Semantics: SURVEY.md A.1 / A.4 (upstream forward.cu preprocessCUDA); replaces the
// per-view call made at /root/reference/src/model/decoder/cuda_splatting.py:113-124.
#include "ps_common.cuh"
#include "raster_math.cuh"

namespace ps {

constexpr int kPreThreads = 128;

// Appends the flat indices of the lanes with `flag` to a compact list: one global atomic per warp.
__device__ __forceinline__ void warp_append(bool flag, uint32_t value, uint32_t *list, long long *counter, int lane) {
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (m == 0u) return;
    const int leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader)
        base = atomicAdd(reinterpret_cast<unsigned long long *>(counter), (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (flag) list[base + __popc(m & ((1u << lane) - 1u))] = value;
}

// Geometry for every (scene, Gaussian) x view.  Only a third of the Gaussians of a pixelSplat
// scene land on a given target view, and they are interleaved with the off-screen ones (three
// depth samples per context pixel), so everything that only on-screen Gaussians need -- the
// 300-byte SH row and its evaluation -- is deferred to k_sh_color, which runs densely over the
// compact list built here.
__global__ void __launch_bounds__(kPreThreads)
k_preprocess(Dims d, Inputs in, Geom geo, int use_smem_hist) {
    extern __shared__ uint32_t s_hist[];                         // [V * tiles] when use_smem_hist
    const int hist_n = d.V * d.tiles;
    const int scene = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int g = blockIdx.x * kPreThreads + threadIdx.x;
    const bool live = g < d.P;
    if (use_smem_hist) {
        for (int i = threadIdx.x; i < hist_n; i += kPreThreads) s_hist[i] = 0;
        __syncthreads();
    }
    const size_t sg = (size_t)scene * d.P + (live ? g : 0);
    float mx0 = 0.0f, my0 = 0.0f, mz0 = 0.0f, opacity = 0.0f;
    if (live) {
        mx0 = in.means[3 * sg + 0]; my0 = in.means[3 * sg + 1]; mz0 = in.means[3 * sg + 2];
        opacity = in.opac[sg];
    }
    const float *covp = in.cov + sg * (d.cov_layout == PS_COV_TRIU6 ? 6 : 9);
    // the covariance is fetched together with the mean (one memory round trip instead of two
    // dependent ones); for the culled two thirds this costs a few extra sectors of traffic
    float cov_raw[6];
    {
        float tmp[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
        if (live) load_cov6(covp, d.cov_layout, 1.0f, tmp);
#pragma unroll
        for (int i = 0; i < 6; ++i) cov_raw[i] = tmp[i];
    }

    for (int v = 0; v < d.V; ++v) {
        const int vid = scene * d.V + v;
        const size_t vg = (size_t)vid * d.P + (live ? g : 0);
        const float *__restrict__ vm = in.view + 16 * vid;
        const float *__restrict__ pm = in.proj + 16 * vid;
        const float sc = in.scale ? in.scale[vid] : 1.0f;
        const float px = in.scale ? mx0 * sc : mx0;
        const float py = in.scale ? my0 * sc : my0;
        const float pz = in.scale ? mz0 * sc : mz0;
        bool vis = live;
        float vz = 0.0f;
        if (vis) {
            geo.radii[vg] = 0;
            vz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
            vis = !(vz <= 0.2f);
        }
        if (vis) {
            const float hx = pm[0] * px + pm[4] * py + pm[8] * pz + pm[12];
            const float hy = pm[1] * px + pm[5] * py + pm[9] * pz + pm[13];
            const float hw = pm[3] * px + pm[7] * py + pm[11] * pz + pm[15];
            const float p_w = 1.0f / (hw + 0.0000001f);
            const float projx = hx * p_w, projy = hy * p_w;
            const float tanfovx = in.tanfov[2 * vid], tanfovy = in.tanfov[2 * vid + 1];
            const float focal_x = (float)d.W / (2.0f * tanfovx);
            const float focal_y = (float)d.H / (2.0f * tanfovy);
            float s6[6];
            {
                const float sc2 = sc * sc;
#pragma unroll
                for (int i = 0; i < 6; ++i) s6[i] = in.scale ? cov_raw[i] * sc2 : cov_raw[i];
            }
            Cov2D cv;
            compute_cov2d(px, py, pz, s6, vm, focal_x, focal_y, tanfovx, tanfovy, cv);
            const float det = cv.a * cv.c - cv.b * cv.b;
            vis = !(det == 0.0f);
            if (vis) {
                const float det_inv = 1.0f / det;
                const float mid = 0.5f * (cv.a + cv.c);
                const float sq = sqrtf(fmaxf(0.1f, mid * mid - det));
                const float lambda1 = mid + sq, lambda2 = mid - sq;
                const float my_radius = ceilf(3.0f * sqrtf(fmaxf(lambda1, lambda2)));
                const float pixx = ((projx + 1.0f) * (float)d.W - 1.0f) * 0.5f;
                const float pixy = ((projy + 1.0f) * (float)d.H - 1.0f) * 0.5f;
                const int r = (int)my_radius;
                const float rf = (float)r;
                const int minx = min(d.gx, max(0, (int)((pixx - rf) / (float)kTile)));
                const int miny = min(d.gy, max(0, (int)((pixy - rf) / (float)kTile)));
                const int maxx = min(d.gx, max(0, (int)((pixx + rf + (float)(kTile - 1)) / (float)kTile)));
                const int maxy = min(d.gy, max(0, (int)((pixy + rf + (float)(kTile - 1)) / (float)kTile)));
                vis = (maxx - minx) * (maxy - miny) != 0;
                if (vis) {
                    geo.depth[vg] = vz;
                    geo.radii[vg] = r;
                    geo.xy[vg] = make_float2(pixx, pixy);
                    geo.conic_opacity[vg] = make_float4(cv.c * det_inv, -cv.b * det_inv, cv.a * det_inv, opacity);
                    {
                        const float2 ext = cull_extent(cv.a, cv.c, opacity);
                        geo.cull[vg] = make_float4(pixx, pixy, ext.x, ext.y);
                    }
                    geo.rect[vg] = make_ushort4((unsigned short)minx, (unsigned short)miny,
                                                (unsigned short)maxx, (unsigned short)maxy);
                    if (d.M == 0) {
                        const float *__restrict__ col = in.sh + sg * 3;
                        const float dv = d.depth_mode ? depth_value(d.depth_mode, vz, in.scale, in.near_far, vid) : 0.0f;
                        geo.rgb[vg] = make_float4(col[0], col[1], col[2], dv);
                        geo.clamped[vg] = 0;
                    }
                    for (int ty = miny; ty < maxy; ++ty)
                        for (int tx = minx; tx < maxx; ++tx) {
                            const int t = ty * d.gx + tx;
                            if (use_smem_hist) atomicAdd(&s_hist[v * d.tiles + t], 1u);
                            else atomicAdd(&geo.tile_count[(size_t)vid * d.tiles + t], 1u);
                        }
                }
            }
        }
        warp_append(vis, (uint32_t)vg, geo.vis_pairs, geo.n_instances + 2, lane);
    }
    if (use_smem_hist) {
        __syncthreads();
        uint32_t *dst = geo.tile_count + (size_t)scene * d.V * d.tiles;
        for (int i = threadIdx.x; i < hist_n; i += kPreThreads) {
            const uint32_t c = s_hist[i];
            if (c) atomicAdd(&dst[i], c);
        }
    }
}

// SH -> RGB for the on-screen (view, Gaussian) pairs only, one thread per pair (dense warps).
// The warp first copies its 32 (scattered) 3M-float rows into shared memory with coalesced
// row-wise loads, then every lane evaluates its own row.
constexpr int kShThreads = 128;

__global__ void __launch_bounds__(kShThreads)
k_sh_color(Dims d, Inputs in, Geom geo, int row_stride) {
    extern __shared__ float s_rows[];                            // [warps][32][row_stride]
    const long long n = geo.n_instances[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long i0 = ((long long)blockIdx.x * kShThreads) + warp * 32;
    if (i0 >= n) return;
    const long long i = i0 + lane;
    const bool live = i < n;
    const uint32_t vg = live ? geo.vis_pairs[i] : 0u;
    const uint32_t vid = vg / (uint32_t)d.P, g = vg - vid * (uint32_t)d.P;
    const uint32_t scene = vid / (uint32_t)d.V;
    const size_t sg = (size_t)scene * d.P + g;
    const int sh_n = 3 * d.M;
    float *wrows = s_rows + (size_t)warp * 32 * row_stride;
    // all 32 rows in flight at once (cp.async), the direction set-up below runs under their latency
    gather_rows_async(in.sh, (unsigned long long)sg, __ballot_sync(0xffffffffu, live), sh_n, wrows, row_stride, lane);
    const float sc = in.scale ? in.scale[vid] : 1.0f;
    const float m0 = in.means[3 * sg + 0], m1 = in.means[3 * sg + 1], m2 = in.means[3 * sg + 2];
    const float px = in.scale ? m0 * sc : m0, py = in.scale ? m1 * sc : m1, pz = in.scale ? m2 * sc : m2;
    const float cx = in.campos[3 * vid], cy = in.campos[3 * vid + 1], cz = in.campos[3 * vid + 2];
    const float ddx = px - cx, ddy = py - cy, ddz = pz - cz;
    const float len = sqrtf(ddx * ddx + ddy * ddy + ddz * ddz);
    const float x = ddx / len, y = ddy / len, z = ddz / len;
    gather_rows_wait();
    if (!live) return;
    const float *row = wrows + lane * row_stride;
    float acc[3] = {0.0f, 0.0f, 0.0f};
    const int M = d.M, layout = d.sh_layout;
    const float3 sa = sh_arg(d.sh_basis, x, y, z);
    const uint32_t flip = sh_flip_mask(d.sh_basis);
    sh_for_each(d.deg, sa.x, sa.y, sa.z, [&](int k, float Yk, float, float, float) {
        const float Y = sh_sign(flip, k, Yk);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const float c = row[sh_index(layout, M, k, ch)];
            acc[ch] = k == 0 ? Y * c : acc[ch] + Y * c;
        }
    });
    float rgb[3];
    uint8_t clamp_bits = 0;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float a = acc[ch] + 0.5f;
        if (a < 0.0f) clamp_bits |= (uint8_t)(1u << ch);
        rgb[ch] = fmaxf(a, 0.0f);
    }
    // depth channel in the spare lane (the same function of the same vz as the colors_precomp branch above)
    const float dv = d.depth_mode ? depth_value(d.depth_mode, geo.depth[vg], in.scale, in.near_far, (int)vid) : 0.0f;
    geo.rgb[vg] = make_float4(rgb[0], rgb[1], rgb[2], dv);
    geo.clamped[vg] = clamp_bits;
}

int launch_sh_color(const Dims &d, const Inputs &in, const Geom &g, cudaStream_t st) {
    if (d.M == 0) return PS_OK;
    // the pair count lives on the device: launch for the worst case, surplus warps exit at once
    const int row_stride = (3 * d.M) | 1;
    const size_t smem = sizeof(float) * kShThreads * row_stride;
    static unsigned long long attr_devices = 0;
    if (first_use_on_device(attr_devices)) {
        PS_CUDA_CHECK(cudaFuncSetAttribute(k_sh_color, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    }
    const long long pairs = (long long)d.S * d.V * d.P;
    k_sh_color<<<(unsigned)((pairs + kShThreads - 1) / kShThreads), kShThreads, smem, st>>>(d, in, g, row_stride);
    PS_LAUNCH_CHECK("k_sh_color");
    return PS_OK;
}

int launch_preprocess(const Dims &d, const Inputs &in, const Geom &g, cudaStream_t st) {
    PS_CUDA_CHECK(cudaMemsetAsync(g.tile_count, 0, sizeof(uint32_t) * (size_t)d.S * d.V * d.tiles, st));
    PS_CUDA_CHECK(cudaMemsetAsync(g.n_instances, 0, 4 * sizeof(long long), st));
    const size_t hist_bytes = sizeof(uint32_t) * (size_t)d.V * d.tiles;
    const int use_smem = hist_bytes <= 32 * 1024;
    dim3 grid((d.P + kPreThreads - 1) / kPreThreads, d.S);
    k_preprocess<<<grid, kPreThreads, use_smem ? hist_bytes : 0, st>>>(d, in, g, use_smem);
    PS_LAUNCH_CHECK("k_preprocess");
    return PS_OK;
}

}  // namespace ps
