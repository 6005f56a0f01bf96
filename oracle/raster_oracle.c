/*
 * oracle/raster_oracle.c -- CPU restatement of the tile rasterizer used by
 * pixelSplat's decoder.  TEST INFRASTRUCTURE ONLY: nothing in pixelsplat_b200/
 * may include, link or call this file; only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs use it, as the checker.
 *
 * PARITY UNPINNED.  The algorithm lives in a third-party dependency that is
 * absent from /root/reference: diff-gaussian-rasterization-modified
 * (requirements.txt:17, a bare git URL, no commit pin), a fork of
 * graphdeco-inria/diff-gaussian-rasterization.  The reference holds no golden
 * vector or known-answer test for it (src/scripts/test_splatter.py is a visual
 * smoke script), so this file restates the *published* 3DGS rasterizer
 * algorithm (SURVEY.md Appendix A) and is anchored on the reference's call
 * site src/model/decoder/cuda_splatting.py:99-124 (argument conventions:
 * column-major view/proj matrices :85-87, cov3D_precomp in triu order
 * :115,123, SH laid out [P, M, 3] :75, sh_degree = isqrt(d_sh)-1 :74,
 * prefiltered=False :110).  Degree-4 SH is the fork's addition; its exact
 * form cannot be read offline and is ASSUMED to be the standard real-SH
 * degree-4 block (SURVEY.md A.4 / A.7).
 *
 * Build twice (see oracle/Makefile): float (bit-level model of the fp32 GPU
 * arithmetic, compiled with -ffp-contract=off so no FMA is formed) and double
 * (-DORACLE_F64, used to pin the hand-derived backward against torch autograd).
 *
 * Every stage is a separate entry point so tests can compare intermediates:
 *   orc_preprocess        SURVEY A.1 + A.4   (upstream forward.cu preprocessCUDA)
 *   orc_bin               SURVEY A.2         (duplicateWithKeys + radix sort + identifyTileRanges)
 *   orc_composite_fwd     SURVEY A.3         (upstream forward.cu renderCUDA)
 *   orc_composite_margins per pixel, how close the forward's walk came to taking another branch
 *   orc_composite_bwd     SURVEY A.5         (upstream backward.cu renderCUDA)
 *   orc_preprocess_bwd    SURVEY A.5         (computeCov2DCUDA + preprocessCUDA backward)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef ORACLE_F64
typedef double real;
#define R_SQRT sqrt
#define R_EXP exp
#define R_CEIL ceil
#else
typedef float real;
#define R_SQRT sqrtf
#define R_EXP expf
#define R_CEIL ceilf
#endif

#define K(x) ((real)(x))
#define TILE 16

static const double SH_C0 = 0.28209479177387814;
static const double SH_C1 = 0.4886025119029199;
static const double SH_C2[5] = {1.0925484305920792, -1.0925484305920792, 0.31539156525252005,
                                -1.0925484305920792, 0.5462742152960396};
static const double SH_C3[7] = {-0.5900435899266435, 2.890611442640554, -0.4570457994644658,
                                0.3731763325901154, -0.4570457994644658, 1.445305721320277,
                                -0.5900435899266435};
static const double SH_C4[9] = {2.5033429417967046, -1.7701307697799304, 0.9461746957575601,
                                -0.6690465435572892, 0.10578554691520431, -0.6690465435572892,
                                0.47308734787878004, -1.7701307697799304, 0.6258357354491761};

static inline real rmin(real a, real b) { return a < b ? a : b; }
static inline real rmax(real a, real b) { return a > b ? a : b; }
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

int orc_real_bytes(void) { return (int)sizeof(real); }

/* Real-SH basis, degrees 0..4, 3DGS sign convention (SURVEY A.4). */
static void sh_basis_3dgs(int deg, real x, real y, real z, real *b) {
    b[0] = K(SH_C0);
    if (deg < 1) return;
    b[1] = -K(SH_C1) * y;
    b[2] = K(SH_C1) * z;
    b[3] = -K(SH_C1) * x;
    if (deg < 2) return;
    real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    b[4] = K(SH_C2[0]) * xy;
    b[5] = K(SH_C2[1]) * yz;
    b[6] = K(SH_C2[2]) * (K(2) * zz - xx - yy);
    b[7] = K(SH_C2[3]) * xz;
    b[8] = K(SH_C2[4]) * (xx - yy);
    if (deg < 3) return;
    b[9] = K(SH_C3[0]) * y * (K(3) * xx - yy);
    b[10] = K(SH_C3[1]) * xy * z;
    b[11] = K(SH_C3[2]) * y * (K(4) * zz - xx - yy);
    b[12] = K(SH_C3[3]) * z * (K(2) * zz - K(3) * xx - K(3) * yy);
    b[13] = K(SH_C3[4]) * x * (K(4) * zz - xx - yy);
    b[14] = K(SH_C3[5]) * z * (xx - yy);
    b[15] = K(SH_C3[6]) * x * (xx - K(3) * yy);
    if (deg < 4) return;
    b[16] = K(SH_C4[0]) * xy * (xx - yy);
    b[17] = K(SH_C4[1]) * yz * (K(3) * xx - yy);
    b[18] = K(SH_C4[2]) * xy * (K(7) * zz - K(1));
    b[19] = K(SH_C4[3]) * yz * (K(7) * zz - K(3));
    b[20] = K(SH_C4[4]) * (zz * (K(35) * zz - K(30)) + K(3));
    b[21] = K(SH_C4[5]) * xz * (K(7) * zz - K(3));
    b[22] = K(SH_C4[6]) * (xx - yy) * (K(7) * zz - K(1));
    b[23] = K(SH_C4[7]) * xz * (xx - K(3) * yy);
    b[24] = K(SH_C4[8]) * (xx * (xx - K(3) * yy) - yy * (K(3) * xx - yy));
}

/* d basis / d (x,y,z), treating x,y,z as independent (the normalisation
 * Jacobian is applied by the caller). */
static void sh_basis_grad_3dgs(int deg, real x, real y, real z, real *dx, real *dy, real *dz) {
    for (int i = 0; i < 25; ++i) dx[i] = dy[i] = dz[i] = 0;
    if (deg < 1) return;
    dy[1] = -K(SH_C1);
    dz[2] = K(SH_C1);
    dx[3] = -K(SH_C1);
    if (deg < 2) return;
    real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    dx[4] = K(SH_C2[0]) * y;            dy[4] = K(SH_C2[0]) * x;
    dy[5] = K(SH_C2[1]) * z;            dz[5] = K(SH_C2[1]) * y;
    dx[6] = K(SH_C2[2]) * K(-2) * x;    dy[6] = K(SH_C2[2]) * K(-2) * y;  dz[6] = K(SH_C2[2]) * K(4) * z;
    dx[7] = K(SH_C2[3]) * z;            dz[7] = K(SH_C2[3]) * x;
    dx[8] = K(SH_C2[4]) * K(2) * x;     dy[8] = K(SH_C2[4]) * K(-2) * y;
    if (deg < 3) return;
    dx[9] = K(SH_C3[0]) * K(6) * xy;                     dy[9] = K(SH_C3[0]) * (K(3) * xx - K(3) * yy);
    dx[10] = K(SH_C3[1]) * yz;  dy[10] = K(SH_C3[1]) * xz;  dz[10] = K(SH_C3[1]) * xy;
    dx[11] = K(SH_C3[2]) * K(-2) * xy;  dy[11] = K(SH_C3[2]) * (K(4) * zz - xx - K(3) * yy);  dz[11] = K(SH_C3[2]) * K(8) * yz;
    dx[12] = K(SH_C3[3]) * K(-6) * xz;  dy[12] = K(SH_C3[3]) * K(-6) * yz;  dz[12] = K(SH_C3[3]) * (K(6) * zz - K(3) * xx - K(3) * yy);
    dx[13] = K(SH_C3[4]) * (K(4) * zz - K(3) * xx - yy);  dy[13] = K(SH_C3[4]) * K(-2) * xy;  dz[13] = K(SH_C3[4]) * K(8) * xz;
    dx[14] = K(SH_C3[5]) * K(2) * xz;   dy[14] = K(SH_C3[5]) * K(-2) * yz;  dz[14] = K(SH_C3[5]) * (xx - yy);
    dx[15] = K(SH_C3[6]) * (K(3) * xx - K(3) * yy);      dy[15] = K(SH_C3[6]) * K(-6) * xy;
    if (deg < 4) return;
    /* b16 = c xy(xx-yy) = c (x^3 y - x y^3) */
    dx[16] = K(SH_C4[0]) * (K(3) * xx * y - yy * y);     dy[16] = K(SH_C4[0]) * (xx * x - K(3) * x * yy);
    /* b17 = c yz(3xx-yy) */
    dx[17] = K(SH_C4[1]) * K(6) * xy * z;  dy[17] = K(SH_C4[1]) * z * (K(3) * xx - K(3) * yy);  dz[17] = K(SH_C4[1]) * y * (K(3) * xx - yy);
    /* b18 = c xy(7zz-1) */
    dx[18] = K(SH_C4[2]) * y * (K(7) * zz - K(1));  dy[18] = K(SH_C4[2]) * x * (K(7) * zz - K(1));  dz[18] = K(SH_C4[2]) * K(14) * xy * z;
    /* b19 = c yz(7zz-3) */
    dy[19] = K(SH_C4[3]) * z * (K(7) * zz - K(3));  dz[19] = K(SH_C4[3]) * y * (K(21) * zz - K(3));
    /* b20 = c (35 z^4 - 30 z^2 + 3) */
    dz[20] = K(SH_C4[4]) * (K(140) * zz * z - K(60) * z);
    /* b21 = c xz(7zz-3) */
    dx[21] = K(SH_C4[5]) * z * (K(7) * zz - K(3));  dz[21] = K(SH_C4[5]) * x * (K(21) * zz - K(3));
    /* b22 = c (xx-yy)(7zz-1) */
    dx[22] = K(SH_C4[6]) * K(2) * x * (K(7) * zz - K(1));  dy[22] = K(SH_C4[6]) * K(-2) * y * (K(7) * zz - K(1));  dz[22] = K(SH_C4[6]) * K(14) * z * (xx - yy);
    /* b23 = c xz(xx-3yy) */
    dx[23] = K(SH_C4[7]) * z * (K(3) * xx - K(3) * yy);  dy[23] = K(SH_C4[7]) * K(-6) * xy * z;  dz[23] = K(SH_C4[7]) * x * (xx - K(3) * yy);
    /* b24 = c (x^4 - 6 x^2 y^2 + y^4) */
    dx[24] = K(SH_C4[8]) * (K(4) * xx * x - K(12) * x * yy);  dy[24] = K(SH_C4[8]) * (K(4) * yy * y - K(12) * xx * y);
}

/* SH convention switch (include/pixelsplat_b200.h PS_SH_BASIS_*): 0 = 3DGS (default), 1 = e3nn, the
 * basis in which the reference rotates its coefficients (src/misc/sh_rotation.py:18-22):
 *   Y_e3nn,k(x, y, z) = (-1)^m Y_3dgs,k(z, x, y),  and (-1)^m = (-1)^k because l^2 + l is even. */
static int g_sh_convention = 0;
void orc_set_sh_basis(int convention) { g_sh_convention = convention; }

static void sh_basis(int deg, real x, real y, real z, real *b) {
    if (g_sh_convention == 0) { sh_basis_3dgs(deg, x, y, z, b); return; }
    sh_basis_3dgs(deg, z, x, y, b);
    for (int k = 1; k < (deg + 1) * (deg + 1); k += 2) b[k] = -b[k];
}

static void sh_basis_grad(int deg, real x, real y, real z, real *dx, real *dy, real *dz) {
    if (g_sh_convention == 0) { sh_basis_grad_3dgs(deg, x, y, z, dx, dy, dz); return; }
    /* f(x, y, z) = g(a, b, c) at (a, b, c) = (z, x, y): df/dx = dg/db, df/dy = dg/dc, df/dz = dg/da */
    sh_basis_grad_3dgs(deg, z, x, y, dz, dx, dy);
    for (int k = 1; k < 25; k += 2) { dx[k] = -dx[k]; dy[k] = -dy[k]; dz[k] = -dz[k]; }
}

typedef struct {
    real tx, ty, tz;            /* view-space mean */
    real ctx, cty;              /* clamped */
    int clamp_x, clamp_y;       /* 1 if the +-1.3 tanfov clamp was active */
    real j00, j02, j11, j12;
    real m[2][3];               /* M = J * R */
    real a, b, c;               /* cov2D + 0.3 I */
} cov2d_t;

static void cov2d(const real *p, const real *cov6, const real *vm, real focal_x, real focal_y,
                  real tanfovx, real tanfovy, cov2d_t *o) {
    real px = p[0], py = p[1], pz = p[2];
    o->tx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12];
    o->ty = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13];
    o->tz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
    real limx = K(1.3) * tanfovx, limy = K(1.3) * tanfovy;
    real txtz = o->tx / o->tz, tytz = o->ty / o->tz;
    o->clamp_x = (txtz < -limx || txtz > limx);
    o->clamp_y = (tytz < -limy || tytz > limy);
    o->ctx = rmin(limx, rmax(-limx, txtz)) * o->tz;
    o->cty = rmin(limy, rmax(-limy, tytz)) * o->tz;
    real tz = o->tz;
    o->j00 = focal_x / tz;
    o->j02 = -(focal_x * o->ctx) / (tz * tz);
    o->j11 = focal_y / tz;
    o->j12 = -(focal_y * o->cty) / (tz * tz);
    /* R[i][j] = vm[4*j+i] */
    for (int j = 0; j < 3; ++j) {
        o->m[0][j] = o->j00 * vm[4 * j + 0] + o->j02 * vm[4 * j + 2];
        o->m[1][j] = o->j11 * vm[4 * j + 1] + o->j12 * vm[4 * j + 2];
    }
    real sxx = cov6[0], sxy = cov6[1], sxz = cov6[2], syy = cov6[3], syz = cov6[4], szz = cov6[5];
    const real *m0 = o->m[0], *m1 = o->m[1];
    real v0x = sxx * m0[0] + sxy * m0[1] + sxz * m0[2];
    real v0y = sxy * m0[0] + syy * m0[1] + syz * m0[2];
    real v0z = sxz * m0[0] + syz * m0[1] + szz * m0[2];
    real v1x = sxx * m1[0] + sxy * m1[1] + sxz * m1[2];
    real v1y = sxy * m1[0] + syy * m1[1] + syz * m1[2];
    real v1z = sxz * m1[0] + syz * m1[1] + szz * m1[2];
    o->a = m0[0] * v0x + m0[1] * v0y + m0[2] * v0z + K(0.3);
    o->b = m0[0] * v1x + m0[1] * v1y + m0[2] * v1z;
    o->c = m1[0] * v1x + m1[1] * v1y + m1[2] * v1z + K(0.3);
}

/*
 * orc_preprocess: one view, P Gaussians.
 *   sh: [P, M, 3] if M > 0 (degree deg), else colors: [P, 3] used as-is.
 *   outputs (all length P unless noted): depth, radii(int32), xy[2P], conic_opacity[4P], rgb[3P],
 *   clamped(uint8)[3P], rect(int32)[4P] = (minx,miny,maxx,maxy) in tiles, tiles_touched(uint32).
 */
void orc_preprocess(int P, int M, int deg, const real *means, const real *cov6, const real *opac,
                    const real *sh_or_colors, const real *vm, const real *pm, const real *campos,
                    real tanfovx, real tanfovy, int W, int H, real *depth, int32_t *radii, real *xy,
                    real *conic_opacity, real *rgb, uint8_t *clamped, int32_t *rect,
                    uint32_t *tiles_touched) {
    int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    real focal_x = (real)W / (K(2) * tanfovx), focal_y = (real)H / (K(2) * tanfovy);
    for (int g = 0; g < P; ++g) {
        radii[g] = 0;
        tiles_touched[g] = 0;
        depth[g] = 0;
        xy[2 * g] = xy[2 * g + 1] = 0;
        for (int k = 0; k < 4; ++k) conic_opacity[4 * g + k] = 0, rect[4 * g + k] = 0;
        for (int k = 0; k < 3; ++k) rgb[3 * g + k] = 0, clamped[3 * g + k] = 0;
        const real *p = means + 3 * g;
        real vz = vm[2] * p[0] + vm[6] * p[1] + vm[10] * p[2] + vm[14];
        if (vz <= K(0.2)) continue;
        real hx = pm[0] * p[0] + pm[4] * p[1] + pm[8] * p[2] + pm[12];
        real hy = pm[1] * p[0] + pm[5] * p[1] + pm[9] * p[2] + pm[13];
        real hw = pm[3] * p[0] + pm[7] * p[1] + pm[11] * p[2] + pm[15];
        real p_w = K(1) / (hw + K(1e-7));
        real projx = hx * p_w, projy = hy * p_w;
        cov2d_t cv;
        cov2d(p, cov6 + 6 * g, vm, focal_x, focal_y, tanfovx, tanfovy, &cv);
        real det = cv.a * cv.c - cv.b * cv.b;
        if (det == K(0)) continue;
        real det_inv = K(1) / det;
        real mid = K(0.5) * (cv.a + cv.c);
        real sq = R_SQRT(rmax(K(0.1), mid * mid - det));
        real lambda1 = mid + sq, lambda2 = mid - sq;
        real my_radius = R_CEIL(K(3) * R_SQRT(rmax(lambda1, lambda2)));
        real pixx = ((projx + K(1)) * (real)W - K(1)) * K(0.5);
        real pixy = ((projy + K(1)) * (real)H - K(1)) * K(0.5);
        int r = (int)my_radius;
        int minx = imin(gx, imax(0, (int)((pixx - (real)r) / K(TILE))));
        int miny = imin(gy, imax(0, (int)((pixy - (real)r) / K(TILE))));
        int maxx = imin(gx, imax(0, (int)((pixx + (real)r + K(TILE - 1)) / K(TILE))));
        int maxy = imin(gy, imax(0, (int)((pixy + (real)r + K(TILE - 1)) / K(TILE))));
        if ((maxx - minx) * (maxy - miny) == 0) continue;
        if (M > 0) {
            real dx = p[0] - campos[0], dy = p[1] - campos[1], dz = p[2] - campos[2];
            real len = R_SQRT(dx * dx + dy * dy + dz * dz);
            real x = dx / len, y = dy / len, z = dz / len;
            real basis[25];
            sh_basis(deg, x, y, z, basis);
            int nb = (deg + 1) * (deg + 1);
            const real *s = sh_or_colors + (size_t)g * M * 3;
            for (int ch = 0; ch < 3; ++ch) {
                real acc = basis[0] * s[ch];
                for (int k = 1; k < nb; ++k) acc = acc + basis[k] * s[3 * k + ch];
                acc = acc + K(0.5);
                clamped[3 * g + ch] = (acc < K(0));
                rgb[3 * g + ch] = rmax(acc, K(0));
            }
        } else {
            for (int ch = 0; ch < 3; ++ch) rgb[3 * g + ch] = sh_or_colors[3 * g + ch];
        }
        depth[g] = vz;
        radii[g] = r;
        xy[2 * g] = pixx;
        xy[2 * g + 1] = pixy;
        conic_opacity[4 * g + 0] = cv.c * det_inv;
        conic_opacity[4 * g + 1] = -cv.b * det_inv;
        conic_opacity[4 * g + 2] = cv.a * det_inv;
        conic_opacity[4 * g + 3] = opac[g];
        rect[4 * g + 0] = minx; rect[4 * g + 1] = miny; rect[4 * g + 2] = maxx; rect[4 * g + 3] = maxy;
        tiles_touched[g] = (uint32_t)((maxx - minx) * (maxy - miny));
    }
}

typedef struct { uint64_t key; uint32_t val; uint32_t seq; } inst_t;
static int inst_cmp(const void *a, const void *b) {
    const inst_t *x = (const inst_t *)a, *y = (const inst_t *)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->seq < y->seq ? -1 : (x->seq > y->seq);
}

/*
 * orc_bin: emission in Gaussian order (rect row-major), key = tile<<32 | float_bits(depth),
 * stable sort, per-tile [start,end).  keys/values must hold sum(tiles_touched) entries.
 * Returns N.
 */
int64_t orc_bin(int P, const real *depth, const int32_t *radii, const int32_t *rect, int W, int H,
                uint64_t *keys, uint32_t *values, uint32_t *ranges /* [tiles][2] */) {
    int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    int64_t N = 0;
    for (int g = 0; g < P; ++g)
        if (radii[g] > 0) N += (int64_t)(rect[4 * g + 2] - rect[4 * g]) * (rect[4 * g + 3] - rect[4 * g + 1]);
    inst_t *inst = (inst_t *)malloc(sizeof(inst_t) * (size_t)(N > 0 ? N : 1));
    int64_t n = 0;
    for (int g = 0; g < P; ++g) {
        if (radii[g] <= 0) continue;
        float df = (float)depth[g];
        uint32_t bits;
        memcpy(&bits, &df, 4);
        for (int y = rect[4 * g + 1]; y < rect[4 * g + 3]; ++y)
            for (int x = rect[4 * g]; x < rect[4 * g + 2]; ++x) {
                inst[n].key = ((uint64_t)(uint32_t)(y * gx + x) << 32) | bits;
                inst[n].val = (uint32_t)g;
                inst[n].seq = (uint32_t)n;
                ++n;
            }
    }
    qsort(inst, (size_t)N, sizeof(inst_t), inst_cmp);
    for (int t = 0; t < gx * gy; ++t) ranges[2 * t] = ranges[2 * t + 1] = 0;
    for (int64_t i = 0; i < N; ++i) {
        keys[i] = inst[i].key;
        values[i] = inst[i].val;
        uint32_t t = (uint32_t)(inst[i].key >> 32);
        if (i == 0 || t != (uint32_t)(inst[i - 1].key >> 32)) ranges[2 * t] = (uint32_t)i;
        if (i == N - 1 || t != (uint32_t)(inst[i + 1].key >> 32)) ranges[2 * t + 1] = (uint32_t)(i + 1);
    }
    free(inst);
    return N;
}

/* orc_composite_fwd: SURVEY A.3.  out_color planar [3,H,W]. */
void orc_composite_fwd(int W, int H, const uint32_t *ranges, const uint32_t *values, const real *xy,
                       const real *conic_opacity, const real *rgb, const real *bg, real *out_color,
                       real *final_T, uint32_t *n_contrib) {
    int gx = (W + TILE - 1) / TILE;
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px) {
            int tile = (py / TILE) * gx + (px / TILE);
            uint32_t s = ranges[2 * tile], e = ranges[2 * tile + 1];
            real T = K(1), C[3] = {0, 0, 0};
            uint32_t contributor = 0, last = 0;
            real pxf = (real)px, pyf = (real)py;
            for (uint32_t i = s; i < e; ++i) {
                ++contributor;
                uint32_t g = values[i];
                real dx = xy[2 * g] - pxf, dy = xy[2 * g + 1] - pyf;
                const real *co = conic_opacity + 4 * g;
                real power = K(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                if (power > K(0)) continue;
                real alpha = rmin(K(0.99), co[3] * R_EXP(power));
                if (alpha < K(1.0 / 255.0)) continue;
                real test_T = T * (K(1) - alpha);
                if (test_T < K(0.0001)) break;
                for (int ch = 0; ch < 3; ++ch) C[ch] += rgb[3 * g + ch] * alpha * T;
                T = test_T;
                last = contributor;
            }
            int pix = py * W + px;
            final_T[pix] = T;
            n_contrib[pix] = last;
            for (int ch = 0; ch < 3; ++ch) out_color[ch * H * W + pix] = C[ch] + T * bg[ch];
        }
}

/*
 * orc_composite_margins: how close each pixel's walk came to taking another branch.  Walks the list exactly as
 * orc_composite_fwd does, up to and including the entry at which it breaks, and writes per pixel [H, W] the
 * smallest distance of each decision value from its threshold over the entries it looked at:
 *   m_alpha  min |alpha / (1/255) - 1|   (alpha after min(0.99, .), over entries that reach the alpha test)
 *   m_T      min |test_T / 1e-4 - 1|     (over entries that reach the T test, the breaking one included)
 *   m_power  min |power|                 (over entries whose sign test can matter: power > 0, or power within
 *            ORC_POWER_REL of zero relative to the products it is a difference of, |co| dx^2 ...; that is as far
 *            as a float32 evaluation in another order or with FMAs can move it across 0.  The margin itself is
 *            absolute, because the threshold is 0 and an implementation may place its test a fixed distance
 *            above 0 to keep such rounding from dropping a pixel that sits on a Gaussian's centre: the
 *            warp-task compositor rejects at log2-power > 1e-4.  A positive power of a positive-definite conic
 *            is a rounding artefact, so every positive value counts.  dx = dy = 0 does not: every product is
 *            then exactly 0 and so is the power, whatever the order.)
 * A margin no entry contributed to is ORC_NO_MARGIN.
 */
#define ORC_POWER_REL 1.0e-5
#define ORC_NO_MARGIN 1.0e30
void orc_composite_margins(int W, int H, const uint32_t *ranges, const uint32_t *values, const real *xy,
                           const real *conic_opacity, real *m_alpha, real *m_T, real *m_power) {
    int gx = (W + TILE - 1) / TILE;
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px) {
            int tile = (py / TILE) * gx + (px / TILE);
            uint32_t s = ranges[2 * tile], e = ranges[2 * tile + 1];
            real T = K(1), ma = K(ORC_NO_MARGIN), mt = K(ORC_NO_MARGIN), mp = K(ORC_NO_MARGIN);
            real pxf = (real)px, pyf = (real)py;
            for (uint32_t i = s; i < e; ++i) {
                uint32_t g = values[i];
                real dx = xy[2 * g] - pxf, dy = xy[2 * g + 1] - pyf;
                const real *co = conic_opacity + 4 * g;
                real power = K(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                real ax = co[0] * dx * dx, ay = co[2] * dy * dy, ab = co[1] * dx * dy;
                real terms = K(0.5) * ((ax < K(0) ? -ax : ax) + (ay < K(0) ? -ay : ay)) + (ab < K(0) ? -ab : ab);
                if (power > K(0) || (terms > K(0) && power >= K(-ORC_POWER_REL) * terms))
                    mp = rmin(mp, power < K(0) ? -power : power);
                if (power > K(0)) continue;
                real alpha = rmin(K(0.99), co[3] * R_EXP(power));
                real da = alpha / K(1.0 / 255.0) - K(1);
                ma = rmin(ma, da < K(0) ? -da : da);
                if (alpha < K(1.0 / 255.0)) continue;
                real test_T = T * (K(1) - alpha);
                real dt = test_T / K(0.0001) - K(1);
                mt = rmin(mt, dt < K(0) ? -dt : dt);
                if (test_T < K(0.0001)) break;
                T = test_T;
            }
            int pix = py * W + px;
            m_alpha[pix] = ma;
            m_T[pix] = mt;
            m_power[pix] = mp;
        }
}

/*
 * orc_composite_bwd: SURVEY A.5.  Gradient sums are accumulated in double (the oracle is the
 * accuracy reference; the GPU's atomic order is arbitrary anyway).
 * Outputs (double, zero-initialised here): dL_dmean2D[2P] (NDC-scaled like upstream),
 * dL_dconic[3P] (x, y(=half-weight B), z), dL_dopacity[P], dL_dcolor[3P].
 */
void orc_composite_bwd(int P, int W, int H, const uint32_t *ranges, const uint32_t *values,
                       const real *xy, const real *conic_opacity, const real *rgb, const real *bg,
                       const real *final_T, const uint32_t *n_contrib, const real *dL_dpix,
                       double *dL_dmean2D, double *dL_dconic, double *dL_dopacity, double *dL_dcolor) {
    int gx = (W + TILE - 1) / TILE;
    memset(dL_dmean2D, 0, sizeof(double) * 2 * (size_t)P);
    memset(dL_dconic, 0, sizeof(double) * 3 * (size_t)P);
    memset(dL_dopacity, 0, sizeof(double) * (size_t)P);
    memset(dL_dcolor, 0, sizeof(double) * 3 * (size_t)P);
    real ddelx_dx = K(0.5) * (real)W, ddely_dy = K(0.5) * (real)H;
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px) {
            int tile = (py / TILE) * gx + (px / TILE);
            uint32_t s = ranges[2 * tile];
            int pix = py * W + px;
            real T_final = final_T[pix], T = T_final;
            uint32_t last = n_contrib[pix];
            real accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_alpha = 0;
            real dpix[3];
            for (int ch = 0; ch < 3; ++ch) dpix[ch] = dL_dpix[ch * H * W + pix];
            real bg_dot = bg[0] * dpix[0] + bg[1] * dpix[1] + bg[2] * dpix[2];
            real pxf = (real)px, pyf = (real)py;
            for (uint32_t k = last; k-- > 0;) { /* contributor index k (0-based) < last */
                uint32_t g = values[s + k];
                real dx = xy[2 * g] - pxf, dy = xy[2 * g + 1] - pyf;
                const real *co = conic_opacity + 4 * g;
                real power = K(-0.5) * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                if (power > K(0)) continue;
                real G = R_EXP(power);
                real alpha = rmin(K(0.99), co[3] * G);
                if (alpha < K(1.0 / 255.0)) continue;
                T = T / (K(1) - alpha);
                real dchannel_dcolor = alpha * T;
                real dL_dalpha = 0;
                for (int ch = 0; ch < 3; ++ch) {
                    real c = rgb[3 * g + ch];
                    accum_rec[ch] = last_alpha * last_color[ch] + (K(1) - last_alpha) * accum_rec[ch];
                    last_color[ch] = c;
                    dL_dalpha += (c - accum_rec[ch]) * dpix[ch];
                    dL_dcolor[3 * g + ch] += (double)(dchannel_dcolor * dpix[ch]);
                }
                dL_dalpha *= T;
                last_alpha = alpha;
                dL_dalpha += (-T_final / (K(1) - alpha)) * bg_dot;
                real dL_dG = co[3] * dL_dalpha;
                real gdx = G * dx, gdy = G * dy;
                real dG_ddelx = -gdx * co[0] - gdy * co[1];
                real dG_ddely = -gdy * co[2] - gdx * co[1];
                dL_dmean2D[2 * g] += (double)(dL_dG * dG_ddelx * ddelx_dx);
                dL_dmean2D[2 * g + 1] += (double)(dL_dG * dG_ddely * ddely_dy);
                dL_dconic[3 * g] += (double)(K(-0.5) * gdx * dx * dL_dG);
                dL_dconic[3 * g + 1] += (double)(K(-0.5) * gdx * dy * dL_dG);
                dL_dconic[3 * g + 2] += (double)(K(-0.5) * gdy * dy * dL_dG);
                dL_dopacity[g] += (double)(G * dL_dalpha);
            }
        }
}

/*
 * orc_preprocess_bwd: SURVEY A.5 (computeCov2DCUDA + preprocessCUDA backward).
 * Inputs: the per-Gaussian gradients produced by orc_composite_bwd (as `real`),
 * outputs dL_dmeans[3P], dL_dcov6[6P], dL_dsh[P*M*3] (or nothing when M == 0; then
 * dL_dcolor already is the colour gradient).
 */
void orc_preprocess_bwd(int P, int M, int deg, const real *means, const real *cov6,
                        const real *sh, const real *vm, const real *pm, const real *campos,
                        real tanfovx, real tanfovy, int W, int H, const int32_t *radii,
                        const uint8_t *clamped, const real *dL_dmean2D, const real *dL_dconic,
                        const real *dL_dcolor, real *dL_dmeans, real *dL_dcov6, real *dL_dsh) {
    real focal_x = (real)W / (K(2) * tanfovx), focal_y = (real)H / (K(2) * tanfovy);
    for (int g = 0; g < P; ++g) {
        for (int k = 0; k < 3; ++k) dL_dmeans[3 * g + k] = 0;
        for (int k = 0; k < 6; ++k) dL_dcov6[6 * g + k] = 0;
        if (M > 0) for (int k = 0; k < 3 * M; ++k) dL_dsh[(size_t)g * 3 * M + k] = 0;
        if (radii[g] <= 0) continue;
        const real *p = means + 3 * g;
        cov2d_t cv;
        cov2d(p, cov6 + 6 * g, vm, focal_x, focal_y, tanfovx, tanfovy, &cv);
        real a = cv.a, b = cv.b, c = cv.c;
        real denom = a * c - b * b;
        real denom2inv = K(1) / (denom * denom + K(0.0000001));
        real gx_ = dL_dconic[3 * g], gy_ = dL_dconic[3 * g + 1], gz_ = dL_dconic[3 * g + 2];
        real dL_da = 0, dL_db = 0, dL_dc = 0;
        const real *m0 = cv.m[0], *m1 = cv.m[1];
        real *dc = dL_dcov6 + 6 * g;
        if (denom2inv != K(0)) {
            dL_da = denom2inv * (-c * c * gx_ + K(2) * b * c * gy_ + (denom - a * c) * gz_);
            dL_dc = denom2inv * (-a * a * gz_ + K(2) * a * b * gy_ + (denom - a * c) * gx_);
            dL_db = denom2inv * K(2) * (b * c * gx_ - (denom + K(2) * b * b) * gy_ + a * b * gz_);
            dc[0] = m0[0] * m0[0] * dL_da + m0[0] * m1[0] * dL_db + m1[0] * m1[0] * dL_dc;
            dc[3] = m0[1] * m0[1] * dL_da + m0[1] * m1[1] * dL_db + m1[1] * m1[1] * dL_dc;
            dc[5] = m0[2] * m0[2] * dL_da + m0[2] * m1[2] * dL_db + m1[2] * m1[2] * dL_dc;
            dc[1] = K(2) * m0[0] * m0[1] * dL_da + (m0[0] * m1[1] + m0[1] * m1[0]) * dL_db + K(2) * m1[0] * m1[1] * dL_dc;
            dc[2] = K(2) * m0[0] * m0[2] * dL_da + (m0[0] * m1[2] + m0[2] * m1[0]) * dL_db + K(2) * m1[0] * m1[2] * dL_dc;
            dc[4] = K(2) * m0[2] * m0[1] * dL_da + (m0[1] * m1[2] + m0[2] * m1[1]) * dL_db + K(2) * m1[1] * m1[2] * dL_dc;
        }
        const real *S = cov6 + 6 * g;
        real V[3][3] = {{S[0], S[1], S[2]}, {S[1], S[3], S[4]}, {S[2], S[4], S[5]}};
        /* dL/dM (2x3) */
        real dM0[3], dM1[3];
        for (int k = 0; k < 3; ++k) {
            real sm0 = m0[0] * V[k][0] + m0[1] * V[k][1] + m0[2] * V[k][2];
            real sm1 = m1[0] * V[k][0] + m1[1] * V[k][1] + m1[2] * V[k][2];
            dM0[k] = K(2) * sm0 * dL_da + sm1 * dL_db;
            dM1[k] = K(2) * sm1 * dL_dc + sm0 * dL_db;
        }
        /* M = J R  ->  dL/dJ = dL/dM R^T ;  R[i][j] = vm[4j+i] */
        real dJ00 = vm[0] * dM0[0] + vm[4] * dM0[1] + vm[8] * dM0[2];
        real dJ02 = vm[2] * dM0[0] + vm[6] * dM0[1] + vm[10] * dM0[2];
        real dJ11 = vm[1] * dM1[0] + vm[5] * dM1[1] + vm[9] * dM1[2];
        real dJ12 = vm[2] * dM1[0] + vm[6] * dM1[1] + vm[10] * dM1[2];
        real tz = K(1) / cv.tz, tz2 = tz * tz, tz3 = tz2 * tz;
        real xm = cv.clamp_x ? K(0) : K(1), ym = cv.clamp_y ? K(0) : K(1);
        real dL_dtx = xm * -focal_x * tz2 * dJ02;
        real dL_dty = ym * -focal_y * tz2 * dJ12;
        real dL_dtz = -focal_x * tz2 * dJ00 - focal_y * tz2 * dJ11 +
                      (K(2) * focal_x * cv.ctx) * tz3 * dJ02 + (K(2) * focal_y * cv.cty) * tz3 * dJ12;
        /* t = R p + trans  ->  dL/dp = R^T dL/dt */
        real dmx = vm[0] * dL_dtx + vm[1] * dL_dty + vm[2] * dL_dtz;
        real dmy = vm[4] * dL_dtx + vm[5] * dL_dty + vm[6] * dL_dtz;
        real dmz = vm[8] * dL_dtx + vm[9] * dL_dty + vm[10] * dL_dtz;
        /* screen-space mean gradient through the perspective divide */
        real hx = pm[0] * p[0] + pm[4] * p[1] + pm[8] * p[2] + pm[12];
        real hy = pm[1] * p[0] + pm[5] * p[1] + pm[9] * p[2] + pm[13];
        real hw = pm[3] * p[0] + pm[7] * p[1] + pm[11] * p[2] + pm[15];
        real m_w = K(1) / (hw + K(1e-7));
        real mul1 = hx * m_w * m_w, mul2 = hy * m_w * m_w;
        real d2x = dL_dmean2D[2 * g], d2y = dL_dmean2D[2 * g + 1];
        dmx += (pm[0] * m_w - pm[3] * mul1) * d2x + (pm[1] * m_w - pm[3] * mul2) * d2y;
        dmy += (pm[4] * m_w - pm[7] * mul1) * d2x + (pm[5] * m_w - pm[7] * mul2) * d2y;
        dmz += (pm[8] * m_w - pm[11] * mul1) * d2x + (pm[9] * m_w - pm[11] * mul2) * d2y;
        if (M > 0) {
            real ddx = p[0] - campos[0], ddy = p[1] - campos[1], ddz = p[2] - campos[2];
            real len2 = ddx * ddx + ddy * ddy + ddz * ddz;
            real len = R_SQRT(len2);
            real x = ddx / len, y = ddy / len, z = ddz / len;
            real basis[25], bx[25], by[25], bz[25];
            sh_basis(deg, x, y, z, basis);
            sh_basis_grad(deg, x, y, z, bx, by, bz);
            int nb = (deg + 1) * (deg + 1);
            const real *s = sh + (size_t)g * M * 3;
            real *ds = dL_dsh + (size_t)g * M * 3;
            real dLdx = 0, dLdy = 0, dLdz = 0;
            for (int ch = 0; ch < 3; ++ch) {
                real dl = clamped[3 * g + ch] ? K(0) : dL_dcolor[3 * g + ch];
                for (int k = 0; k < nb; ++k) {
                    ds[3 * k + ch] = basis[k] * dl;
                    dLdx += bx[k] * s[3 * k + ch] * dl;
                    dLdy += by[k] * s[3 * k + ch] * dl;
                    dLdz += bz[k] * s[3 * k + ch] * dl;
                }
            }
            /* through v/|v| */
            real inv3 = K(1) / (len2 * len);
            dmx += ((len2 - ddx * ddx) * dLdx - ddy * ddx * dLdy - ddz * ddx * dLdz) * inv3;
            dmy += (-ddx * ddy * dLdx + (len2 - ddy * ddy) * dLdy - ddz * ddy * dLdz) * inv3;
            dmz += (-ddx * ddz * dLdx - ddy * ddz * dLdy + (len2 - ddz * ddz) * dLdz) * inv3;
        }
        dL_dmeans[3 * g] = dmx;
        dL_dmeans[3 * g + 1] = dmy;
        dL_dmeans[3 * g + 2] = dmz;
    }
}
