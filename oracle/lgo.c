/*
 * lgo.c -- CPU ORACLE for the LightGaussian rasterizer hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is a plain-C restatement of the algorithm
 * implemented by the reference's CUDA rasterizer
 * (submodules/compress-diff-gaussian-rasterization, abbreviated RAST/ below).  It is
 * used only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg as the
 * checker; nothing in the product path (lightgaussian_b200/) may import or link it.
 *
 * Parity pin: the reference ships no tests or golden vectors for this path
 * (SURVEY.md section 4).  The oracle is pinned instead by
 *   (1) tests/golden/ref_*.npz -- outputs of the reference's own CUDA kernels, compiled
 *       unmodified from the reference checkout by oracle/Makefile into oracle/_ref and
 *       executed on the GPU (generator: tests/golden/make_ref_golden.py);
 *   (2) tests/golden/pyref_*.npz -- outputs of the reference's Python sub-steps
 *       (utils/sh_utils.py eval_sh) imported on CPU (generator: make_pyref_golden.py);
 *   (3) a finite-difference check of the backward pass against the double-precision
 *       build of this same file (-DLGO_DOUBLE).
 *
 * Arithmetic order.  The forward functions reproduce the reference's *compiled*
 * float operation order (which multiply-adds are fused) as read from the SASS that
 * nvcc 12.9 emits for RAST/cuda_rasterizer/forward.cu on sm_90a, so that every
 * discrete decision (near-plane cull, radius ceil, tile rectangle truncation, depth
 * sort key) matches the GPU bit for bit.  sqrt, division and reciprocal are IEEE
 * correctly rounded on both sides.  The one exception is exp(): the GPU uses
 * libdevice expf built on the MUFU.EX2 hardware approximation, which cannot be
 * reproduced on a CPU; glibc expf is used and pixels whose alpha / transmittance
 * tests sit within rounding distance of their thresholds are reported in `fragile`.
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -shared -fPIC lgo.c -lm
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef LGO_DOUBLE
typedef double real;
#define R_FMA fma
#define R_SQRT sqrt
#define R_EXP exp
#define R_CEIL ceil
#define R_FABS fabs
#define LGO_NAME(x) lgo_d_##x
#else
typedef float real;
#define R_FMA fmaf
#define R_SQRT sqrtf
#define R_EXP expf
#define R_CEIL ceilf
#define R_FABS fabsf
#define LGO_NAME(x) lgo_##x
#endif

#define TILE 16 /* RAST/cuda_rasterizer/config.h:16-17 BLOCK_X = BLOCK_Y = 16 */

/* SH basis constants, RAST/cuda_rasterizer/auxiliary.h:22-39 */
static const real C0 = (real)0.28209479177387814;
static const real C1 = (real)0.4886025119029199;
static const real C2[5] = {(real)1.0925484305920792, (real)-1.0925484305920792, (real)0.31539156525252005,
                           (real)-1.0925484305920792, (real)0.5462742152960396};
static const real C3[7] = {(real)-0.5900435899266435, (real)2.890611442640554, (real)-0.4570457994644658,
                           (real)0.3731763325901154, (real)-0.4570457994644658, (real)1.445305721320277,
                           (real)-0.5900435899266435};

static inline real rmin(real a, real b) { return a < b ? a : b; }
static inline real rmax(real a, real b) { return a > b ? a : b; }

/* One row of the (transposed-storage) 4x4 transform, RAST/cuda_rasterizer/auxiliary.h:58-77.
 * Compiled order: ((y*m[4+k]) fused with x*m[k]) fused with z*m[8+k], then + m[12+k]. */
static inline real xform_row(const real *m, int k, real x, real y, real z)
{
    return R_FMA(z, m[8 + k], R_FMA(x, m[k], y * m[4 + k])) + m[12 + k];
}

/* three-term product sum in the order the reference's matrix products compile to:
 * a1*b1 is the plain multiply, a0*b0 is fused onto it, a2*b2 is fused last. */
static inline real dot3_m(real a0, real b0, real a1, real b1, real a2, real b2)
{
    return R_FMA(a2, b2, R_FMA(a0, b0, a1 * b1));
}

/* world-space covariance from scale and (un-normalised) quaternion.
 * RAST/cuda_rasterizer/forward.cu:120-154. */
static void cov3d_from_scale_rot(const real *s, real mod, const real *q, real *cov)
{
    const real r = q[0], x = q[1], y = q[2], z = q[3];
    const real xz = x * z, rx = r * x, rz = r * z, yy = y * y, zz = z * z;
    const real xz_p_ry = R_FMA(r, y, xz), xz_m_ry = R_FMA(-r, y, xz);
    const real yz_m_rx = R_FMA(y, z, -rx), yz_p_rx = R_FMA(y, z, rx);
    const real xy_m_rz = R_FMA(x, y, -rz), xy_p_rz = R_FMA(x, y, rz);
    const real xx_yy = R_FMA(x, x, yy), yy_zz = yy + zz, xx_zz = R_FMA(x, x, zz);
    /* rot[a][b]: row a of the usual rotation matrix */
    real rot[3][3];
    rot[0][0] = (real)1 - (yy_zz + yy_zz);
    rot[0][1] = xy_m_rz + xy_m_rz;
    rot[0][2] = xz_p_ry + xz_p_ry;
    rot[1][0] = xy_p_rz + xy_p_rz;
    rot[1][1] = (real)1 - (xx_zz + xx_zz);
    rot[1][2] = yz_m_rx + yz_m_rx;
    rot[2][0] = xz_m_ry + xz_m_ry;
    rot[2][1] = yz_p_rx + yz_p_rx;
    rot[2][2] = (real)1 - (xx_yy + xx_yy);
    const real sc[3] = {s[0] * mod, s[1] * mod, s[2] * mod};
    real m[3][3]; /* m[a][k] = sc[k] * rot[a][k] */
    for (int a = 0; a < 3; a++)
        for (int k = 0; k < 3; k++) m[a][k] = sc[k] * rot[a][k];
    int o = 0;
    for (int a = 0; a < 3; a++)
        for (int b = a; b < 3; b++) cov[o++] = dot3_m(m[a][0], m[b][0], m[a][1], m[b][1], m[a][2], m[b][2]);
}

/* Everything computeCov2D needs from the camera-space position, shared by forward and backward. */
typedef struct {
    real tx, ty, tz;       /* t after the fov clamp (x,y rescaled by z) */
    real txtz, tytz;       /* unclamped ratios */
    real limx, limy;
    real j00, j02, j11, j12;
    real T0[3], T1[3];     /* the two non-zero columns of W*J (see forward.cu:91-101) */
} ewa_t;

static void ewa_setup(const real *p, const real *view, real fx, real fy, real tanx, real tany, ewa_t *e)
{
    const real tx = xform_row(view, 0, p[0], p[1], p[2]);
    const real ty = xform_row(view, 1, p[0], p[1], p[2]);
    const real tz = xform_row(view, 2, p[0], p[1], p[2]);
    e->limx = (real)1.3f * tanx;
    e->limy = (real)1.3f * tany;
    e->txtz = tx / tz;
    e->tytz = ty / tz;
    const real cx = rmin(e->limx, rmax(-e->limx, e->txtz));
    const real cy = rmin(e->limy, rmax(-e->limy, e->tytz));
    e->tz = tz;
    e->tx = cx * tz;
    e->ty = cy * tz;
    const real tz2 = tz * tz;
    e->j00 = fx / tz;
    e->j02 = ((tz * -cx) * fx) / tz2;
    e->j11 = fy / tz;
    e->j12 = ((tz * -cy) * fy) / tz2;
    /* T = W * J; W = rotation part of the view matrix. */
    e->T0[0] = R_FMA(view[2], e->j02, R_FMA(view[0], e->j00, (real)0 * view[1]));
    e->T0[1] = R_FMA(view[6], e->j02, R_FMA(view[4], e->j00, (real)0 * view[5]));
    e->T0[2] = R_FMA(view[10], e->j02, R_FMA(view[8], e->j00, (real)0 * view[9]));
    e->T1[0] = R_FMA(view[2], e->j12, R_FMA((real)0, view[0], view[1] * e->j11));
    e->T1[1] = R_FMA(view[6], e->j12, R_FMA((real)0, view[4], view[5] * e->j11));
    e->T1[2] = R_FMA(view[10], e->j12, R_FMA((real)0, view[8], view[9] * e->j11));
}

/* screen-space covariance (before the +0.3 low-pass): RAST/cuda_rasterizer/forward.cu:76-115 */
static void cov2d_from_ewa(const ewa_t *e, const real *c, real *a, real *b, real *cc)
{
    const real *T0 = e->T0, *T1 = e->T1;
    /* P = T^T * Vrk ; Vrk = [[c0,c1,c2],[c1,c3,c4],[c2,c4,c5]] */
    const real p00 = dot3_m(T0[0], c[0], T0[1], c[1], T0[2], c[2]);
    const real p10 = dot3_m(T0[0], c[1], T0[1], c[3], T0[2], c[4]);
    const real p20 = dot3_m(T0[0], c[2], T0[1], c[4], T0[2], c[5]);
    const real p01 = dot3_m(T1[0], c[0], T1[1], c[1], T1[2], c[2]);
    const real p11 = dot3_m(T1[0], c[1], T1[1], c[3], T1[2], c[4]);
    const real p21 = dot3_m(T1[0], c[2], T1[1], c[4], T1[2], c[5]);
    *a = dot3_m(T0[0], p00, T0[1], p10, T0[2], p20);
    *b = dot3_m(T0[0], p01, T0[1], p11, T0[2], p21);
    *cc = dot3_m(T1[0], p01, T1[1], p11, T1[2], p21);
}

/* RAST/cuda_rasterizer/auxiliary.h:41-44: evaluated in double, narrowed to float. */
static inline real ndc2pix(real v, int S)
{
    return (real)(fma((double)v + 1.0, (double)S, -1.0) * 0.5);
}

/* RAST/cuda_rasterizer/auxiliary.h:46-56 */
static void tile_rect(real px, real py, int radius, int gx, int gy, int *x0, int *y0, int *x1, int *y1)
{
    const real rf = (real)radius;
    int v;
    v = (int)((px - rf) * (real)0.0625f);
    *x0 = v < 0 ? 0 : (v > gx ? gx : v);
    v = (int)((py - rf) * (real)0.0625f);
    *y0 = v < 0 ? 0 : (v > gy ? gy : v);
    v = (int)((((px + rf) + (real)TILE) - (real)1) * (real)0.0625f);
    *x1 = v < 0 ? 0 : (v > gx ? gx : v);
    v = (int)((((py + rf) + (real)TILE) - (real)1) * (real)0.0625f);
    *y1 = v < 0 ? 0 : (v > gy ? gy : v);
}

/* SH -> RGB for one Gaussian: RAST/cuda_rasterizer/forward.cu:22-73 */
static void sh_to_rgb(int deg, const real *sh /* [M][3] */, const real *pos, const real *cam, real *rgb, uint8_t *clamped)
{
    const real dx = pos[0] - cam[0], dy = pos[1] - cam[1], dz = pos[2] - cam[2];
    const real len = R_SQRT(R_FMA(dz, dz, R_FMA(dx, dx, dy * dy)));
    const real x = dx / len, y = dy / len, z = dz / len;
    real res[3];
    for (int c = 0; c < 3; c++) res[c] = sh[c] * C0;
    if (deg > 0) {
        const real by = y * C1, bz = z * C1, bx = x * C1;
        for (int c = 0; c < 3; c++) {
            res[c] = R_FMA(-by, sh[3 + c], res[c]);
            res[c] = R_FMA(bz, sh[6 + c], res[c]);
            res[c] = R_FMA(-bx, sh[9 + c], res[c]);
        }
        if (deg > 1) {
            const real xy = y * x, yz = z * y, xz = z * x, xx = x * x, yy = y * y, zz = z * z;
            const real zz2 = zz + zz;
            const real b4 = xy * C2[0], b5 = yz * C2[1];
            const real b6 = ((zz2 - xx) - yy) * C2[2];
            const real b7 = xz * C2[3];
            const real xx_yy = xx - yy;
            const real b8 = xx_yy * C2[4];
            for (int c = 0; c < 3; c++) {
                res[c] = R_FMA(b4, sh[12 + c], res[c]);
                res[c] = R_FMA(b5, sh[15 + c], res[c]);
                res[c] = R_FMA(b6, sh[18 + c], res[c]);
                res[c] = R_FMA(b7, sh[21 + c], res[c]);
                res[c] = R_FMA(b8, sh[24 + c], res[c]);
            }
            if (deg > 2) {
                const real b9 = (y * C3[0]) * R_FMA(xx, (real)3, -yy);
                const real b10 = (xy * C3[1]) * z;
                const real q4 = R_FMA(zz, (real)4, -xx) - yy; /* 4zz - xx - yy */
                const real b11 = (y * C3[2]) * q4;
                const real b12 = (z * C3[3]) * R_FMA(yy, (real)-3, R_FMA(xx, (real)-3, zz2));
                const real b13 = q4 * (x * C3[4]);
                const real b14 = xx_yy * (z * C3[5]);
                const real b15 = (x * C3[6]) * R_FMA(yy, (real)-3, xx);
                for (int c = 0; c < 3; c++) {
                    res[c] = R_FMA(b9, sh[27 + c], res[c]);
                    res[c] = R_FMA(b10, sh[30 + c], res[c]);
                    res[c] = R_FMA(b11, sh[33 + c], res[c]);
                    res[c] = R_FMA(b12, sh[36 + c], res[c]);
                    res[c] = R_FMA(b13, sh[39 + c], res[c]);
                    res[c] = R_FMA(b14, sh[42 + c], res[c]);
                    res[c] = R_FMA(b15, sh[45 + c], res[c]);
                }
            }
        }
    }
    for (int c = 0; c < 3; c++) {
        const real v = res[c] + (real)0.5;
        clamped[c] = (v < (real)0);
        rgb[c] = v < (real)0 ? (real)0 : v;
    }
}

/* ------------------------------------------------------------------------------------------
 * preprocess: RAST/cuda_rasterizer/forward.cu:158-258 (+ rasterizer_impl.cu:223-224 for focal).
 * Outputs are zero-initialised here (the reference leaves culled rows uninitialised).
 * ------------------------------------------------------------------------------------------ */
void LGO_NAME(preprocess)(int P, int D, int M, const real *means3D, const real *scales, real scale_modifier,
                          const real *rotations, const real *opacities, const real *shs, const real *cov3D_precomp,
                          const real *colors_precomp, const real *view, const real *proj, const real *campos, int W, int H,
                          real tan_fovx, real tan_fovy, int32_t *radii, real *means2D, real *depths, real *cov3D, real *rgb,
                          real *conic_opacity, uint8_t *clamped, uint32_t *tiles_touched)
{
    const real fy = (real)H / ((real)2 * tan_fovy);
    const real fx = (real)W / ((real)2 * tan_fovx);
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    memset(radii, 0, sizeof(int32_t) * P);
    memset(means2D, 0, sizeof(real) * 2 * P);
    memset(depths, 0, sizeof(real) * P);
    memset(cov3D, 0, sizeof(real) * 6 * P);
    memset(rgb, 0, sizeof(real) * 3 * P);
    memset(conic_opacity, 0, sizeof(real) * 4 * P);
    memset(clamped, 0, 3 * (size_t)P);
    memset(tiles_touched, 0, sizeof(uint32_t) * P);
    for (int i = 0; i < P; i++) {
        const real *p = means3D + 3 * i;
        /* near-plane cull only (auxiliary.h:139-164) */
        const real depth = xform_row(view, 2, p[0], p[1], p[2]);
        if (depth <= (real)0.2f) continue;
        const real hx = xform_row(proj, 0, p[0], p[1], p[2]);
        const real hy = xform_row(proj, 1, p[0], p[1], p[2]);
        const real hw = xform_row(proj, 3, p[0], p[1], p[2]);
        const real pw = (real)1 / (hw + (real)0.0000001f);
        const real ndc_x = hx * pw, ndc_y = hy * pw;

        const real *c3;
        if (cov3D_precomp) {
            c3 = cov3D_precomp + 6 * i;
        } else {
            cov3d_from_scale_rot(scales + 3 * i, scale_modifier, rotations + 4 * i, cov3D + 6 * i);
            c3 = cov3D + 6 * i;
        }
        ewa_t e;
        ewa_setup(p, view, fx, fy, tan_fovx, tan_fovy, &e);
        real a, b, c;
        cov2d_from_ewa(&e, c3, &a, &b, &c);
        a = a + (real)0.3f;
        c = c + (real)0.3f;
        const real det = R_FMA(a, c, -(b * b));
        if (det == (real)0) continue;
        const real det_inv = (real)1 / det;
        const real conic_x = c * det_inv, conic_y = b * -det_inv, conic_z = a * det_inv;
        const real mid = (a + c) * (real)0.5;
        const real sq = R_SQRT(rmax(R_FMA(mid, mid, -det), (real)0.1f));
        const real lam = rmax(mid + sq, mid - sq);
        const int radius = (int)R_CEIL(R_SQRT(lam) * (real)3);
        const real px = ndc2pix(ndc_x, W), py = ndc2pix(ndc_y, H);
        int x0, y0, x1, y1;
        tile_rect(px, py, radius, gx, gy, &x0, &y0, &x1, &y1);
        if ((x1 - x0) * (y1 - y0) == 0) continue;

        if (!colors_precomp) sh_to_rgb(D, shs + (size_t)i * M * 3, p, campos, rgb + 3 * i, clamped + 3 * i);
        depths[i] = depth;
        radii[i] = radius;
        means2D[2 * i] = px;
        means2D[2 * i + 1] = py;
        conic_opacity[4 * i] = conic_x;
        conic_opacity[4 * i + 1] = conic_y;
        conic_opacity[4 * i + 2] = conic_z;
        conic_opacity[4 * i + 3] = opacities[i];
        tiles_touched[i] = (uint32_t)((y1 - y0) * (x1 - x0));
    }
}

/* RAST/cuda_rasterizer/rasterizer_impl.cu:54-66 (markVisible) */
void LGO_NAME(mark_visible)(int P, const real *means3D, const real *view, const real *proj, uint8_t *present)
{
    (void)proj;
    for (int i = 0; i < P; i++) {
        const real *p = means3D + 3 * i;
        present[i] = xform_row(view, 2, p[0], p[1], p[2]) > (real)0.2f;
    }
}

/* ------------------------------------------------------------------------------------------
 * binning: RAST/cuda_rasterizer/rasterizer_impl.cu:70-138,278-319.
 * key = (tile << 32) | float_bits(depth); stable sort; ties keep ascending Gaussian id.
 * point_list must hold sum(tiles_touched) entries; ranges holds 2*tiles entries (start,end).
 * Returns the number of instances written.
 * ------------------------------------------------------------------------------------------ */
int64_t LGO_NAME(bin)(int P, const real *means2D, const real *depths, const int32_t *radii, int W, int H,
                      uint32_t *point_list, uint32_t *ranges)
{
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    int64_t R = 0;
    for (int i = 0; i < P; i++) {
        if (radii[i] <= 0) continue;
        int x0, y0, x1, y1;
        tile_rect(means2D[2 * i], means2D[2 * i + 1], radii[i], gx, gy, &x0, &y0, &x1, &y1);
        R += (int64_t)(x1 - x0) * (y1 - y0);
    }
    uint64_t *keys = (uint64_t *)malloc(sizeof(uint64_t) * (R ? R : 1));
    uint64_t *keys2 = (uint64_t *)malloc(sizeof(uint64_t) * (R ? R : 1));
    uint32_t *vals = (uint32_t *)malloc(sizeof(uint32_t) * (R ? R : 1));
    uint32_t *vals2 = (uint32_t *)malloc(sizeof(uint32_t) * (R ? R : 1));
    int64_t off = 0;
    for (int i = 0; i < P; i++) {
        if (radii[i] <= 0) continue;
        int x0, y0, x1, y1;
        tile_rect(means2D[2 * i], means2D[2 * i + 1], radii[i], gx, gy, &x0, &y0, &x1, &y1);
        float df = (float)depths[i]; /* the key always carries the float32 bit pattern */
        uint32_t dbits;
        memcpy(&dbits, &df, 4);
        for (int y = y0; y < y1; y++)
            for (int x = x0; x < x1; x++) {
                keys[off] = ((uint64_t)(uint32_t)(y * gx + x) << 32) | dbits;
                vals[off] = (uint32_t)i;
                off++;
            }
    }
    /* stable LSD radix sort, 8 passes of 8 bits */
    for (int pass = 0; pass < 8; pass++) {
        int64_t hist[257];
        memset(hist, 0, sizeof(hist));
        const int sh = pass * 8;
        for (int64_t k = 0; k < R; k++) hist[((keys[k] >> sh) & 0xff) + 1]++;
        for (int k = 0; k < 256; k++) hist[k + 1] += hist[k];
        for (int64_t k = 0; k < R; k++) {
            int64_t d = hist[(keys[k] >> sh) & 0xff]++;
            keys2[d] = keys[k];
            vals2[d] = vals[k];
        }
        uint64_t *tk = keys; keys = keys2; keys2 = tk;
        uint32_t *tv = vals; vals = vals2; vals2 = tv;
    }
    memset(ranges, 0, sizeof(uint32_t) * 2 * (size_t)gx * gy);
    for (int64_t k = 0; k < R; k++) {
        point_list[k] = vals[k];
        uint32_t t = (uint32_t)(keys[k] >> 32);
        if (k == 0 || (uint32_t)(keys[k - 1] >> 32) != t) ranges[2 * t] = (uint32_t)k;
        if (k == R - 1 || (uint32_t)(keys[k + 1] >> 32) != t) ranges[2 * t + 1] = (uint32_t)(k + 1);
    }
    free(keys); free(keys2); free(vals); free(vals2);
    return R;
}

/* per-(pixel, Gaussian) blending weight, shared by forward and backward.
 * RAST/cuda_rasterizer/forward.cu:334-347 in its compiled operation order. */
static inline int pair_alpha(real gx_, real gy_, real px, real py, const real *co, real *d_x, real *d_y, real *G, real *alpha,
                             real *power_out)
{
    const real dx = gx_ - px, dy = gy_ - py;
    const real s = R_FMA(dx, dx * co[0], dy * (dy * co[2]));
    const real power = R_FMA(s, (real)-0.5, -(dy * (dx * co[1])));
    *d_x = dx; *d_y = dy; *power_out = power;
    if (power > (real)0) return 0;
    const real g = R_EXP(power);
    const real a = rmin(co[3] * g, (real)0.99f);
    *G = g; *alpha = a;
    if (a < (real)(1.0f / 255.0f)) return 0;
    return 1;
}

/* ------------------------------------------------------------------------------------------
 * forward blend: RAST/cuda_rasterizer/forward.cu:263-376; significance: forward.cu:455-474
 * with the *intended* (race-free) semantics count[g] += 1 per contributing (pixel, g) pair.
 * count (int64[P]) may be NULL; it is accumulated into, not cleared.
 * fragile (uint8[H*W]) may be NULL; set to 1 where a threshold test is within rounding noise.
 * ------------------------------------------------------------------------------------------ */
void LGO_NAME(blend_forward)(int W, int H, const uint32_t *ranges, const uint32_t *point_list, const real *means2D,
                             const real *colors, const real *conic_opacity, const real *bg, real *out_color, real *final_T,
                             uint32_t *n_contrib, int64_t *count, uint8_t *fragile)
{
    const int gx = (W + TILE - 1) / TILE;
    for (int py = 0; py < H; py++)
        for (int px = 0; px < W; px++) {
            const int tile = (py / TILE) * gx + px / TILE;
            const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
            real T = (real)1, C[3] = {0, 0, 0};
            uint32_t contributor = 0, last = 0;
            uint8_t frag = 0;
            for (uint32_t k = r0; k < r1; k++) {
                const uint32_t g = point_list[k];
                contributor++;
                real dx, dy, G = 0, alpha = 0, power;
                const int ok = pair_alpha(means2D[2 * g], means2D[2 * g + 1], (real)px, (real)py, conic_opacity + 4 * g, &dx, &dy, &G,
                                          &alpha, &power);
                if (fragile) {
                    if (R_FABS(power) < (real)1e-6) frag = 1;
                    if (power <= 0 && R_FABS(alpha * (real)255 - (real)1) < (real)2e-5) frag = 1;
                }
                if (!ok) continue;
                const real test_T = T * ((real)1 - alpha);
                if (fragile && R_FABS(test_T - (real)0.0001f) < (real)1e-8) frag = 1;
                if (test_T < (real)0.0001f) break; /* pixel done; this Gaussian is not blended */
                for (int c = 0; c < 3; c++) C[c] = R_FMA(T, alpha * colors[3 * g + c], C[c]);
                if (count) count[g] += 1;
                T = test_T;
                last = contributor;
            }
            const size_t pix = (size_t)py * W + px;
            final_T[pix] = T;
            n_contrib[pix] = last;
            for (int c = 0; c < 3; c++) out_color[(size_t)c * H * W + pix] = R_FMA(bg[c], T, C[c]);
            if (fragile) fragile[pix] = frag;
        }
}

/* ------------------------------------------------------------------------------------------
 * backward blend: RAST/cuda_rasterizer/backward.cu:399-557.  Per-Gaussian sums are accumulated
 * in double (the reference uses float atomics in nondeterministic order).
 * Outputs (zeroed here): dL_dmean2D[P*2] (x,y), dL_dconic[P*3] (.x,.y,.w), dL_dopacity[P], dL_dcolor[P*3].
 * ------------------------------------------------------------------------------------------ */
void LGO_NAME(blend_backward)(int P, int W, int H, const uint32_t *ranges, const uint32_t *point_list, const real *means2D,
                              const real *conic_opacity, const real *colors, const real *bg, const real *final_T,
                              const uint32_t *n_contrib, const real *dL_dpix, real *dL_dmean2D, real *dL_dconic,
                              real *dL_dopacity, real *dL_dcolor)
{
    const int gx = (W + TILE - 1) / TILE;
    double *acc = (double *)calloc((size_t)P * 9, sizeof(double));
    const real ddelx_dx = (real)0.5 * (real)W, ddely_dy = (real)0.5 * (real)H;
    for (int py = 0; py < H; py++)
        for (int px = 0; px < W; px++) {
            const int tile = (py / TILE) * gx + px / TILE;
            const uint32_t r0 = ranges[2 * tile];
            const size_t pix = (size_t)py * W + px;
            const real T_final = final_T[pix];
            real T = T_final;
            const uint32_t last = n_contrib[pix];
            real dpix[3], accum[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_alpha = 0;
            for (int c = 0; c < 3; c++) dpix[c] = dL_dpix[(size_t)c * H * W + pix];
            real bg_dot = 0;
            for (int c = 0; c < 3; c++) bg_dot += bg[c] * dpix[c];
            for (uint32_t k = last; k-- > 0;) { /* list positions last-1 .. 0, back to front */
                const uint32_t g = point_list[r0 + k];
                const real *co = conic_opacity + 4 * g;
                real dx, dy, G = 0, alpha = 0, power;
                if (!pair_alpha(means2D[2 * g], means2D[2 * g + 1], (real)px, (real)py, co, &dx, &dy, &G, &alpha, &power)) continue;
                T = T / ((real)1 - alpha);
                const real w = alpha * T;
                real dL_dalpha = 0;
                for (int c = 0; c < 3; c++) {
                    const real col = colors[3 * g + c];
                    accum[c] = last_alpha * last_color[c] + ((real)1 - last_alpha) * accum[c];
                    last_color[c] = col;
                    dL_dalpha += (col - accum[c]) * dpix[c];
                    acc[(size_t)g * 9 + c] += (double)(w * dpix[c]);
                }
                dL_dalpha *= T;
                last_alpha = alpha;
                dL_dalpha += (-T_final / ((real)1 - alpha)) * bg_dot;
                const real dL_dG = co[3] * dL_dalpha;
                const real gdx = G * dx, gdy = G * dy;
                const real dG_ddelx = -gdx * co[0] - gdy * co[1];
                const real dG_ddely = -gdy * co[2] - gdx * co[1];
                acc[(size_t)g * 9 + 3] += (double)(dL_dG * dG_ddelx * ddelx_dx);
                acc[(size_t)g * 9 + 4] += (double)(dL_dG * dG_ddely * ddely_dy);
                acc[(size_t)g * 9 + 5] += (double)((real)-0.5 * gdx * dx * dL_dG);
                acc[(size_t)g * 9 + 6] += (double)((real)-0.5 * gdx * dy * dL_dG);
                acc[(size_t)g * 9 + 7] += (double)((real)-0.5 * gdy * dy * dL_dG);
                acc[(size_t)g * 9 + 8] += (double)(G * dL_dalpha);
            }
        }
    for (int i = 0; i < P; i++) {
        const double *a = acc + (size_t)i * 9;
        for (int c = 0; c < 3; c++) dL_dcolor[3 * i + c] = (real)a[c];
        dL_dmean2D[2 * i] = (real)a[3];
        dL_dmean2D[2 * i + 1] = (real)a[4];
        dL_dconic[3 * i] = (real)a[5];
        dL_dconic[3 * i + 1] = (real)a[6];
        dL_dconic[3 * i + 2] = (real)a[7];
        dL_dopacity[i] = (real)a[8];
    }
    free(acc);
}

/* ------------------------------------------------------------------------------------------
 * preprocess backward: RAST/cuda_rasterizer/backward.cu:144-396 (computeCov2DCUDA + preprocessCUDA
 * + computeColorFromSH + computeCov3D), written in ordinary row/column matrix notation.
 * All outputs are zeroed here; only Gaussians with radii > 0 receive gradients.
 * cov3D is the array used by the forward (computed, or the caller's precomputed one).
 * shs / scales / rotations may be NULL (then dL_dsh / dL_dscale+dL_drot stay zero).
 * ------------------------------------------------------------------------------------------ */
void LGO_NAME(preprocess_backward)(int P, int D, int M, const real *means3D, const int32_t *radii, const real *shs,
                                   const uint8_t *clamped, const real *scales, const real *rotations, real scale_modifier,
                                   const real *cov3D, const real *view, const real *proj, const real *campos, int W, int H,
                                   real tan_fovx, real tan_fovy, const real *dL_dmean2D, const real *dL_dconic,
                                   const real *dL_dcolor, real *dL_dmeans3D, real *dL_dcov3D, real *dL_dsh, real *dL_dscale,
                                   real *dL_drot)
{
    const real fy = (real)H / ((real)2 * tan_fovy);
    const real fx = (real)W / ((real)2 * tan_fovx);
    memset(dL_dmeans3D, 0, sizeof(real) * 3 * P);
    memset(dL_dcov3D, 0, sizeof(real) * 6 * P);
    if (M > 0) memset(dL_dsh, 0, sizeof(real) * 3 * (size_t)M * P);
    memset(dL_dscale, 0, sizeof(real) * 3 * P);
    memset(dL_drot, 0, sizeof(real) * 4 * P);
    for (int i = 0; i < P; i++) {
        if (!(radii[i] > 0)) continue;
        const real *p = means3D + 3 * i;
        const real *c3 = cov3D + 6 * i;
        /* ---- conic -> cov2D -> cov3D and mean (backward.cu:144-274) ---- */
        ewa_t e;
        ewa_setup(p, view, fx, fy, tan_fovx, tan_fovy, &e);
        real a, b, c;
        cov2d_from_ewa(&e, c3, &a, &b, &c);
        a += (real)0.3f;
        c += (real)0.3f;
        const real dA = dL_dconic[3 * i], dB = dL_dconic[3 * i + 1], dC = dL_dconic[3 * i + 2];
        const real denom = a * c - b * b;
        const real denom2inv = (real)1 / (denom * denom + (real)0.0000001f);
        real da = 0, db = 0, dc = 0;
        real *dcov = dL_dcov3D + 6 * i;
        const real *T0 = e.T0, *T1 = e.T1;
        if (denom2inv != 0) {
            da = denom2inv * (-c * c * dA + 2 * b * c * dB + (denom - a * c) * dC);
            dc = denom2inv * (-a * a * dC + 2 * a * b * dB + (denom - a * c) * dA);
            db = denom2inv * 2 * (b * c * dA - (denom + 2 * b * b) * dB + a * b * dC);
            dcov[0] = T0[0] * T0[0] * da + T0[0] * T1[0] * db + T1[0] * T1[0] * dc;
            dcov[3] = T0[1] * T0[1] * da + T0[1] * T1[1] * db + T1[1] * T1[1] * dc;
            dcov[5] = T0[2] * T0[2] * da + T0[2] * T1[2] * db + T1[2] * T1[2] * dc;
            dcov[1] = 2 * T0[0] * T0[1] * da + (T0[0] * T1[1] + T0[1] * T1[0]) * db + 2 * T1[0] * T1[1] * dc;
            dcov[2] = 2 * T0[0] * T0[2] * da + (T0[0] * T1[2] + T0[2] * T1[0]) * db + 2 * T1[0] * T1[2] * dc;
            dcov[4] = 2 * T0[2] * T0[1] * da + (T0[1] * T1[2] + T0[2] * T1[1]) * db + 2 * T1[1] * T1[2] * dc;
        }
        /* V*T0 and V*T1 (V symmetric) */
        const real V[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
        real vt0[3], vt1[3];
        for (int k = 0; k < 3; k++) {
            vt0[k] = T0[0] * V[k][0] + T0[1] * V[k][1] + T0[2] * V[k][2];
            vt1[k] = T1[0] * V[k][0] + T1[1] * V[k][1] + T1[2] * V[k][2];
        }
        real dT0[3], dT1[3];
        for (int k = 0; k < 3; k++) {
            dT0[k] = 2 * vt0[k] * da + vt1[k] * db;
            dT1[k] = 2 * vt1[k] * dc + vt0[k] * db;
        }
        /* T = W*J with W rows (view[0],view[4],view[8]), (view[1],view[5],view[9]), (view[2],view[6],view[10]) */
        const real dJ00 = view[0] * dT0[0] + view[4] * dT0[1] + view[8] * dT0[2];
        const real dJ02 = view[2] * dT0[0] + view[6] * dT0[1] + view[10] * dT0[2];
        const real dJ11 = view[1] * dT1[0] + view[5] * dT1[1] + view[9] * dT1[2];
        const real dJ12 = view[2] * dT1[0] + view[6] * dT1[1] + view[10] * dT1[2];
        const real xmul = (e.txtz < -e.limx || e.txtz > e.limx) ? (real)0 : (real)1;
        const real ymul = (e.tytz < -e.limy || e.tytz > e.limy) ? (real)0 : (real)1;
        const real iz = (real)1 / e.tz, iz2 = iz * iz, iz3 = iz2 * iz;
        const real dtx = xmul * -fx * iz2 * dJ02;
        const real dty = ymul * -fy * iz2 * dJ12;
        const real dtz = -fx * iz2 * dJ00 - fy * iz2 * dJ11 + (2 * fx * e.tx) * iz3 * dJ02 + (2 * fy * e.ty) * iz3 * dJ12;
        real dmean[3];
        dmean[0] = view[0] * dtx + view[1] * dty + view[2] * dtz;
        dmean[1] = view[4] * dtx + view[5] * dty + view[6] * dtz;
        dmean[2] = view[8] * dtx + view[9] * dty + view[10] * dtz;
        /* ---- projected mean -> 3D mean (backward.cu:370-387) ---- */
        const real hw = proj[3] * p[0] + proj[7] * p[1] + proj[11] * p[2] + proj[15];
        const real mw = (real)1 / (hw + (real)0.0000001f);
        const real mul1 = (proj[0] * p[0] + proj[4] * p[1] + proj[8] * p[2] + proj[12]) * mw * mw;
        const real mul2 = (proj[1] * p[0] + proj[5] * p[1] + proj[9] * p[2] + proj[13]) * mw * mw;
        const real g2x = dL_dmean2D[2 * i], g2y = dL_dmean2D[2 * i + 1];
        dmean[0] += (proj[0] * mw - proj[3] * mul1) * g2x + (proj[1] * mw - proj[3] * mul2) * g2y;
        dmean[1] += (proj[4] * mw - proj[7] * mul1) * g2x + (proj[5] * mw - proj[7] * mul2) * g2y;
        dmean[2] += (proj[8] * mw - proj[11] * mul1) * g2x + (proj[9] * mw - proj[11] * mul2) * g2y;
        /* ---- colour -> SH and view direction (backward.cu:20-139) ---- */
        if (shs) {
            const real *sh = shs + (size_t)i * M * 3;
            real *dsh = dL_dsh + (size_t)i * M * 3;
            const real ox = p[0] - campos[0], oy = p[1] - campos[1], oz = p[2] - campos[2];
            const real len = R_SQRT(ox * ox + oy * oy + oz * oz);
            const real x = ox / len, y = oy / len, z = oz / len;
            real dRGB[3];
            for (int ch = 0; ch < 3; ch++) dRGB[ch] = clamped[3 * i + ch] ? (real)0 : dL_dcolor[3 * i + ch];
            real basis[16];
            real dbx[16], dby[16], dbz[16]; /* d basis_k / d(x,y,z) */
            memset(dbx, 0, sizeof(dbx)); memset(dby, 0, sizeof(dby)); memset(dbz, 0, sizeof(dbz));
            int nb = 1;
            basis[0] = C0;
            if (D > 0) {
                nb = 4;
                basis[1] = -C1 * y; dby[1] = -C1;
                basis[2] = C1 * z;  dbz[2] = C1;
                basis[3] = -C1 * x; dbx[3] = -C1;
                if (D > 1) {
                    nb = 9;
                    const real xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    basis[4] = C2[0] * xy;                    dbx[4] = C2[0] * y;  dby[4] = C2[0] * x;
                    basis[5] = C2[1] * yz;                    dby[5] = C2[1] * z;  dbz[5] = C2[1] * y;
                    basis[6] = C2[2] * (2 * zz - xx - yy);    dbx[6] = C2[2] * 2 * -x; dby[6] = C2[2] * 2 * -y; dbz[6] = C2[2] * 2 * 2 * z;
                    basis[7] = C2[3] * xz;                    dbx[7] = C2[3] * z;  dbz[7] = C2[3] * x;
                    basis[8] = C2[4] * (xx - yy);             dbx[8] = C2[4] * 2 * x; dby[8] = C2[4] * 2 * -y;
                    if (D > 2) {
                        nb = 16;
                        basis[9] = C3[0] * y * (3 * xx - yy);
                        basis[10] = C3[1] * xy * z;
                        basis[11] = C3[2] * y * (4 * zz - xx - yy);
                        basis[12] = C3[3] * z * (2 * zz - 3 * xx - 3 * yy);
                        basis[13] = C3[4] * x * (4 * zz - xx - yy);
                        basis[14] = C3[5] * z * (xx - yy);
                        basis[15] = C3[6] * x * (xx - 3 * yy);
                        dbx[9] = C3[0] * 3 * 2 * xy;            dby[9] = C3[0] * 3 * (xx - yy);
                        dbx[10] = C3[1] * yz;                   dby[10] = C3[1] * xz;                     dbz[10] = C3[1] * xy;
                        dbx[11] = C3[2] * -2 * xy;              dby[11] = C3[2] * (-3 * yy + 4 * zz - xx); dbz[11] = C3[2] * 4 * 2 * yz;
                        dbx[12] = C3[3] * -3 * 2 * xz;          dby[12] = C3[3] * -3 * 2 * yz;            dbz[12] = C3[3] * 3 * (2 * zz - xx - yy);
                        dbx[13] = C3[4] * (-3 * xx + 4 * zz - yy); dby[13] = C3[4] * -2 * xy;            dbz[13] = C3[4] * 4 * 2 * xz;
                        dbx[14] = C3[5] * 2 * xz;               dby[14] = C3[5] * -2 * yz;                dbz[14] = C3[5] * (xx - yy);
                        dbx[15] = C3[6] * 3 * (xx - yy);        dby[15] = C3[6] * -3 * 2 * xy;
                    }
                }
            }
            real ddir[3] = {0, 0, 0};
            for (int k = 0; k < nb; k++)
                for (int ch = 0; ch < 3; ch++) {
                    dsh[3 * k + ch] = basis[k] * dRGB[ch];
                    ddir[0] += dbx[k] * sh[3 * k + ch] * dRGB[ch];
                    ddir[1] += dby[k] * sh[3 * k + ch] * dRGB[ch];
                    ddir[2] += dbz[k] * sh[3 * k + ch] * dRGB[ch];
                }
            /* through dir = o/|o|  (auxiliary.h:107-117) */
            const real s2 = ox * ox + oy * oy + oz * oz;
            const real inv32 = (real)1 / R_SQRT(s2 * s2 * s2);
            dmean[0] += ((s2 - ox * ox) * ddir[0] - oy * ox * ddir[1] - oz * ox * ddir[2]) * inv32;
            dmean[1] += (-ox * oy * ddir[0] + (s2 - oy * oy) * ddir[1] - oz * oy * ddir[2]) * inv32;
            dmean[2] += (-ox * oz * ddir[0] - oy * oz * ddir[1] + (s2 - oz * oz) * ddir[2]) * inv32;
        }
        for (int k = 0; k < 3; k++) dL_dmeans3D[3 * i + k] = dmean[k];
        /* ---- cov3D -> scale, quaternion (backward.cu:278-341); Sigma = Rm diag(s)^2 Rm^T ---- */
        if (scales) {
            const real *q = rotations + 4 * i;
            const real r = q[0], x = q[1], y = q[2], z = q[3];
            const real Rm[3][3] = {{1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)},
                                   {2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)},
                                   {2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)}};
            const real s[3] = {scale_modifier * scales[3 * i], scale_modifier * scales[3 * i + 1], scale_modifier * scales[3 * i + 2]};
            /* dL/dSigma as a symmetric matrix: off-diagonals carry half of the stored (doubled) gradient */
            const real dS[3][3] = {{dcov[0], (real)0.5 * dcov[1], (real)0.5 * dcov[2]},
                                   {(real)0.5 * dcov[1], dcov[3], (real)0.5 * dcov[4]},
                                   {(real)0.5 * dcov[2], (real)0.5 * dcov[4], dcov[5]}};
            /* N = diag(s) Rm^T  (N[k][a] = s_k Rm[a][k]);  Sigma = N^T N;  dL/dN = 2 N dS */
            real dN[3][3];
            for (int k = 0; k < 3; k++)
                for (int a2 = 0; a2 < 3; a2++) {
                    real v = 0;
                    for (int m2 = 0; m2 < 3; m2++) v += s[k] * Rm[m2][k] * dS[m2][a2];
                    dN[k][a2] = 2 * v;
                }
            real dRm[3][3];
            for (int k = 0; k < 3; k++) {
                real v = 0;
                for (int a2 = 0; a2 < 3; a2++) v += Rm[a2][k] * dN[k][a2];
                dL_dscale[3 * i + k] = v; /* derivative w.r.t. (mod * scale_k); see backward.cu:321-325 */
                for (int a2 = 0; a2 < 3; a2++) dRm[a2][k] = s[k] * dN[k][a2];
            }
            /* Rm(q) derivative, quaternion not normalised (backward.cu:332-340) */
            real *dq = dL_drot + 4 * i;
            dq[0] = 2 * z * (dRm[1][0] - dRm[0][1]) + 2 * y * (dRm[0][2] - dRm[2][0]) + 2 * x * (dRm[2][1] - dRm[1][2]);
            dq[1] = 2 * y * (dRm[0][1] + dRm[1][0]) + 2 * z * (dRm[0][2] + dRm[2][0]) + 2 * r * (dRm[2][1] - dRm[1][2]) -
                    4 * x * (dRm[2][2] + dRm[1][1]);
            dq[2] = 2 * x * (dRm[0][1] + dRm[1][0]) + 2 * r * (dRm[0][2] - dRm[2][0]) + 2 * z * (dRm[2][1] + dRm[1][2]) -
                    4 * y * (dRm[2][2] + dRm[0][0]);
            dq[3] = 2 * r * (dRm[1][0] - dRm[0][1]) + 2 * x * (dRm[0][2] + dRm[2][0]) + 2 * y * (dRm[2][1] + dRm[1][2]) -
                    4 * z * (dRm[1][1] + dRm[0][0]);
        }
    }
}

int LGO_NAME(sizeof_real)(void) { return (int)sizeof(real); }
