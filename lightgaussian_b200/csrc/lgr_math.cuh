// lgr_math.cuh -- per-Gaussian and per-(pixel, Gaussian) arithmetic of the rasterizer.
//
// Forward math is written with explicitly rounded operations (LGR_MUL/ADD/FMA/...) in exactly the
// operation order of the reference's compiled kernels (RAST/cuda_rasterizer/forward.cu:22-258,334-364
// as nvcc 12.9 emits them for sm_90a), because the forward pass is full of discrete decisions that a
// one-ulp difference can flip: the z<=0.2 cull, ceil() of the splat radius, int truncation of the tile
// rectangle, the depth sort key, and the alpha / transmittance thresholds of the blend.  With the
// order pinned, our forward output is bit-identical to the reference's on the same GPU.
// Backward math only has to meet 1e-3 relative, and is written for speed.
//
// The header is also compilable by a plain host C++ compiler (LGR_HOST_ONLY) so that the CPU test
// suite can check this exact code against the oracle without a GPU (tests/native/math_host.cpp).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define LGR_HD __device__ __forceinline__
#else
#define LGR_HD static inline
#endif

#if defined(__CUDA_ARCH__)
#define LGR_MUL(a, b) __fmul_rn((a), (b))
#define LGR_ADD(a, b) __fadd_rn((a), (b))
#define LGR_SUB(a, b) __fsub_rn((a), (b))
#define LGR_FMA(a, b, c) __fmaf_rn((a), (b), (c))
#define LGR_DIV(a, b) __fdiv_rn((a), (b))
#define LGR_RCP(a) __frcp_rn((a))
#define LGR_SQRT(a) __fsqrt_rn((a))
#define LGR_F2I_CEIL(a) __float2int_ru((a))
#define LGR_F2I_TRUNC(a) __float2int_rz((a))
#define LGR_I2F(a) __int2float_rn((a))
#else  // host build: compile with -ffp-contract=off so that * and + round once each
#define LGR_MUL(a, b) ((float)((float)(a) * (float)(b)))
#define LGR_ADD(a, b) ((float)((float)(a) + (float)(b)))
#define LGR_SUB(a, b) ((float)((float)(a) - (float)(b)))
#define LGR_FMA(a, b, c) fmaf((a), (b), (c))
#define LGR_DIV(a, b) ((float)((float)(a) / (float)(b)))
#define LGR_RCP(a) ((float)(1.0f / (float)(a)))
#define LGR_SQRT(a) sqrtf((a))
#define LGR_F2I_CEIL(a) ((int)ceilf((a)))
#define LGR_F2I_TRUNC(a) ((int)(a))
#define LGR_I2F(a) ((float)(a))
#endif

#define LGR_TILE 16  // RAST/cuda_rasterizer/config.h:16-17

namespace lgr {

// SH basis constants (RAST/cuda_rasterizer/auxiliary.h:22-39)
#define LGR_C0 0.28209479177387814f
#define LGR_C1 0.4886025119029199f
#define LGR_C2_0 1.0925484305920792f
#define LGR_C2_1 -1.0925484305920792f
#define LGR_C2_2 0.31539156525252005f
#define LGR_C2_3 -1.0925484305920792f
#define LGR_C2_4 0.5462742152960396f
#define LGR_C3_0 -0.5900435899266435f
#define LGR_C3_1 2.890611442640554f
#define LGR_C3_2 -0.4570457994644658f
#define LGR_C3_3 0.3731763325901154f
#define LGR_C3_4 -0.4570457994644658f
#define LGR_C3_5 1.445305721320277f
#define LGR_C3_6 -0.5900435899266435f

// out = m[k]*x + m[4+k]*y + m[8+k]*z + m[12+k] in the compiled order of transformPoint4x4/4x3
// (RAST/cuda_rasterizer/auxiliary.h:58-77).
LGR_HD float xform_row(const float* m, int k, float x, float y, float z)
{
    return LGR_ADD(LGR_FMA(z, m[8 + k], LGR_FMA(x, m[k], LGR_MUL(y, m[4 + k]))), m[12 + k]);
}

// a1*b1 plain, a0*b0 fused onto it, a2*b2 fused last: the shape every 3-term matrix product of the
// reference compiles to.
LGR_HD float dot3m(float a0, float b0, float a1, float b1, float a2, float b2)
{
    return LGR_FMA(a2, b2, LGR_FMA(a0, b0, LGR_MUL(a1, b1)));
}

// Sigma = R diag(mod*s)^2 R^T, upper triangle (RAST/cuda_rasterizer/forward.cu:120-154; the quaternion
// is used as given, not normalised).
LGR_HD void cov3d_from_scale_rot(float s0, float s1, float s2, float mod, float r, float x, float y, float z, float* cov)
{
    const float xz = LGR_MUL(x, z), rx = LGR_MUL(r, x), rz = LGR_MUL(r, z), yy = LGR_MUL(y, y), zz = LGR_MUL(z, z);
    const float xz_p_ry = LGR_FMA(r, y, xz), xz_m_ry = LGR_FMA(-r, y, xz);
    const float yz_m_rx = LGR_FMA(y, z, -rx), yz_p_rx = LGR_FMA(y, z, rx);
    const float xy_m_rz = LGR_FMA(x, y, -rz), xy_p_rz = LGR_FMA(x, y, rz);
    const float xx_yy = LGR_FMA(x, x, yy), yy_zz = LGR_ADD(yy, zz), xx_zz = LGR_FMA(x, x, zz);
    const float sx = LGR_MUL(s0, mod), sy = LGR_MUL(s1, mod), sz = LGR_MUL(s2, mod);
    // m[a][k] = (mod*s_k) * Rot[a][k]
    const float m00 = LGR_MUL(sx, LGR_SUB(1.0f, LGR_ADD(yy_zz, yy_zz)));
    const float m01 = LGR_MUL(sy, LGR_ADD(xy_m_rz, xy_m_rz));
    const float m02 = LGR_MUL(sz, LGR_ADD(xz_p_ry, xz_p_ry));
    const float m10 = LGR_MUL(sx, LGR_ADD(xy_p_rz, xy_p_rz));
    const float m11 = LGR_MUL(sy, LGR_SUB(1.0f, LGR_ADD(xx_zz, xx_zz)));
    const float m12 = LGR_MUL(sz, LGR_ADD(yz_m_rx, yz_m_rx));
    const float m20 = LGR_MUL(sx, LGR_ADD(xz_m_ry, xz_m_ry));
    const float m21 = LGR_MUL(sy, LGR_ADD(yz_p_rx, yz_p_rx));
    const float m22 = LGR_MUL(sz, LGR_SUB(1.0f, LGR_ADD(xx_yy, xx_yy)));
    cov[0] = dot3m(m00, m00, m01, m01, m02, m02);
    cov[1] = dot3m(m00, m10, m01, m11, m02, m12);
    cov[2] = dot3m(m00, m20, m01, m21, m02, m22);
    cov[3] = dot3m(m10, m10, m11, m11, m12, m12);
    cov[4] = dot3m(m10, m20, m11, m21, m12, m22);
    cov[5] = dot3m(m20, m20, m21, m21, m22, m22);
}

// EWA projection set-up shared by forward and backward (RAST/cuda_rasterizer/forward.cu:76-101).
struct Ewa {
    float tx, ty, tz;  // camera-space mean; x,y after the 1.3*tanfov clamp
    float txtz, tytz, limx, limy;
    float T00, T01, T02, T10, T11, T12;  // the two non-zero columns of W*J
};

LGR_HD void ewa_setup(float px, float py, float pz, const float* v, float fx, float fy, float tanx, float tany, Ewa& e)
{
    const float tx = xform_row(v, 0, px, py, pz);
    const float ty = xform_row(v, 1, px, py, pz);
    const float tz = xform_row(v, 2, px, py, pz);
    e.limx = LGR_MUL(tanx, 1.3f);
    e.limy = LGR_MUL(tany, 1.3f);
    e.txtz = LGR_DIV(tx, tz);
    e.tytz = LGR_DIV(ty, tz);
    const float cx = fminf(fmaxf(e.txtz, -e.limx), e.limx);
    const float cy = fminf(fmaxf(e.tytz, -e.limy), e.limy);
    e.tz = tz;
    e.tx = LGR_MUL(cx, tz);
    e.ty = LGR_MUL(cy, tz);
    const float tz2 = LGR_MUL(tz, tz);
    const float j00 = LGR_DIV(fx, tz);
    const float j02 = LGR_DIV(LGR_MUL(LGR_MUL(tz, -cx), fx), tz2);
    const float j11 = LGR_DIV(fy, tz);
    const float j12 = LGR_DIV(LGR_MUL(LGR_MUL(tz, -cy), fy), tz2);
    e.T00 = LGR_FMA(v[2], j02, LGR_FMA(v[0], j00, LGR_MUL(0.0f, v[1])));
    e.T01 = LGR_FMA(v[6], j02, LGR_FMA(v[4], j00, LGR_MUL(0.0f, v[5])));
    e.T02 = LGR_FMA(v[10], j02, LGR_FMA(v[8], j00, LGR_MUL(0.0f, v[9])));
    e.T10 = LGR_FMA(v[2], j12, LGR_FMA(0.0f, v[0], LGR_MUL(v[1], j11)));
    e.T11 = LGR_FMA(v[6], j12, LGR_FMA(0.0f, v[4], LGR_MUL(v[5], j11)));
    e.T12 = LGR_FMA(v[10], j12, LGR_FMA(0.0f, v[8], LGR_MUL(v[9], j11)));
}

// cov2D = T^T Vrk T (before the +0.3 low-pass), RAST/cuda_rasterizer/forward.cu:103-114
LGR_HD void cov2d_from_ewa(const Ewa& e, const float* c, float& a, float& b, float& cc)
{
    const float p00 = dot3m(e.T00, c[0], e.T01, c[1], e.T02, c[2]);
    const float p10 = dot3m(e.T00, c[1], e.T01, c[3], e.T02, c[4]);
    const float p20 = dot3m(e.T00, c[2], e.T01, c[4], e.T02, c[5]);
    const float p01 = dot3m(e.T10, c[0], e.T11, c[1], e.T12, c[2]);
    const float p11 = dot3m(e.T10, c[1], e.T11, c[3], e.T12, c[4]);
    const float p21 = dot3m(e.T10, c[2], e.T11, c[4], e.T12, c[5]);
    a = dot3m(e.T00, p00, e.T01, p10, e.T02, p20);
    b = dot3m(e.T00, p01, e.T01, p11, e.T02, p21);
    cc = dot3m(e.T10, p01, e.T11, p11, e.T12, p21);
}

// RAST/cuda_rasterizer/auxiliary.h:41-44 (double arithmetic, narrowed)
LGR_HD float ndc2pix(float v, int S)
{
#if defined(__CUDA_ARCH__)
    return __double2float_rn(__dmul_rn(__fma_rn(__dadd_rn((double)v, 1.0), (double)S, -1.0), 0.5));
#else
    return (float)(fma((double)v + 1.0, (double)S, -1.0) * 0.5);
#endif
}

struct TileRect {
    int x0, y0, x1, y1;
};

// RAST/cuda_rasterizer/auxiliary.h:46-56
LGR_HD TileRect tile_rect(float px, float py, int radius, int gx, int gy)
{
    const float rf = LGR_I2F(radius);
    TileRect r;
    int v;
    v = LGR_F2I_TRUNC(LGR_MUL(LGR_SUB(px, rf), 0.0625f));
    r.x0 = v < 0 ? 0 : (v > gx ? gx : v);
    v = LGR_F2I_TRUNC(LGR_MUL(LGR_SUB(py, rf), 0.0625f));
    r.y0 = v < 0 ? 0 : (v > gy ? gy : v);
    v = LGR_F2I_TRUNC(LGR_MUL(LGR_ADD(LGR_ADD(LGR_ADD(px, rf), 16.0f), -1.0f), 0.0625f));
    r.x1 = v < 0 ? 0 : (v > gx ? gx : v);
    v = LGR_F2I_TRUNC(LGR_MUL(LGR_ADD(LGR_ADD(LGR_ADD(py, rf), 16.0f), -1.0f), 0.0625f));
    r.y1 = v < 0 ? 0 : (v > gy ? gy : v);
    return r;
}

// Per-Gaussian forward geometry.  Returns false when the Gaussian is culled (nothing valid in `g`).
struct Geom {
    float depth;
    float px, py;
    float conic_x, conic_y, conic_z;
    int radius;
    TileRect rect;
};

LGR_HD bool project_gaussian(float x, float y, float z, const float* view, const float* proj, const float* cov3D, float fx,
                             float fy, float tanx, float tany, int W, int H, int gx, int gy, Geom& g)
{
    const float depth = xform_row(view, 2, x, y, z);
    if (depth <= 0.2f) return false;  // RAST/cuda_rasterizer/auxiliary.h:152
    const float hx = xform_row(proj, 0, x, y, z);
    const float hy = xform_row(proj, 1, x, y, z);
    const float hw = xform_row(proj, 3, x, y, z);
    const float pw = LGR_RCP(LGR_ADD(hw, 0.0000001f));
    const float ndc_x = LGR_MUL(hx, pw), ndc_y = LGR_MUL(hy, pw);
    Ewa e;
    ewa_setup(x, y, z, view, fx, fy, tanx, tany, e);
    float a, b, c;
    cov2d_from_ewa(e, cov3D, a, b, c);
    a = LGR_ADD(a, 0.3f);
    c = LGR_ADD(c, 0.3f);
    const float det = LGR_FMA(a, c, -LGR_MUL(b, b));
    if (det == 0.0f) return false;
    const float det_inv = LGR_RCP(det);
    g.conic_x = LGR_MUL(c, det_inv);
    g.conic_y = LGR_MUL(b, -det_inv);
    g.conic_z = LGR_MUL(a, det_inv);
    const float mid = LGR_MUL(LGR_ADD(a, c), 0.5f);
    const float sq = LGR_SQRT(fmaxf(LGR_FMA(mid, mid, -det), 0.1f));
    const float lam = fmaxf(LGR_ADD(mid, sq), LGR_SUB(mid, sq));
    g.radius = LGR_F2I_CEIL(LGR_MUL(LGR_SQRT(lam), 3.0f));
    g.px = ndc2pix(ndc_x, W);
    g.py = ndc2pix(ndc_y, H);
    g.rect = tile_rect(g.px, g.py, g.radius, gx, gy);
    if ((g.rect.x1 - g.rect.x0) * (g.rect.y1 - g.rect.y0) == 0) return false;
    g.depth = depth;
    return true;
}

// SH -> RGB (RAST/cuda_rasterizer/forward.cu:22-73).  sh points at this Gaussian's [M][3] floats with
// element stride `st` floats (1 for global memory; used as given for staged copies).
// clamp_bits: bit c set when channel c was clamped at 0.
template <typename ShLoad>
LGR_HD void sh_to_rgb(int deg, ShLoad sh, float px, float py, float pz, const float* cam, float* rgb, unsigned& clamp_bits)
{
    const float dx = LGR_SUB(px, cam[0]), dy = LGR_SUB(py, cam[1]), dz = LGR_SUB(pz, cam[2]);
    const float len = LGR_SQRT(LGR_FMA(dz, dz, LGR_FMA(dx, dx, LGR_MUL(dy, dy))));
    const float x = LGR_DIV(dx, len), y = LGR_DIV(dy, len), z = LGR_DIV(dz, len);
    float res[3];
#pragma unroll
    for (int c = 0; c < 3; c++) res[c] = LGR_MUL(sh(c), LGR_C0);
    if (deg > 0) {
        const float by = LGR_MUL(y, LGR_C1), bz = LGR_MUL(z, LGR_C1), bx = LGR_MUL(x, LGR_C1);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            res[c] = LGR_FMA(-by, sh(3 + c), res[c]);
            res[c] = LGR_FMA(bz, sh(6 + c), res[c]);
            res[c] = LGR_FMA(-bx, sh(9 + c), res[c]);
        }
        if (deg > 1) {
            const float xy = LGR_MUL(y, x), yz = LGR_MUL(z, y), xz = LGR_MUL(z, x);
            const float xx = LGR_MUL(x, x), yy = LGR_MUL(y, y), zz = LGR_MUL(z, z);
            const float zz2 = LGR_ADD(zz, zz);
            const float b4 = LGR_MUL(xy, LGR_C2_0), b5 = LGR_MUL(yz, LGR_C2_1);
            const float b6 = LGR_MUL(LGR_SUB(LGR_SUB(zz2, xx), yy), LGR_C2_2);
            const float b7 = LGR_MUL(xz, LGR_C2_3);
            const float xx_yy = LGR_SUB(xx, yy);
            const float b8 = LGR_MUL(xx_yy, LGR_C2_4);
#pragma unroll
            for (int c = 0; c < 3; c++) {
                res[c] = LGR_FMA(b4, sh(12 + c), res[c]);
                res[c] = LGR_FMA(b5, sh(15 + c), res[c]);
                res[c] = LGR_FMA(b6, sh(18 + c), res[c]);
                res[c] = LGR_FMA(b7, sh(21 + c), res[c]);
                res[c] = LGR_FMA(b8, sh(24 + c), res[c]);
            }
            if (deg > 2) {
                const float b9 = LGR_MUL(LGR_MUL(y, LGR_C3_0), LGR_FMA(xx, 3.0f, -yy));
                const float b10 = LGR_MUL(LGR_MUL(xy, LGR_C3_1), z);
                const float q4 = LGR_SUB(LGR_FMA(zz, 4.0f, -xx), yy);
                const float b11 = LGR_MUL(LGR_MUL(y, LGR_C3_2), q4);
                const float b12 = LGR_MUL(LGR_MUL(z, LGR_C3_3), LGR_FMA(yy, -3.0f, LGR_FMA(xx, -3.0f, zz2)));
                const float b13 = LGR_MUL(q4, LGR_MUL(x, LGR_C3_4));
                const float b14 = LGR_MUL(xx_yy, LGR_MUL(z, LGR_C3_5));
                const float b15 = LGR_MUL(LGR_MUL(x, LGR_C3_6), LGR_FMA(yy, -3.0f, xx));
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    res[c] = LGR_FMA(b9, sh(27 + c), res[c]);
                    res[c] = LGR_FMA(b10, sh(30 + c), res[c]);
                    res[c] = LGR_FMA(b11, sh(33 + c), res[c]);
                    res[c] = LGR_FMA(b12, sh(36 + c), res[c]);
                    res[c] = LGR_FMA(b13, sh(39 + c), res[c]);
                    res[c] = LGR_FMA(b14, sh(42 + c), res[c]);
                    res[c] = LGR_FMA(b15, sh(45 + c), res[c]);
                }
            }
        }
    }
    clamp_bits = 0;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const bool neg = res[c] < -0.5f;  // (res + 0.5f) < 0, as compiled
        const float v = LGR_ADD(res[c], 0.5f);
        rgb[c] = neg ? 0.0f : v;
        clamp_bits |= neg ? (1u << c) : 0u;
    }
}

// (pixel, Gaussian) exponent in the compiled order of RAST/cuda_rasterizer/forward.cu:334-337
LGR_HD float pair_power(float dx, float dy, float A, float B, float Cc)
{
    const float s = LGR_FMA(dx, LGR_MUL(dx, A), LGR_MUL(dy, LGR_MUL(dy, Cc)));
    return LGR_FMA(s, -0.5f, -LGR_MUL(dy, LGR_MUL(dx, B)));
}

// ------------------------------------------------------------------------------------------------
// Exact culling (DESIGN.md section 4): may a rectangle of pixel centres be skipped for a Gaussian?  The offsets dx = px - x and
// dy = py - y of its pixel centres span [dx_lo, dx_hi] x [dy_lo, dy_hi]; hA = A/2, hC = C/2 and B are the conic's, nba = -B/A,
// nbc = -B/C.  With the Gaussian's centre outside the rectangle, the smallest q = hA dx^2 + hC dy^2 + B dx dy over it lies on the edge
// nearest the centre in x or in y; rect_qmin evaluates both candidates (each edge's minimiser clamped to the rectangle) and returns the
// smaller q with mag, the size of the terms it cancelled.  Returns false when the centre lies inside (q = 0 there).  The operations are
// pinned: the API path's per-lane mask and the fused path's warp-cooperative mask inline this in different contexts, and must agree bit
// for bit.
// ------------------------------------------------------------------------------------------------
LGR_HD bool rect_qmin(float hA, float hC, float B, float nba, float nbc, float dx_lo, float dx_hi, float dy_lo, float dy_hi, float& q,
                      float& mag)
{
    const float cx = fminf(fmaxf(0.f, dx_lo), dx_hi), cy = fminf(fmaxf(0.f, dy_lo), dy_hi);
    q = 0.f;
    mag = 0.f;
    if (cx == 0.f && cy == 0.f) return false;
    q = 3.0e38f;
    if (cx != 0.f) {
        const float dy = fminf(fmaxf(LGR_MUL(nbc, cx), dy_lo), dy_hi);
        const float t0 = LGR_MUL(LGR_MUL(hA, cx), cx), t1 = LGR_MUL(LGR_MUL(hC, dy), dy), t2 = LGR_MUL(LGR_MUL(B, cx), dy);
        q = LGR_ADD(LGR_ADD(t0, t1), t2);
        mag = LGR_ADD(LGR_MUL(2.f, LGR_ADD(t0, t1)), fabsf(t2));
    }
    if (cy != 0.f) {
        const float dx = fminf(fmaxf(LGR_MUL(nba, cy), dx_lo), dx_hi);
        const float t0 = LGR_MUL(LGR_MUL(hA, dx), dx), t1 = LGR_MUL(LGR_MUL(hC, cy), cy), t2 = LGR_MUL(LGR_MUL(B, dx), cy);
        const float qy = LGR_ADD(LGR_ADD(t0, t1), t2);
        if (qy < q) {
            q = qy;
            mag = LGR_ADD(LGR_MUL(2.f, LGR_ADD(t0, t1)), fabsf(t2));
        }
    }
    return true;
}

// Relative rounding bound of rect_qmin's q and of the reference's own power at a pixel, in units of mag (A dx^2 + C dy^2 + |B dx dy|,
// the bound lgr_blend.cuh's subtile_cull2 uses).  The 1 % alpha margin in thr = ln(255 * 1.01 * opacity) covers the rounding of q only
// while its terms stay below ~1e4; a needle far from the rectangle cancels terms of 1e5-1e7 down to a small q.
#define LGR_CULL_REL 2.0e-6f

// true when no pixel centre of the rectangle can reach alpha >= 1/255 (the reference skips every such pair, forward.cu:345-347).
LGR_HD bool rect_culled(float hA, float hC, float B, float nba, float nbc, float thr, float dx_lo, float dx_hi, float dy_lo, float dy_hi)
{
    float q, mag;
    return rect_qmin(hA, hC, B, nba, nbc, dx_lo, dx_hi, dy_lo, dy_hi, q, mag) && q > LGR_FMA(LGR_CULL_REL, mag, thr);
}

// ------------------------------------------------------------------------------------------------
// Backward per-Gaussian math (RAST/cuda_rasterizer/backward.cu:144-396), free-form float.
// ------------------------------------------------------------------------------------------------
struct GradIn {
    float dconic_x, dconic_y, dconic_w;  // dL/d conic (x, y, w)
    float dmean2d_x, dmean2d_y;
};

// conic gradient -> dL/dcov3D[6] and the covariance part of dL/dmean3D.  cov3D = forward's 6 floats.
// dcam (optional, camera gradients): [0..2] = dL/dt, the camera-space mean gradient of the J path (clamp masks applied);
// [3 + 3r + k] = dL/dV[4r + k] for r, k < 3 through T = J W, i.e. (J^T dT)[k][r] with J at the clamped tx, ty.  When dcam is NULL
// the function is the leaf-only backward it always was.
LGR_HD void cov2d_backward(float px, float py, float pz, const float* v, const float* c3, float fx, float fy, float tanx,
                           float tany, float dA, float dB, float dC, float* dcov, float* dmean, float* dcam = nullptr)
{
    Ewa e;
    ewa_setup(px, py, pz, v, fx, fy, tanx, tany, e);
    float a, b, c;
    cov2d_from_ewa(e, c3, a, b, c);
    a += 0.3f;
    c += 0.3f;
    const float denom = a * c - b * b;
    const float denom2inv = 1.0f / (denom * denom + 0.0000001f);
    float da = 0.f, db = 0.f, dc = 0.f;
    if (denom2inv != 0.f) {
        da = denom2inv * (-c * c * dA + 2.f * b * c * dB + (denom - a * c) * dC);
        dc = denom2inv * (-a * a * dC + 2.f * a * b * dB + (denom - a * c) * dA);
        db = denom2inv * 2.f * (b * c * dA - (denom + 2.f * b * b) * dB + a * b * dC);
        dcov[0] = e.T00 * e.T00 * da + e.T00 * e.T10 * db + e.T10 * e.T10 * dc;
        dcov[3] = e.T01 * e.T01 * da + e.T01 * e.T11 * db + e.T11 * e.T11 * dc;
        dcov[5] = e.T02 * e.T02 * da + e.T02 * e.T12 * db + e.T12 * e.T12 * dc;
        dcov[1] = 2.f * e.T00 * e.T01 * da + (e.T00 * e.T11 + e.T01 * e.T10) * db + 2.f * e.T10 * e.T11 * dc;
        dcov[2] = 2.f * e.T00 * e.T02 * da + (e.T00 * e.T12 + e.T02 * e.T10) * db + 2.f * e.T10 * e.T12 * dc;
        dcov[4] = 2.f * e.T02 * e.T01 * da + (e.T01 * e.T12 + e.T02 * e.T11) * db + 2.f * e.T11 * e.T12 * dc;
    } else {
        for (int k = 0; k < 6; k++) dcov[k] = 0.f;
    }
    // V*T0, V*T1
    const float vt00 = e.T00 * c3[0] + e.T01 * c3[1] + e.T02 * c3[2];
    const float vt01 = e.T00 * c3[1] + e.T01 * c3[3] + e.T02 * c3[4];
    const float vt02 = e.T00 * c3[2] + e.T01 * c3[4] + e.T02 * c3[5];
    const float vt10 = e.T10 * c3[0] + e.T11 * c3[1] + e.T12 * c3[2];
    const float vt11 = e.T10 * c3[1] + e.T11 * c3[3] + e.T12 * c3[4];
    const float vt12 = e.T10 * c3[2] + e.T11 * c3[4] + e.T12 * c3[5];
    const float dT00 = 2.f * vt00 * da + vt10 * db, dT01 = 2.f * vt01 * da + vt11 * db, dT02 = 2.f * vt02 * da + vt12 * db;
    const float dT10 = 2.f * vt10 * dc + vt00 * db, dT11 = 2.f * vt11 * dc + vt01 * db, dT12 = 2.f * vt12 * dc + vt02 * db;
    const float dJ00 = v[0] * dT00 + v[4] * dT01 + v[8] * dT02;
    const float dJ02 = v[2] * dT00 + v[6] * dT01 + v[10] * dT02;
    const float dJ11 = v[1] * dT10 + v[5] * dT11 + v[9] * dT12;
    const float dJ12 = v[2] * dT10 + v[6] * dT11 + v[10] * dT12;
    const float xmul = (e.txtz < -e.limx || e.txtz > e.limx) ? 0.f : 1.f;
    const float ymul = (e.tytz < -e.limy || e.tytz > e.limy) ? 0.f : 1.f;
    const float iz = 1.f / e.tz, iz2 = iz * iz, iz3 = iz2 * iz;
    const float dtx = xmul * -fx * iz2 * dJ02;
    const float dty = ymul * -fy * iz2 * dJ12;
    const float dtz = -fx * iz2 * dJ00 - fy * iz2 * dJ11 + (2.f * fx * e.tx) * iz3 * dJ02 + (2.f * fy * e.ty) * iz3 * dJ12;
    dmean[0] = v[0] * dtx + v[1] * dty + v[2] * dtz;
    dmean[1] = v[4] * dtx + v[5] * dty + v[6] * dtz;
    dmean[2] = v[8] * dtx + v[9] * dty + v[10] * dtz;
    if (dcam) {
        // T[i][r] = sum_k J[i][k] V[4r + k] with J = [[j00, 0, j02], [0, j11, j12]] (ewa_setup)
        const float j00 = fx * iz, j02 = -fx * e.tx * iz2, j11 = fy * iz, j12 = -fy * e.ty * iz2;
        const float dT0[3] = {dT00, dT01, dT02}, dT1[3] = {dT10, dT11, dT12};
        dcam[0] = dtx; dcam[1] = dty; dcam[2] = dtz;
        for (int r = 0; r < 3; r++) {
            dcam[3 + 3 * r + 0] = j00 * dT0[r];
            dcam[3 + 3 * r + 1] = j11 * dT1[r];
            dcam[3 + 3 * r + 2] = j02 * dT0[r] + j12 * dT1[r];
        }
    }
}

// screen-space mean gradient -> 3D mean (RAST/cuda_rasterizer/backward.cu:370-387); accumulates into dmean.
// dh (optional, camera gradients): dL/dh for the homogeneous mean h = (h_x, h_y, h_w), ndc = (h_x, h_y) / (h_w + 1e-7).
LGR_HD void mean2d_backward(float px, float py, float pz, const float* proj, float g2x, float g2y, float* dmean, float* dh = nullptr)
{
    const float hw = proj[3] * px + proj[7] * py + proj[11] * pz + proj[15];
    const float mw = 1.0f / (hw + 0.0000001f);
    const float mul1 = (proj[0] * px + proj[4] * py + proj[8] * pz + proj[12]) * mw * mw;
    const float mul2 = (proj[1] * px + proj[5] * py + proj[9] * pz + proj[13]) * mw * mw;
    dmean[0] += (proj[0] * mw - proj[3] * mul1) * g2x + (proj[1] * mw - proj[3] * mul2) * g2y;
    dmean[1] += (proj[4] * mw - proj[7] * mul1) * g2x + (proj[5] * mw - proj[7] * mul2) * g2y;
    dmean[2] += (proj[8] * mw - proj[11] * mul1) * g2x + (proj[9] * mw - proj[11] * mul2) * g2y;
    if (dh) {
        const float hx = proj[0] * px + proj[4] * py + proj[8] * pz + proj[12];
        const float hy = proj[1] * px + proj[5] * py + proj[9] * pz + proj[13];
        dh[0] = g2x * mw;
        dh[1] = g2y * mw;
        dh[2] = -(g2x * hx + g2y * hy) * (mw * mw);
    }
}

// SH backward (RAST/cuda_rasterizer/backward.cu:20-139).  dRGB already masked by the clamp bits.
// Calls store(k, c, value) for every k < (deg+1)^2 and accumulates the view-direction term into dmean.
// ddir (optional, camera gradients): receives that view-direction term itself; dL/dcampos is its negative.
template <typename ShLoad, typename ShStore>
LGR_HD void sh_backward(int deg, ShLoad sh, ShStore store, float px, float py, float pz, const float* cam, const float* dRGB,
                        float* dmean, float* ddir = nullptr)
{
    const float ox = px - cam[0], oy = py - cam[1], oz = pz - cam[2];
    const float s2 = ox * ox + oy * oy + oz * oz;
    const float inv_len = 1.0f / sqrtf(s2);
    const float x = ox * inv_len, y = oy * inv_len, z = oz * inv_len;
    float ddx = 0.f, ddy = 0.f, ddz = 0.f;  // dL/d dir
#define LGR_SHB(k, basis, gx_, gy_, gz_)                                                                \
    {                                                                                                   \
        const float bb = (basis);                                                                       \
        const float w = sh(3 * (k)) * dRGB[0] + sh(3 * (k) + 1) * dRGB[1] + sh(3 * (k) + 2) * dRGB[2];   \
        store((k), 0, bb * dRGB[0]);                                                                    \
        store((k), 1, bb * dRGB[1]);                                                                    \
        store((k), 2, bb * dRGB[2]);                                                                    \
        ddx += (gx_) * w;                                                                               \
        ddy += (gy_) * w;                                                                               \
        ddz += (gz_) * w;                                                                               \
    }
    LGR_SHB(0, LGR_C0, 0.f, 0.f, 0.f)
    if (deg > 0) {
        LGR_SHB(1, -LGR_C1 * y, 0.f, -LGR_C1, 0.f)
        LGR_SHB(2, LGR_C1 * z, 0.f, 0.f, LGR_C1)
        LGR_SHB(3, -LGR_C1 * x, -LGR_C1, 0.f, 0.f)
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            LGR_SHB(4, LGR_C2_0 * xy, LGR_C2_0 * y, LGR_C2_0 * x, 0.f)
            LGR_SHB(5, LGR_C2_1 * yz, 0.f, LGR_C2_1 * z, LGR_C2_1 * y)
            LGR_SHB(6, LGR_C2_2 * (2.f * zz - xx - yy), LGR_C2_2 * -2.f * x, LGR_C2_2 * -2.f * y, LGR_C2_2 * 4.f * z)
            LGR_SHB(7, LGR_C2_3 * xz, LGR_C2_3 * z, 0.f, LGR_C2_3 * x)
            LGR_SHB(8, LGR_C2_4 * (xx - yy), LGR_C2_4 * 2.f * x, LGR_C2_4 * -2.f * y, 0.f)
            if (deg > 2) {
                LGR_SHB(9, LGR_C3_0 * y * (3.f * xx - yy), LGR_C3_0 * 6.f * xy, LGR_C3_0 * 3.f * (xx - yy), 0.f)
                LGR_SHB(10, LGR_C3_1 * xy * z, LGR_C3_1 * yz, LGR_C3_1 * xz, LGR_C3_1 * xy)
                LGR_SHB(11, LGR_C3_2 * y * (4.f * zz - xx - yy), LGR_C3_2 * -2.f * xy, LGR_C3_2 * (-3.f * yy + 4.f * zz - xx),
                        LGR_C3_2 * 8.f * yz)
                LGR_SHB(12, LGR_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy), LGR_C3_3 * -6.f * xz, LGR_C3_3 * -6.f * yz,
                        LGR_C3_3 * 3.f * (2.f * zz - xx - yy))
                LGR_SHB(13, LGR_C3_4 * x * (4.f * zz - xx - yy), LGR_C3_4 * (-3.f * xx + 4.f * zz - yy), LGR_C3_4 * -2.f * xy,
                        LGR_C3_4 * 8.f * xz)
                LGR_SHB(14, LGR_C3_5 * z * (xx - yy), LGR_C3_5 * 2.f * xz, LGR_C3_5 * -2.f * yz, LGR_C3_5 * (xx - yy))
                LGR_SHB(15, LGR_C3_6 * x * (xx - 3.f * yy), LGR_C3_6 * 3.f * (xx - yy), LGR_C3_6 * -6.f * xy, 0.f)
            }
        }
    }
#undef LGR_SHB
    // through dir = o/|o| (RAST/cuda_rasterizer/auxiliary.h:107-117)
    const float inv32 = inv_len * inv_len * inv_len;
    dmean[0] += ((s2 - ox * ox) * ddx - oy * ox * ddy - oz * ox * ddz) * inv32;
    dmean[1] += (-ox * oy * ddx + (s2 - oy * oy) * ddy - oz * oy * ddz) * inv32;
    dmean[2] += (-ox * oz * ddx - oy * oz * ddy + (s2 - oz * oz) * ddz) * inv32;
    if (ddir) {   // explicitly rounded products: a second use of the contractable ones above would keep them out of dmean's FMAs
        ddir[0] = LGR_MUL((s2 - ox * ox) * ddx - oy * ox * ddy - oz * ox * ddz, inv32);
        ddir[1] = LGR_MUL(-ox * oy * ddx + (s2 - oy * oy) * ddy - oz * oy * ddz, inv32);
        ddir[2] = LGR_MUL(-ox * oz * ddx - oy * oz * ddy + (s2 - oz * oz) * ddz, inv32);
    }
}

// dL/dSigma (6, doubled off-diagonals) -> dL/d(mod*scale) and dL/dquaternion
// (RAST/cuda_rasterizer/backward.cu:278-341).  Sigma = Rm diag(s)^2 Rm^T.
LGR_HD void cov3d_backward(float s0, float s1, float s2_, float mod, float r, float x, float y, float z, const float* dcov,
                           float* dscale, float* dq)
{
    const float Rm[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                            {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                            {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
    const float s[3] = {mod * s0, mod * s1, mod * s2_};
    const float dS[3][3] = {{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]},
                            {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]},
                            {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}};
    float dRm[3][3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        float dN[3];
#pragma unroll
        for (int a = 0; a < 3; a++) dN[a] = 2.f * s[k] * (Rm[0][k] * dS[0][a] + Rm[1][k] * dS[1][a] + Rm[2][k] * dS[2][a]);
        dscale[k] = Rm[0][k] * dN[0] + Rm[1][k] * dN[1] + Rm[2][k] * dN[2];
#pragma unroll
        for (int a = 0; a < 3; a++) dRm[a][k] = s[k] * dN[a];
    }
    dq[0] = 2.f * z * (dRm[1][0] - dRm[0][1]) + 2.f * y * (dRm[0][2] - dRm[2][0]) + 2.f * x * (dRm[2][1] - dRm[1][2]);
    dq[1] = 2.f * y * (dRm[0][1] + dRm[1][0]) + 2.f * z * (dRm[0][2] + dRm[2][0]) + 2.f * r * (dRm[2][1] - dRm[1][2]) -
            4.f * x * (dRm[2][2] + dRm[1][1]);
    dq[2] = 2.f * x * (dRm[0][1] + dRm[1][0]) + 2.f * r * (dRm[0][2] - dRm[2][0]) + 2.f * z * (dRm[2][1] + dRm[1][2]) -
            4.f * y * (dRm[2][2] + dRm[0][0]);
    dq[3] = 2.f * r * (dRm[1][0] - dRm[0][1]) + 2.f * x * (dRm[0][2] + dRm[2][0]) + 2.f * y * (dRm[2][1] + dRm[1][2]) -
            4.f * z * (dRm[1][1] + dRm[0][0]);
}

// torch.norm(g[:, :2], dim=-1) of one row, as torch evaluates it: sqrt(a*a + b*b), each operation rounded on its own.  The densification
// statistics (lgr_densify.cuh) and the norm the sparse exchange publishes per row (lgr_sparse.cuh) share this one definition.
LGR_HD float den_norm2(float a, float b) { return LGR_SQRT(LGR_ADD(LGR_MUL(a, a), LGR_MUL(b, b))); }

}  // namespace lgr
