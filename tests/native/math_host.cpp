// Host build of the PRODUCT's per-Gaussian math (lightgaussian_b200/csrc/lgr_math.cuh) so that the CPU test
// suite can compare it with the oracle without a GPU.  Test harness only -- not part of liblgrast.so.
// Build: g++ -O2 -ffp-contract=off -fno-fast-math -shared -fPIC math_host.cpp -o _build/libmath_host.so
#include <cstdint>
#include <cstring>
#include "../../lightgaussian_b200/csrc/lgr_math.cuh"

extern "C" {

void mh_preprocess(int P, int D, int M, const float* means3D, const float* scales, float mod, const float* rotations,
                   const float* opacities, const float* shs, const float* cov3D_precomp, const float* colors_precomp,
                   const float* view, const float* proj, const float* campos, int W, int H, float tanx, float tany, int32_t* radii,
                   float* means2D, float* depths, float* cov3D, float* rgb, float* conic_opacity, uint8_t* clamped,
                   uint32_t* tiles_touched)
{
    const float fy = H / (2.0f * tany), fx = W / (2.0f * tanx);
    const int gx = (W + 15) / 16, gy = (H + 15) / 16;
    for (int i = 0; i < P; i++) {
        radii[i] = 0; tiles_touched[i] = 0; depths[i] = 0; clamped[i] = 0;
        means2D[2 * i] = means2D[2 * i + 1] = 0;
        for (int k = 0; k < 4; k++) conic_opacity[4 * i + k] = 0;
        for (int k = 0; k < 3; k++) rgb[3 * i + k] = 0;
        for (int k = 0; k < 6; k++) cov3D[6 * i + k] = 0;
        const float x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
        if (!(lgr::xform_row(view, 2, x, y, z) > 0.2f)) continue;
        float cov[6];
        if (cov3D_precomp) memcpy(cov, cov3D_precomp + 6 * i, sizeof(cov));
        else {
            lgr::cov3d_from_scale_rot(scales[3 * i], scales[3 * i + 1], scales[3 * i + 2], mod, rotations[4 * i], rotations[4 * i + 1],
                                      rotations[4 * i + 2], rotations[4 * i + 3], cov);
            memcpy(cov3D + 6 * i, cov, sizeof(cov));
        }
        lgr::Geom g;
        if (!lgr::project_gaussian(x, y, z, view, proj, cov, fx, fy, tanx, tany, W, H, gx, gy, g)) continue;
        unsigned cb = 0;
        if (!colors_precomp) {
            const float* sh = shs + (size_t)i * M * 3;
            lgr::sh_to_rgb(D, [&](int k) { return sh[k]; }, x, y, z, campos, rgb + 3 * i, cb);
        }
        radii[i] = g.radius; depths[i] = g.depth;
        means2D[2 * i] = g.px; means2D[2 * i + 1] = g.py;
        conic_opacity[4 * i] = g.conic_x; conic_opacity[4 * i + 1] = g.conic_y; conic_opacity[4 * i + 2] = g.conic_z;
        conic_opacity[4 * i + 3] = opacities[i];
        clamped[i] = (uint8_t)cb;
        tiles_touched[i] = (uint32_t)((g.rect.y1 - g.rect.y0) * (g.rect.x1 - g.rect.x0));
    }
}

float mh_pair_power(float dx, float dy, float A, float B, float C) { return lgr::pair_power(dx, dy, A, B, C); }

// For each of n (Gaussian, pixel rectangle) pairs: the largest pinned pair_power over the pixel centres x0..x1, y0..y1 (inclusive) at
// which the reference blends at all (power <= 0), -inf when there is none.  The reference blends a pixel when o * exp(power) >= 1/255.
void mh_rect_max_power(int n, const float* px, const float* py, const float* A, const float* B, const float* C, const int32_t* x0,
                       const int32_t* x1, const int32_t* y0, const int32_t* y1, float* out)
{
    for (int i = 0; i < n; i++) {
        float best = -INFINITY;
        for (int y = y0[i]; y <= y1[i]; y++)
            for (int x = x0[i]; x <= x1[i]; x++) {
                const float p = lgr::pair_power(px[i] - (float)x, py[i] - (float)y, A[i], B[i], C[i]);
                if (p <= 0.0f && p > best) best = p;
            }
        out[i] = best;
    }
}

// The binning-time tile cull on the host, with the per-Gaussian set-up of tile_keep_mask (lgrast.cu): culled[i] = rect_culled over the
// pixel centres x0..x1, y0..y1, and the rect_qmin q and mag it compared.
void mh_rect_cull(int n, const float* px, const float* py, const float* A, const float* B, const float* C, const float* o, const int32_t* x0,
                  const int32_t* x1, const int32_t* y0, const int32_t* y1, uint8_t* culled, float* q, float* mag)
{
    for (int i = 0; i < n; i++) {
        const float thr = logf(257.55f * o[i]);
        const float hA = 0.5f * A[i], hC = 0.5f * C[i], nba = -B[i] / A[i], nbc = -B[i] / C[i];
        const float dx_lo = px[i] - (float)x1[i], dx_hi = px[i] - (float)x0[i], dy_lo = py[i] - (float)y1[i], dy_hi = py[i] - (float)y0[i];
        lgr::rect_qmin(hA, hC, B[i], nba, nbc, dx_lo, dx_hi, dy_lo, dy_hi, q[i], mag[i]);
        culled[i] = lgr::rect_culled(hA, hC, B[i], nba, nbc, thr, dx_lo, dx_hi, dy_lo, dy_hi) ? 1 : 0;
    }
}

// K7+K8 on the host: the same helper sequence preprocess_backward_kernel runs per Gaussian.
void mh_preprocess_backward(int P, int D, int M, const float* means3D, const int32_t* radii, const float* shs, const uint8_t* clamped,
                            const float* scales, const float* rotations, float mod, const float* cov3D, const float* view,
                            const float* proj, const float* campos, int W, int H, float tanx, float tany, const float* dL_dmean2D,
                            const float* dL_dconic, const float* dL_dcolor, float* dL_dmeans3D, float* dL_dcov3D, float* dL_dsh,
                            float* dL_dscale, float* dL_drot)
{
    const float fy = H / (2.0f * tany), fx = W / (2.0f * tanx);
    for (int i = 0; i < P; i++) {
        for (int k = 0; k < 3; k++) dL_dmeans3D[3 * i + k] = 0, dL_dscale[3 * i + k] = 0;
        for (int k = 0; k < 6; k++) dL_dcov3D[6 * i + k] = 0;
        for (int k = 0; k < 4; k++) dL_drot[4 * i + k] = 0;
        for (int k = 0; k < 3 * M; k++) dL_dsh[(size_t)i * 3 * M + k] = 0;
        if (!(radii[i] > 0)) continue;
        const float x = means3D[3 * i], y = means3D[3 * i + 1], z = means3D[3 * i + 2];
        float dcov[6], dmean[3];
        lgr::cov2d_backward(x, y, z, view, cov3D + 6 * i, fx, fy, tanx, tany, dL_dconic[3 * i], dL_dconic[3 * i + 1], dL_dconic[3 * i + 2],
                            dcov, dmean);
        lgr::mean2d_backward(x, y, z, proj, dL_dmean2D[2 * i], dL_dmean2D[2 * i + 1], dmean);
        for (int k = 0; k < 6; k++) dL_dcov3D[6 * i + k] = dcov[k];
        if (shs) {
            const unsigned cb = clamped[i];
            const float dRGB[3] = {(cb & 1u) ? 0.f : dL_dcolor[3 * i], (cb & 2u) ? 0.f : dL_dcolor[3 * i + 1], (cb & 4u) ? 0.f : dL_dcolor[3 * i + 2]};
            const float* sh = shs + (size_t)i * M * 3;
            float* out = dL_dsh + (size_t)i * M * 3;
            lgr::sh_backward(D, [&](int k) { return sh[k]; }, [&](int k, int c, float v) { out[3 * k + c] = v; }, x, y, z, campos, dRGB, dmean);
        }
        for (int k = 0; k < 3; k++) dL_dmeans3D[3 * i + k] = dmean[k];
        if (scales)
            lgr::cov3d_backward(scales[3 * i], scales[3 * i + 1], scales[3 * i + 2], mod, rotations[4 * i], rotations[4 * i + 1],
                                rotations[4 * i + 2], rotations[4 * i + 3], dcov, dL_dscale + 3 * i, dL_drot + 4 * i);
    }
}
}
