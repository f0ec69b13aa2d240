/* Float64 arbiter of the absolute-gradient densification statistic, for tests/test_absgrad_cpu.py and tests/test_gpu_absgrad.py.
 *
 * The blend backward of RAST/cuda_rasterizer/backward.cu:399-557 in float64, on a given forward state (ranges, point_list, means2D,
 * conic_opacity, colours, final_T, n_contrib), walking each pixel's list back to front exactly as oracle/lgo.c's blend_backward does,
 * but keeping, per pair, only the two terms the reference adds to dL/dmean2D (backward.cu:538-546):
 *     gx = dL_dG * dG_ddelx * 0.5W,   gy = dL_dG * dG_ddely * 0.5H
 * and summing their absolute values per Gaussian:  absgrad[2i] = sum_p |gx(p,i)|,  absgrad[2i+1] = sum_p |gy(p,i)|  (zeroed here).
 * A pair is blended when power <= 0 and alpha = min(0.99, o*exp(power)) >= 1/255 (the pair test of lgo.c, in double).
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -shared -fPIC absgrad_host.c -lm */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define TILE 16

void absgrad_blend_backward(int P, int W, int H, const uint32_t *ranges, const uint32_t *point_list, const double *means2D,
                            const double *conic_opacity, const double *colors, const double *bg, const double *final_T,
                            const uint32_t *n_contrib, const double *dL_dpix, double *absgrad)
{
    const int gx = (W + TILE - 1) / TILE;
    const double ddelx_dx = 0.5 * (double)W, ddely_dy = 0.5 * (double)H;
    for (int i = 0; i < 2 * P; i++) absgrad[i] = 0.0;
    for (int py = 0; py < H; py++)
        for (int px = 0; px < W; px++) {
            const int tile = (py / TILE) * gx + px / TILE;
            const uint32_t r0 = ranges[2 * tile];
            const size_t pix = (size_t)py * W + px;
            const double T_final = final_T[pix];
            double T = T_final;
            double dpix[3], accum[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, last_alpha = 0, bg_dot = 0;
            for (int c = 0; c < 3; c++) {
                dpix[c] = dL_dpix[(size_t)c * H * W + pix];
                bg_dot += bg[c] * dpix[c];
            }
            for (uint32_t k = n_contrib[pix]; k-- > 0;) {   /* list positions last-1 .. 0, back to front */
                const uint32_t g = point_list[r0 + k];
                const double *co = conic_opacity + 4 * g;
                const double dx = means2D[2 * g] - (double)px, dy = means2D[2 * g + 1] - (double)py;
                const double s = fma(dx, dx * co[0], dy * (dy * co[2]));
                const double power = fma(s, -0.5, -(dy * (dx * co[1])));
                if (power > 0) continue;
                const double G = exp(power);
                const double alpha = fmin(co[3] * G, (double)0.99f);
                if (alpha < (double)(1.0f / 255.0f)) continue;
                T = T / (1.0 - alpha);
                double dL_dalpha = 0;
                for (int c = 0; c < 3; c++) {
                    const double col = colors[3 * g + c];
                    accum[c] = last_alpha * last_color[c] + (1.0 - last_alpha) * accum[c];
                    last_color[c] = col;
                    dL_dalpha += (col - accum[c]) * dpix[c];
                }
                dL_dalpha *= T;
                last_alpha = alpha;
                dL_dalpha += (-T_final / (1.0 - alpha)) * bg_dot;
                const double dL_dG = co[3] * dL_dalpha;
                const double gdx = G * dx, gdy = G * dy;
                const double dG_ddelx = -gdx * co[0] - gdy * co[1];
                const double dG_ddely = -gdy * co[2] - gdx * co[1];
                absgrad[2 * g] += fabs(dL_dG * dG_ddelx * ddelx_dx);
                absgrad[2 * g + 1] += fabs(dL_dG * dG_ddely * ddely_dy);
            }
        }
}
