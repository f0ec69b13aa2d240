/*
 * knn_oracle.c -- CPU ORACLE for distCUDA2 of submodules/simple-knn (SK/ below).  TEST INFRASTRUCTURE ONLY: used by
 * tests/test_knn_oracle.py and tests/test_gpu_knn.py; nothing in lightgaussian_b200/ links it.
 *
 * Brute force, O(P^2) (meant for P up to ~20 000).  out[i] = ((b0 + b1) + b2) / 3 (SK/simple_knn.cu:182) where b0 <= b1 <= b2 are
 * the three smallest pair values over j != i (excluded by index, SK/simple_knn.cu:158,177), initialised to FLT_MAX (:154) and
 * replaced only by a strictly smaller value (updateKBest, :136-144).  The pair value is the order nvcc 12.9 compiles :134-135 to on
 * sm_90a (the SASS of boxMeanDist): d = candidate - query per axis, then fma(dz, dz, fma(dx, dx, dy * dy)).  Every step is monotone
 * in non-negative arguments, so a pair whose dy*dy or fma(dx, dx, dy*dy) already reaches b2 cannot enter and is skipped early.
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -shared -fPIC knn_oracle.c -lm   (oracle/knn_oracle.py does this)
 */
#include <float.h>
#include <math.h>

void lgo_knn_mean_dist3(int P, const float *pts, float *out)
{
    for (int i = 0; i < P; i++) {
        const float qx = pts[3 * i], qy = pts[3 * i + 1], qz = pts[3 * i + 2];
        float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
        for (int j = 0; j < P; j++) {
            if (j == i) continue;
            const float dx = pts[3 * j] - qx, dy = pts[3 * j + 1] - qy, dz = pts[3 * j + 2] - qz;
            const float s = dy * dy;
            if (!(s < b2)) continue;
            const float t = fmaf(dx, dx, s);
            if (!(t < b2)) continue;
            const float d = fmaf(dz, dz, t);
            if (d < b2) {
                if (d < b1) {
                    b2 = b1;
                    if (d < b0) { b1 = b0; b0 = d; } else { b1 = d; }
                } else {
                    b2 = d;
                }
            }
        }
        out[i] = ((b0 + b1) + b2) / 3.0f;
    }
}
