// Experiment (not product): which explicit float operation order reproduces the torch operations of GaussianModel's densification
// bit for bit (scripts/exp_densify.py).  Build:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -shared -Xcompiler -fPIC scripts/exp_densify.cu -o scripts/_build/libexp_densify.so
#include <cuda_runtime.h>

// torch.norm(g[:, :2], dim=-1) of add_densification_stats
__global__ void k_norm2(const float* g, float* y, int n, int variant)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float a = g[3 * i], b = g[3 * i + 1];
    float s;
    if (variant == 0) s = __fmaf_rn(b, b, __fmul_rn(a, a));
    else if (variant == 1) s = __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b));
    else s = __fmaf_rn(a, a, __fmul_rn(b, b));
    y[i] = __fsqrt_rn(s);
}

// build_rotation (utils/general_utils.py), every eager torch operation rounded on its own
__global__ void k_rot(const float* r, float* R, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float r0 = r[4 * i], r1 = r[4 * i + 1], r2 = r[4 * i + 2], r3 = r[4 * i + 3];
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r0, r0), __fmul_rn(r1, r1)), __fmul_rn(r2, r2)), __fmul_rn(r3, r3)));
    const float w = __fdiv_rn(r0, nrm), x = __fdiv_rn(r1, nrm), y = __fdiv_rn(r2, nrm), z = __fdiv_rn(r3, nrm);
    float* o = R + 9 * i;
    o[0] = __fsub_rn(1.f, 2.f * __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z)));
    o[1] = 2.f * __fsub_rn(__fmul_rn(x, y), __fmul_rn(w, z));
    o[2] = 2.f * __fadd_rn(__fmul_rn(x, z), __fmul_rn(w, y));
    o[3] = 2.f * __fadd_rn(__fmul_rn(x, y), __fmul_rn(w, z));
    o[4] = __fsub_rn(1.f, 2.f * __fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z)));
    o[5] = 2.f * __fsub_rn(__fmul_rn(y, z), __fmul_rn(w, x));
    o[6] = 2.f * __fsub_rn(__fmul_rn(x, z), __fmul_rn(w, y));
    o[7] = 2.f * __fadd_rn(__fmul_rn(y, z), __fmul_rn(w, x));
    o[8] = __fsub_rn(1.f, 2.f * __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
}

__device__ float dot3(const float* m, const float* s, int variant)
{
    static const int perm[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
    const float p0 = __fmul_rn(m[0], s[0]), p1 = __fmul_rn(m[1], s[1]), p2 = __fmul_rn(m[2], s[2]);
    if (variant < 6) {
        const int a = perm[variant][0], b = perm[variant][1], c = perm[variant][2];
        return __fmaf_rn(m[c], s[c], __fmaf_rn(m[b], s[b], __fmul_rn(m[a], s[a])));
    }
    if (variant == 6) return __fadd_rn(__fadd_rn(p0, p1), p2);
    if (variant == 7) return __fadd_rn(p0, __fadd_rn(p1, p2));
    return __fadd_rn(__fadd_rn(p0, p2), p1);
}

// torch.bmm(R[n,3,3], s[n,3,1])
__global__ void k_bmm(const float* R, const float* s, float* y, int n, int variant)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int r = 0; r < 3; r++) y[3 * i + r] = dot3(R + 9 * i + 3 * r, s + 3 * i, variant);
}

// log(exp(s) / (0.8 * 2))
__global__ void k_child_scale(const float* s, float* y, int n, int variant)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float e = expf(s[i]);
    y[i] = logf(variant == 0 ? __fmul_rn(e, __fdiv_rn(1.0f, 1.6f)) : __fdiv_rn(e, 1.6f));
}

extern "C" {
static unsigned nb(int n) { return (unsigned)((n + 255) / 256); }
void run_norm2(const float* g, float* y, int n, int v) { k_norm2<<<nb(n), 256>>>(g, y, n, v); }
void run_rot(const float* r, float* R, int n) { k_rot<<<nb(n), 256>>>(r, R, n); }
void run_bmm(const float* R, const float* s, float* y, int n, int v) { k_bmm<<<nb(n), 256>>>(R, s, y, n, v); }
void run_child_scale(const float* s, float* y, int n, int v) { k_child_scale<<<nb(n), 256>>>(s, y, n, v); }
}
