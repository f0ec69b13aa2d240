// lgr_optim.cuh -- optimizer side of the training loops (SURVEY.md section 8f, row N3):
//   * adamw_multi_kernel   torch.optim.AdamW(l, lr=0.0, eps=1e-15) over the six parameter groups of GaussianModel
//                          (scene/gaussian_model.py:184-217) as ONE launch: every tensor of every group is a row of a
//                          pointer table, a block handles one 4096-element chunk of one tensor.  28 B of HBM traffic per
//                          element (read p,g,m,v; write p,m,v) against ~80 B for the ~9 foreach passes torch launches per group.
//   * adamw_selective_kernel  the same update on the rows (Gaussians) whose gradient is not all zero only (opt-in SelectiveAdamW).
//   * compact_gather_kernel  the row compaction of GaussianModel._prune_optimizer / prune_points (:564-600): parameters and both
//                          Adam moments of all groups gathered through one source-row index in one launch (the reference does
//                          18 boolean-mask indexings, each with its own nonzero() and host synchronisation).
//
// Arithmetic of one element, op for op what torch's default (foreach) AdamW path evaluates in fp32 -- torch/optim/adam.py
// _multi_tensor_adam, weight decay decoupled, amsgrad off, with the scalars computed on the host in double precision and
// rounded to fp32 at the kernel boundary exactly as the foreach functors receive them:
//     p  = p * (1 - lr*wd)                          _foreach_mul_
//     m  = m + (1-beta1) * (g - m)                  _foreach_lerp_           (weight < 0.5 branch; one FMA)
//     v  = v * beta2                                _foreach_mul_
//     v  = v + (1-beta2) * (g*g)                    _foreach_addcmul_        (g*g rounded, then one FMA)
//     d  = sqrt(v) / sqrt(1-beta2^t) + eps          _foreach_sqrt, _foreach_div_, _foreach_add_   (IEEE sqrt and division)
//     p  = p + (-lr/(1-beta1^t)) * (m / d)          _foreach_addcdiv_        (IEEE division, then one FMA)
// Every operation is pinned with an _rn intrinsic so that ptxas cannot re-associate or fuse differently.
// Denormals are kept (no FTZ), as torch's kernels keep them.
#pragma once

#include <cstdint>

namespace {

constexpr int OPT_MAX_TENSORS = 8;
constexpr int OPT_CHUNK = 4096;      // elements per block: 256 threads x 4 x float4

struct AdamTable {
    float* p[OPT_MAX_TENSORS];
    const float* g[OPT_MAX_TENSORS];
    float* m[OPT_MAX_TENSORS];
    float* v[OPT_MAX_TENSORS];
    long long n[OPT_MAX_TENSORS];
    int row_elems[OPT_MAX_TENSORS];         // 0 = contiguous parameter; else elements per row of a row-strided parameter view
    int row_stride[OPT_MAX_TENSORS];        // its row stride in elements
    int chunk_start[OPT_MAX_TENSORS + 1];   // prefix sum of ceil(n / OPT_CHUNK)
    float decay[OPT_MAX_TENSORS];           // 1 - lr*wd
    float neg_step[OPT_MAX_TENSORS];        // -(lr / (1 - beta1^t))
    float bc2_sqrt[OPT_MAX_TENSORS];        // sqrt(1 - beta2^t)
    float w1, beta2, w2, eps;               // 1-beta1, beta2, 1-beta2, eps
    int count;
};

// IEEE-correct division / square root whose cost does not depend on the data.  __fdiv_rn / __fsqrt_rn fall into a ~100-instruction
// subroutine whenever ONE lane of the warp holds a zero, a denormal or an extreme exponent -- and real gradients are full of them
// (exact zeros for culled Gaussians, g*g underflowing for the faint ones): measured 1.35 ms per 3M-Gaussian step on rendered
// gradients against 0.73 ms on well-scaled data (routing those lanes through fp64 was worse still: 2.4 ms).  Instead every lane is
// given operands the fast path accepts, and the result is fixed up exactly:
//   * zero operand: substitute 1, select the exact result (0, or the signed zero of the numerator) afterwards;
//   * |x| < 2^-60 (denormals included): scale by 2^64 first -- exact -- and scale the result back by 2^-32 (root) or 2^-64 (quotient);
//     exact as long as the final result is a normal number, which holds for every root (>= 2^-74.5) and for every quotient
//     >= 2^-122.  Only quotients that may land in the subnormal range (|m| < 2^-122 d: a first moment that has decayed for
//     hundreds of steps) would round twice; those rare lanes take binary64 division, whose second rounding to binary32 is innocuous
//     (53 >= 2*24+2).
//   * infinities, NaNs and exponents above 2^60 are left to the intrinsic's own slow path (absent from sane training runs).
__device__ __forceinline__ float opt_sqrt(float v)   // v >= +0 (a sum of squares), or inf / NaN
{
    const bool tiny = v < 0x1p-60f;
    const float vs = tiny ? __fmul_rn(v, 0x1p64f) : v;
    const bool zero = vs == 0.f;
    float s = __fsqrt_rn(zero ? 1.f : vs);
    s = tiny ? __fmul_rn(s, 0x1p-32f) : s;
    return zero ? 0.f : s;
}
__device__ __forceinline__ float opt_div_pos(float a, float b)   // b > 0 and b >= 2^-60 (here: >= 1e-15)
{
    const bool tiny = fabsf(a) < 0x1p-60f;
    const float as = tiny ? __fmul_rn(a, 0x1p64f) : a;
    const bool zero = as == 0.f && b > 0.f;
    if (tiny && !zero && fabsf(as) < __fmul_rn(b, 0x1p-58f))          // quotient may be subnormal: exact route, rare
        return __double2float_rn(__ddiv_rn((double)a, (double)b));
    float q = __fdiv_rn(zero ? 1.f : as, b);
    q = tiny ? __fmul_rn(q, 0x1p-64f) : q;
    return zero ? a : q;
}

__device__ __forceinline__ void adamw_element(float& p, float g, float& m, float& v, float decay, float neg_step, float bc2_sqrt,
                                              float w1, float beta2, float w2, float eps)
{
    const float p1 = __fmul_rn(p, decay);
    m = __fmaf_rn(w1, __fsub_rn(g, m), m);
    v = __fmaf_rn(w2, __fmul_rn(g, g), __fmul_rn(v, beta2));
    const float d = __fadd_rn(opt_div_pos(opt_sqrt(v), bc2_sqrt), eps);
    p = __fmaf_rn(neg_step, opt_div_pos(m, d), p1);
}

__global__ void __launch_bounds__(256) adamw_multi_kernel(const AdamTable t)
{
    int k = 0;
#pragma unroll
    for (int i = 1; i < OPT_MAX_TENSORS; i++)
        if (i < t.count && (int)blockIdx.x >= t.chunk_start[i]) k = i;
    const long long base = (long long)((int)blockIdx.x - t.chunk_start[k]) * OPT_CHUNK;
    const long long n = t.n[k];
    float* __restrict__ P = t.p[k];
    const float* __restrict__ G = t.g[k];
    float* __restrict__ M = t.m[k];
    float* __restrict__ V = t.v[k];
    const float decay = t.decay[k], neg_step = t.neg_step[k], bc2 = t.bc2_sqrt[k];
    const bool vec = ((reinterpret_cast<uintptr_t>(P) | reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(M) |
                       reinterpret_cast<uintptr_t>(V)) & 15) == 0;
    const int re = t.row_elems[k];
    if (re > 0) {  // row-strided parameter (the distillation student's _features_rest[:, :8, :]): gradient and moments are dense
        const long long rs = t.row_stride[k];
#pragma unroll 4
        for (int i = threadIdx.x; i < OPT_CHUNK; i += 256) {
            const long long e = base + i;
            if (e >= n) break;
            const long long row = e / re;
            float* pp = P + row * rs + (e - row * re);
            float p = *pp, m = M[e], v = V[e];
            adamw_element(p, G[e], m, v, decay, neg_step, bc2, t.w1, t.beta2, t.w2, t.eps);
            *pp = p; M[e] = m; V[e] = v;
        }
    } else if (vec && base + OPT_CHUNK <= n) {
        float4 p4[4], g4[4], m4[4], v4[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const long long e = base + (long long)(u * 256 + threadIdx.x) * 4;
            p4[u] = *reinterpret_cast<const float4*>(P + e);
            g4[u] = __ldcs(reinterpret_cast<const float4*>(G + e));     // gradients are read once: evict first
            m4[u] = *reinterpret_cast<const float4*>(M + e);
            v4[u] = *reinterpret_cast<const float4*>(V + e);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            adamw_element(p4[u].x, g4[u].x, m4[u].x, v4[u].x, decay, neg_step, bc2, t.w1, t.beta2, t.w2, t.eps);
            adamw_element(p4[u].y, g4[u].y, m4[u].y, v4[u].y, decay, neg_step, bc2, t.w1, t.beta2, t.w2, t.eps);
            adamw_element(p4[u].z, g4[u].z, m4[u].z, v4[u].z, decay, neg_step, bc2, t.w1, t.beta2, t.w2, t.eps);
            adamw_element(p4[u].w, g4[u].w, m4[u].w, v4[u].w, decay, neg_step, bc2, t.w1, t.beta2, t.w2, t.eps);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const long long e = base + (long long)(u * 256 + threadIdx.x) * 4;
            *reinterpret_cast<float4*>(P + e) = p4[u];
            *reinterpret_cast<float4*>(M + e) = m4[u];
            *reinterpret_cast<float4*>(V + e) = v4[u];
        }
    } else {  // last chunk of a tensor, or unaligned views
        for (int i = threadIdx.x; i < OPT_CHUNK; i += 256) {
            const long long e = base + i;
            if (e >= n) break;
            float p = P[e], m = M[e], v = V[e];
            adamw_element(p, G[e], m, v, decay, neg_step, bc2, t.w1, t.beta2, t.w2, t.eps);
            P[e] = p; M[e] = m; V[e] = v;
        }
    }
}

// ---- selective AdamW: only the rows (Gaussians) with a non-zero gradient -------------------------------------------------
// Every tensor is a [rows, width] view with its own (row stride, column stride) per array: dense [P, ...] is (width, 1), the
// distillation student's _features_rest[:, :8, :] is (45, 1) for the parameter and (24, 1) for its dense gradient and moments, the
// permuted _xyz of create_from_pcd is (1, P).  A block owns SEL_ROWS rows:
//   1. the gradient slice of every tensor for those rows goes to shared memory ([SEL_ROWS][width] per tensor) -- one TMA bulk copy
//      per tensor when the slice is one 16-byte aligned span (row-contiguous gradients), plain streaming loads otherwise;
//   2. a row is active when any element of it, in any tensor, compares unequal to zero (+0 and -0 do not, NaN does); one ballot per
//      warp and a 4-entry prefix turn the flags into an ascending list of active rows;
//   3. only the active rows are walked: p, m, v loaded, adamw_element (the dense kernel's arithmetic, unchanged), stored back.
// Inactive rows are never read or written.  Traffic: the gradients once, plus 24 B per element of the active rows.
constexpr int SEL_ROWS = 128;
constexpr int SEL_THREADS = 256;
constexpr int SEL_MAX_ROW_FLOATS = 400;       // sum of the widths: SEL_ROWS * 400 * 4 B = 200 KB of shared memory at most

struct SelAdamTable {
    float* p[OPT_MAX_TENSORS];
    const float* g[OPT_MAX_TENSORS];
    float* m[OPT_MAX_TENSORS];
    float* v[OPT_MAX_TENSORS];
    long long rs[OPT_MAX_TENSORS][4];       // row strides of p, g, m, v (elements)
    long long cs[OPT_MAX_TENSORS][4];       // column strides of p, g, m, v (elements)
    int width[OPT_MAX_TENSORS];
    int smem_off[OPT_MAX_TENSORS];          // float offset of the tensor's [SEL_ROWS][width] gradient slice in shared memory
    float decay[OPT_MAX_TENSORS];           // as AdamTable
    float neg_step[OPT_MAX_TENSORS];
    float bc2_sqrt[OPT_MAX_TENSORS];
    float w1, beta2, w2, eps;
    long long rows;
    int count;
};

__global__ void __launch_bounds__(SEL_THREADS) adamw_selective_kernel(const SelAdamTable t)
{
    extern __shared__ __align__(16) float sel_grad[];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int active_list[SEL_ROWS];
    __shared__ int warp_active[SEL_ROWS / 32];

    const long long r0 = (long long)blockIdx.x * SEL_ROWS;
    const int nr = (int)min((long long)SEL_ROWS, t.rows - r0);
    const int tid = threadIdx.x;

    // 1. gradient slices -> shared memory
    uint32_t bulk_bytes = 0;
    for (int k = 0; k < t.count; k++) {
        const int w = t.width[k];
        const float* src = t.g[k] + r0 * t.rs[k][1];
        const uint32_t bytes = (uint32_t)(nr * w) * 4u;
        if (t.cs[k][1] == 1 && t.rs[k][1] == w && ((reinterpret_cast<uintptr_t>(src) | bytes) & 15) == 0) {
            bulk_bytes += bytes;
            continue;
        }
        float* dst = sel_grad + t.smem_off[k];
        const long long rs = t.rs[k][1], cs = t.cs[k][1];
        if (cs == 1) {
            for (int e = tid; e < nr * w; e += SEL_THREADS) {
                const int r = e / w, c = e - r * w;
                dst[e] = __ldcs(src + r * rs + c);
            }
        } else {   // column-major walk: consecutive threads read consecutive rows of one column (the permuted _xyz)
            for (int e = tid; e < nr * w; e += SEL_THREADS) {
                const int c = e / nr, r = e - c * nr;
                dst[r * w + c] = __ldcs(src + r * rs + c * cs);
            }
        }
    }
    if (tid == 0 && bulk_bytes) {
        mbar_init(&bar, 1);
        fence_mbar_init();
        mbar_expect_tx(&bar, bulk_bytes);
        for (int k = 0; k < t.count; k++) {
            const int w = t.width[k];
            const float* src = t.g[k] + r0 * t.rs[k][1];
            const uint32_t bytes = (uint32_t)(nr * w) * 4u;
            if (t.cs[k][1] == 1 && t.rs[k][1] == w && ((reinterpret_cast<uintptr_t>(src) | bytes) & 15) == 0)
                bulk_g2s(sel_grad + t.smem_off[k], src, bytes, &bar);
        }
    }
    __syncthreads();                 // plain loads visible; the barrier is initialised before anyone waits on it
    if (bulk_bytes) mbar_wait(&bar, 0);

    // 2. active rows -> ascending list
    bool active = false;
    if (tid < nr) {
        for (int k = 0; k < t.count; k++) {
            const int w = t.width[k];
            const float* row = sel_grad + t.smem_off[k] + tid * w;
            for (int c = 0; c < w; c++) active |= row[c] != 0.f;
        }
    }
    const int lane = tid & 31, warp = tid >> 5;
    int rank = 0;
    if (warp < SEL_ROWS / 32) {
        const unsigned bal = __ballot_sync(FULL, active);
        rank = __popc(bal & ((1u << lane) - 1u));
        if (lane == 0) warp_active[warp] = __popc(bal);
    }
    __syncthreads();
    int n_active = 0, base = 0;
#pragma unroll
    for (int i = 0; i < SEL_ROWS / 32; i++) {
        if (i < warp) base += warp_active[i];
        n_active += warp_active[i];
    }
    if (active) active_list[base + rank] = tid;
    __syncthreads();
    if (n_active == 0) return;

    // 3. AdamW on the active rows only
    for (int k = 0; k < t.count; k++) {
        const int w = t.width[k];
        const float* G = sel_grad + t.smem_off[k];
        float* __restrict__ P = t.p[k];
        float* __restrict__ M = t.m[k];
        float* __restrict__ V = t.v[k];
        const long long rsp = t.rs[k][0], csp = t.cs[k][0], rsm = t.rs[k][2], csm = t.cs[k][2], rsv = t.rs[k][3], csv = t.cs[k][3];
        const float decay = t.decay[k], neg_step = t.neg_step[k], bc2 = t.bc2_sqrt[k];
        const bool by_column = csp != 1;   // permuted layouts: walk column by column so that a warp reads consecutive rows
        for (int e = tid; e < n_active * w; e += SEL_THREADS) {
            int i, c;
            if (by_column) { c = e / n_active; i = e - c * n_active; }
            else           { i = e / w; c = e - i * w; }
            const int r = active_list[i];
            const long long row = r0 + r;
            float* pp = P + row * rsp + c * csp;
            float* mp = M + row * rsm + c * csm;
            float* vp = V + row * rsv + c * csv;
            float p = *pp, m = *mp, v = *vp;
            adamw_element(p, G[r * w + c], m, v, decay, neg_step, bc2, t.w1, t.beta2, t.w2, t.eps);
            *pp = p; *mp = m; *vp = v;
        }
    }
}

// ---- row compaction -------------------------------------------------------------------------------------------------
constexpr int CMP_MAX_TENSORS = 24;
constexpr int CMP_CHUNK = 2048;      // output elements per block

struct CompactTable {
    const float* src[CMP_MAX_TENSORS];
    float* dst[CMP_MAX_TENSORS];
    int width[CMP_MAX_TENSORS];             // 4-byte words per row
    int chunk_start[CMP_MAX_TENSORS + 1];   // prefix sum of ceil(rows_out*width / CMP_CHUNK)
    int count;
    int rows_out;
};

__global__ void __launch_bounds__(256) compact_gather_kernel(const CompactTable t, const int* __restrict__ src_row)
{
    int k = 0;
    for (int i = 1; i < t.count; i++)
        if ((int)blockIdx.x >= t.chunk_start[i]) k = i;
    const int w = t.width[k];
    const long long total = (long long)t.rows_out * w;
    const long long base = (long long)((int)blockIdx.x - t.chunk_start[k]) * CMP_CHUNK;
    const float* __restrict__ S = t.src[k];
    float* __restrict__ D = t.dst[k];
#pragma unroll 4
    for (int i = threadIdx.x; i < CMP_CHUNK; i += 256) {
        const long long e = base + i;
        if (e >= total) break;
        const int j = (int)(e / w), c = (int)(e - (long long)j * w);
        D[e] = S[(long long)src_row[j] * w + c];
    }
}

}  // namespace
