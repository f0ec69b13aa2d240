// lgr_densify.cuh -- densification of GaussianModel (scene/gaussian_model.py:602-788), bit-identical to the reference's torch code:
//   * densify_stats_kernel  add_densification_stats (:784-788): accum += ||grad[i,:2]||, denom += 1 on the rows of the update filter,
//                           one pass, no host synchronisation (the reference's boolean indexing costs a nonzero() and a sync each).
//   * densify_plan_kernel   densify_and_prune's decisions for every row (:745-761): clone (:710-735), split (:666-708) and the final
//                           prune, as one class byte per row.  Every decision depends on the state only, not on the random samples:
//                           a split child's opacity is its parent's and its scaling is known before the draw.  A CUB scan of the four
//                           class counts then gives every output row its destination, and the totals are the one value read back.
//   * densify_rows_kernel   writes every output tensor in one pass, one warp per source row: the 6 parameters, the 12 Adam
//                           moments (zero for new rows) and the 3 auxiliary buffers (all zero).
//   * densify_split_inputs_kernel  the operands of the split's batched product bmm(build_rotation(q), samples) for the 2S children.
//                           No fixed operation order of the 3x3 . 3x1 product reproduces torch.bmm (cuBLAS) on every sample
//                           (scripts/exp_densify.py), so the caller runs torch.bmm on exactly the reference's [2S,3,3] x [2S,3,1]
//                           operands and densify_rows_kernel adds the parents' xyz to that product.
//
// Output row order, as the reference's three torch.cat + two prune_points leave it: unsplit original rows, clones, first copy of the
// split children, second copy (.repeat(2, 1) order), each ascending and without the pruned rows.
//
// Arithmetic, pinned with _rn intrinsics to what torch's kernels evaluate (scripts/exp_densify.py checks each on the GPU):
//   torch.norm(g[:, :2], dim=-1)   sqrt(a*a + b*b), each operation rounded on its own
//   torch.norm(grads, dim=-1)      sqrt(g*g) on a one-element row (not |g|)
//   build_rotation                 every eager operation rounded on its own
//   exp(s) / (0.8*2)               exp(s) * (1.0f / 1.6f): torch divides by a CPU scalar through its reciprocal
//   torch.normal(0, std)           n * std + 0, n from normal_(0, 1) drawn by the caller through torch's generator
// Denormals are kept (no FTZ), as torch's kernels keep them.
#pragma once

#include <cstdint>

namespace {

constexpr int DEN_MAX_TENSORS = 24;
constexpr uint8_t DEN_KEEP = 1, DEN_CLONE = 2, DEN_CHILD = 4, DEN_SPLIT = 8;   // class bits of a source row

using lgr::den_norm2;   // lgr_math.cuh: the sparse exchange publishes the same norm

// torch.max(x, dim=1).values of three values: NaN propagates
__device__ __forceinline__ float den_max3(float a, float b, float c)
{
    float m = a;
    if (b > m || isnan(b)) m = b;
    if (c > m || isnan(c)) m = c;
    return m;
}

// scaling_inverse_activation(get_scaling / (0.8 * N)) with N = 2
__device__ __forceinline__ float den_child_scale(float s) { return logf(__fmul_rn(act_exp(s), __fdiv_rn(1.0f, 1.6f))); }

// utils/general_utils.py build_rotation: R(q / |q|), row-major
__device__ __forceinline__ void den_rotation(float4 q, float R[9])
{
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.x, q.x), __fmul_rn(q.y, q.y)), __fmul_rn(q.z, q.z)), __fmul_rn(q.w, q.w)));
    const float r = __fdiv_rn(q.x, nrm), x = __fdiv_rn(q.y, nrm), y = __fdiv_rn(q.z, nrm), z = __fdiv_rn(q.w, nrm);
    R[0] = __fsub_rn(1.f, 2.f * __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z)));
    R[1] = 2.f * __fsub_rn(__fmul_rn(x, y), __fmul_rn(r, z));
    R[2] = 2.f * __fadd_rn(__fmul_rn(x, z), __fmul_rn(r, y));
    R[3] = 2.f * __fadd_rn(__fmul_rn(x, y), __fmul_rn(r, z));
    R[4] = __fsub_rn(1.f, 2.f * __fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z)));
    R[5] = 2.f * __fsub_rn(__fmul_rn(y, z), __fmul_rn(r, x));
    R[6] = 2.f * __fsub_rn(__fmul_rn(x, z), __fmul_rn(r, y));
    R[7] = 2.f * __fadd_rn(__fmul_rn(y, z), __fmul_rn(r, x));
    R[8] = __fsub_rn(1.f, 2.f * __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
}

__global__ void __launch_bounds__(256) densify_stats_kernel(int P, const float* __restrict__ grad, int grad_stride,
                                                            const uint8_t* __restrict__ filter, float* __restrict__ accum,
                                                            float* __restrict__ denom)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P || !filter[i]) return;
    const float* g = grad + (long long)i * grad_stride;
    accum[i] = __fadd_rn(accum[i], den_norm2(g[0], g[1]));
    denom[i] = __fadd_rn(denom[i], 1.0f);
}

// View-parallel statistics when the step's backward did not publish them in the sparse exchange: every rank encodes its view as one
// float per Gaussian (the norm on the rows of its filter, DEN_NO_VIEW elsewhere: a norm is never negative), the ranks all-gather the
// rows into [world, P], and densify_stats_views_kernel adds them in rank order with densify_stats_kernel's arithmetic.
constexpr uint32_t DEN_NO_VIEW = 0xBF800000u;   // -1.0f

__global__ void __launch_bounds__(256) densify_stats_encode_kernel(int P, const float* __restrict__ grad, int grad_stride,
                                                                   const uint8_t* __restrict__ filter, float* __restrict__ out)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P) return;
    const float* g = grad + (long long)i * grad_stride;
    out[i] = filter[i] ? den_norm2(g[0], g[1]) : __uint_as_float(DEN_NO_VIEW);
}

__global__ void __launch_bounds__(256) densify_stats_views_kernel(int P, int world, const float* __restrict__ views,
                                                                  float* __restrict__ accum, float* __restrict__ denom)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P) return;
    float acc = accum[i], den = denom[i];
    bool any = false;
    for (int v = 0; v < world; v++) {
        const float x = views[(long long)v * P + i];
        if (__float_as_uint(x) == DEN_NO_VIEW) continue;
        acc = __fadd_rn(acc, x);
        den = __fadd_rn(den, 1.0f);
        any = true;
    }
    if (any) { accum[i] = acc; denom[i] = den; }
}

struct DensifyPlanArgs {
    const float* accum;     // [P,1]
    const float* denom;     // [P,1]
    const float* scaling;   // [P,3] raw
    const float* opacity;   // [P,1] raw
    float max_grad, dense_scale, min_opacity, big_scale;   // thresholds as float32, as torch compares a float tensor with a scalar
    int prune_all, prune_big;
};

__device__ __forceinline__ bool den_pruned(float opacity_raw, float max_scale, const DensifyPlanArgs& a)
{
    return act_sigmoid(opacity_raw) < a.min_opacity || a.prune_all || (a.prune_big && max_scale > a.big_scale);
}

__global__ void __launch_bounds__(256) densify_plan_kernel(int P, const DensifyPlanArgs a, uint8_t* __restrict__ cls)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P) return;
    float g = __fdiv_rn(a.accum[i], a.denom[i]);
    if (isnan(g)) g = 0.f;
    const float s0 = a.scaling[3 * i], s1 = a.scaling[3 * i + 1], s2 = a.scaling[3 * i + 2];
    const float ms = den_max3(act_exp(s0), act_exp(s1), act_exp(s2));
    const float op = a.opacity[i];
    uint8_t c = 0;
    if (g >= a.max_grad && ms > a.dense_scale) {
        c = DEN_SPLIT;
        const float cm = den_max3(act_exp(den_child_scale(s0)), act_exp(den_child_scale(s1)), act_exp(den_child_scale(s2)));
        if (!den_pruned(op, cm, a)) c |= DEN_CHILD;
    } else if (!den_pruned(op, ms, a)) {
        c = DEN_KEEP;
        if (__fsqrt_rn(__fmul_rn(g, g)) >= a.max_grad && ms <= a.dense_scale) c |= DEN_CLONE;
    }
    cls[i] = c;
}

// class byte -> (kept original, kept clone, kept child pair, split) counts, scanned together
struct DenClassCounts {
    __host__ __device__ int4 operator()(uint8_t c) const
    {
        return make_int4(c & DEN_KEEP ? 1 : 0, c & DEN_CLONE ? 1 : 0, c & DEN_CHILD ? 1 : 0, c & DEN_SPLIT ? 1 : 0);
    }
};
struct DenInt4Sum {
    __host__ __device__ int4 operator()(const int4& a, const int4& b) const { return make_int4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
};

struct DensifyTable {
    const float* src[DEN_MAX_TENSORS];
    float* dst[DEN_MAX_TENSORS];
    int width[DEN_MAX_TENSORS];     // 4-byte words per row
    int role[DEN_MAX_TENSORS];      // LGR_DENSIFY_* of include/lgrast.h
    int count;
};

struct DensifyRowsArgs {
    const uint8_t* cls;
    const int4* scan;               // inclusive scan of DenClassCounts
    const float* xyz;
    const float* offsets;          // [2S,3] torch.bmm(R, samples) of the split children
    int kept, clones, children, splits;
};

__global__ void __launch_bounds__(256) densify_rows_kernel(int P, const DensifyTable t, const DensifyRowsArgs a)
{
    const int i = (int)((blockIdx.x * 256u + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= P) return;
    const uint8_t c = a.cls[i];
    if (!(c & (DEN_KEEP | DEN_CHILD))) return;
    const int4 inc = a.scan[i];
    const bool child = c & DEN_CHILD;
    long long d0 = -1, d1 = -1;                 // destination rows: original / first child, clone / second child
    if (child) {
        d0 = (long long)a.kept + a.clones + (inc.z - 1);
        d1 = d0 + a.children;
    } else {
        d0 = inc.x - 1;
        if (c & DEN_CLONE) d1 = (long long)a.kept + (inc.y - 1);
    }
    float x0 = 0.f, x1 = 0.f;                   // lanes 0..2: the children's xyz component `lane`
    if (child && lane < 3) {
        const long long r = inc.w - 1;          // rank among the split rows: children r and S + r
        const float p = a.xyz[3 * i + lane];
        x0 = __fadd_rn(a.offsets[3 * r + lane], p);
        x1 = __fadd_rn(a.offsets[3 * (a.splits + r) + lane], p);
    }
    for (int k = 0; k < t.count; k++) {
        const int w = t.width[k], role = t.role[k];
        const float* __restrict__ S = t.src[k];
        float* __restrict__ D = t.dst[k];
        for (int e = lane; e < w; e += 32) {
            float v0 = 0.f, v1 = 0.f;
            if (role == LGR_DENSIFY_MOMENT) {
                if (!child) v0 = S[(long long)i * w + e];
            } else if (role != LGR_DENSIFY_ZERO) {
                if (child && role == LGR_DENSIFY_XYZ) {
                    v0 = x0; v1 = x1;
                } else {
                    v0 = S[(long long)i * w + e];
                    if (child && role == LGR_DENSIFY_SCALING) v0 = den_child_scale(v0);
                    v1 = v0;
                }
            }
            D[d0 * w + e] = v0;
            if (d1 >= 0) D[d1 * w + e] = v1;
        }
    }
}

// rows r and S + r of the reference's rots = build_rotation(_rotation[sel]).repeat(2, 1, 1) and
// samples = torch.normal(mean=0, std=get_scaling[sel].repeat(2, 1)) = normal_(0, 1) * std + 0, for the split row of rank r
__global__ void __launch_bounds__(256) densify_split_inputs_kernel(int P, const uint8_t* __restrict__ cls, const int4* __restrict__ scan,
                                                                   const float* __restrict__ scaling, const float* __restrict__ rotation,
                                                                   const float* __restrict__ normals, int splits, float* __restrict__ R,
                                                                   float* __restrict__ samples)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P || !(cls[i] & DEN_SPLIT)) return;
    const long long r = scan[i].w - 1;
    float m[9];
    den_rotation(reinterpret_cast<const float4*>(rotation)[i], m);
    const float sd[3] = {act_exp(scaling[3 * i]), act_exp(scaling[3 * i + 1]), act_exp(scaling[3 * i + 2])};
    for (int copy = 0; copy < 2; copy++) {
        const long long row = r + (long long)copy * splits;
        for (int k = 0; k < 9; k++) R[9 * row + k] = m[k];
        for (int k = 0; k < 3; k++) samples[3 * row + k] = __fadd_rn(__fmul_rn(normals[3 * row + k], sd[k]), 0.0f);
    }
}

}  // namespace
