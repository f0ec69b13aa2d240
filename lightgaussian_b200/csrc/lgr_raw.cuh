// lgr_raw.cuh -- "raw leaves" variants of K1 and K7+K8 (SURVEY.md section 8f, row N1).
//
// gaussian_renderer.render() feeds the rasterizer activated copies of GaussianModel's leaves
// (scene/gaussian_model.py:98-118): exp(_scaling), normalize(_rotation), sigmoid(_opacity) and
// cat(_features_dc, _features_rest).  At 3M Gaussians that is ~1.3 GB of materialise-and-reread traffic plus the
// autograd backward of each op, per view.  These kernels read the leaves directly, apply the activations in
// registers -- in the exact float operation order of the torch CUDA kernels, so the activated values are
// bit-identical (asserted by tests/test_gpu_fused.py) -- and the backward writes gradients for the leaves.
//
// SH rows: a warp's 32 Gaussians own one contiguous run of _features_rest (32*(M-1)*12 B, 16-byte aligned) and of
// _features_dc (384 B).  Each warp that has at least one visible Gaussian fetches its run with ONE pair of TMA bulk
// copies (cp.async.bulk ... mbarrier::complete_tx) into its private shared-memory slice while the lanes finish the
// projection math; lanes then read their row with a (M-1)*3-word stride (45 words at degree 3: odd, so
// bank-conflict free).  The backward overwrites the row in place with dL/dSH and the warp writes it back with one
// bulk store.  Warps never synchronise with each other.
#pragma once

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
    return ok != 0;
}
// bounded wait: a lost copy becomes a trap (an error), never a hang
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
        if (spin > (1u << 24)) {
            printf("lgrast: bulk copy did not complete\n");
            __trap();
        }
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- activations, in the operation order of torch's CUDA kernels (exp_kernel_cuda, sigmoid_kernel_cuda, F.normalize) ----
__device__ __forceinline__ float act_exp(float x) { return expf(x); }
__device__ __forceinline__ float act_sigmoid(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }
// F.normalize(v, dim=1): v / max(||v||_2, 1e-12); the 4-element sum of squares reduces as (x^2 + z^2) + (y^2 + w^2)
__device__ __forceinline__ float4 act_normalize(float4 v, float& denom)
{
    const float s = __fadd_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.z, v.z)), __fadd_rn(__fmul_rn(v.y, v.y), __fmul_rn(v.w, v.w)));
    denom = fmaxf(__fsqrt_rn(s), 1e-12f);
    return make_float4(__fdiv_rn(v.x, denom), __fdiv_rn(v.y, denom), __fdiv_rn(v.z, denom), __fdiv_rn(v.w, denom));
}

struct RawArgs {
    int P, D, M, W, H, gx, gy;
    float fx, fy, tanx, tany, mod;
    const float* xyz;
    const float* view;
    const float* proj;
    const float* campos;
    int prefiltered;
    int rest_stride;  // floats per staged features_rest row (>= (M-1)*3; equal when the rows are dense)
};

// dynamic shared memory: 8 warp slices [32*stride floats rest | 32*3 floats dc], then 8 mbarriers, then camera (36 floats).
// `stride` = floats per staged features_rest row: (M-1)*3 for a dense leaf, the leaf's row stride for a row-strided view
// (the distillation student's _features_rest[:, :8, :], scene/gaussian_model.py:129-136, has stride 45 for 24 used floats).
__host__ __device__ inline size_t raw_smem_bytes_stride(int stride) { return (size_t)8 * 128 * (stride + 3) + 64 + 36 * 4; }
__host__ __device__ inline size_t raw_smem_bytes(int M) { return raw_smem_bytes_stride((M - 1) * 3); }

// Stage one warp's SH rows.  `first` = index of the warp's first Gaussian, `n` = valid Gaussians in the warp (<= 32),
// `nrest` = floats per row of `rest` in memory (the row stride: whole rows are staged, lanes read theirs at that stride).
__device__ __forceinline__ bool warp_stage_sh_begin(const float* __restrict__ rest, const float* __restrict__ dc, int nrest, int first, int n,
                                                    float* s_rest, float* s_dc, uint64_t* bar, int lane)
{
    const bool bulk = (n == 32);  // full warp: both runs are 16-byte aligned multiples of 16 bytes
    if (bulk) {
        if (lane == 0) {
            const uint32_t b_rest = 128u * (uint32_t)nrest, b_dc = 384u;
            mbar_expect_tx(bar, b_rest + b_dc);
            bulk_g2s(s_rest, rest + (size_t)first * nrest, b_rest, bar);
            bulk_g2s(s_dc, dc + (size_t)first * 3, b_dc, bar);
        }
    } else {  // ragged tail warp: plain loads
        for (int k = lane; k < n * nrest; k += 32) s_rest[k] = rest[(size_t)first * nrest + k];
        for (int k = lane; k < n * 3; k += 32) s_dc[k] = dc[(size_t)first * 3 + k];
    }
    return bulk;
}

// ---- attribute and colour sources of preprocess_raw_kernel ----
// A source hands the kernel the RAW (pre-activation) scaling, rotation and opacity of Gaussian i and stages a warp's SH rows into
// shared memory as float32 in the leaves' layout (per lane: rest [(M-1)][3] at `nrest` floats per lane, dc [3]).  Everything else
// -- projection, activations, tile-keep mask, sh_to_rgb -- is the one kernel body, so every source renders bit-identically to the
// float32 leaves holding the same values.

// GaussianModel's six float32 leaves (scene/gaussian_model.py:46-56); features_rest rows may be row-strided (RawArgs::rest_stride).
struct LeafSource {
    const float* dc;
    const float* rest;
    const float* scaling_;
    const float* rotation_;
    const float* opacity_;
    __device__ __forceinline__ float scaling(int i, int k) const { return scaling_[3 * (size_t)i + k]; }
    __device__ __forceinline__ float4 rotation(int i) const { return reinterpret_cast<const float4*>(rotation_)[i]; }
    __device__ __forceinline__ float opacity(int i) const { return opacity_[i]; }
    __device__ __forceinline__ bool stage(int nrest, int first, int n, unsigned, float* s_rest, float* s_dc, uint64_t* bar, int lane) const
    {
        return warp_stage_sh_begin(rest, dc, nrest, first, n, s_rest, s_dc, bar, lane);
    }
};

// A VecTree-compressed model as extreme_saving/ stores it (lgr_vq_resident_params): attributes [P,8] = opacity | scale x3 | rot x4 in
// fp16 or float32, and per Gaussian either a codebook row (slot >= 0) or its own row of `nonvq` (slot = -(row) - 1).  Colour rows
// hold D = 3M values in PLY order, f_dc_0..2 then f_rest CHANNEL-major (row[3 + c*(M-1) + j]), `Dp` elements apart; staging
// transposes them to the leaves' coefficient-major layout.  fp16 -> float32 is exact, so the staged values are those of the
// float32 leaves GaussianModel.load_vq builds from the same files.
struct VqSource {
    const void* attr;
    const int* slot;
    const __half* codebook;
    const void* nonvq;
    int attr_half, nonvq_half, D, Dp, M;
    __device__ __forceinline__ float attr_at(int i, int k) const
    {
        return attr_half ? __half2float(static_cast<const __half*>(attr)[8 * (size_t)i + k]) : static_cast<const float*>(attr)[8 * (size_t)i + k];
    }
    __device__ __forceinline__ float scaling(int i, int k) const { return attr_at(i, 1 + k); }
    __device__ __forceinline__ float opacity(int i) const { return attr_at(i, 0); }
    __device__ __forceinline__ float4 rotation(int i) const
    {
        if (!attr_half) return reinterpret_cast<const float4*>(attr)[2 * (size_t)i + 1];
        const uint2 u = reinterpret_cast<const uint2*>(attr)[2 * (size_t)i + 1];
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        return make_float4(a.x, a.y, b.x, b.y);
    }
    // The warp's visible rows are fetched in 16-byte pieces spread over all lanes: consecutive non-VQ rows (slots are a prefix
    // count) are read coalesced, codebook rows are gathers from an L2-resident table.  Plain stores: the caller's __syncwarp orders them.
    __device__ __forceinline__ bool stage(int nrest, int first, int n, unsigned vis, float* s_rest, float* s_dc, uint64_t*, int lane) const
    {
        const int per_row = nonvq_half ? Dp / 8 : Dp / 4;  // 16-byte pieces of the widest row
        const int total = n * per_row;
        const int my_slot = lane < n ? slot[first + lane] : 0;  // one coalesced load; pieces get their row's slot by shuffle
        for (int base = 0; base < total; base += 32) {      // warp-uniform trip count: every lane takes part in the shuffle
            const int c = base + lane;
            const int g = min(c, total - 1) / per_row, part = c - g * per_row;
            const int s = __shfl_sync(0xffffffffu, my_slot, g);
            if (c >= total || !((vis >> g) & 1u)) continue;
            float v[8];
            int e0, cnt;
            if (s >= 0 || nonvq_half) {
                if (part * 8 >= Dp) continue;
                const __half* row = s >= 0 ? codebook + (size_t)s * Dp : static_cast<const __half*>(nonvq) + (size_t)(-s - 1) * Dp;
                const uint4 u = *reinterpret_cast<const uint4*>(row + part * 8);
                const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float2 f = __half22float2(h[k]);
                    v[2 * k] = f.x;
                    v[2 * k + 1] = f.y;
                }
                e0 = part * 8;
                cnt = 8;
            } else {
                const float4 f = reinterpret_cast<const float4*>(static_cast<const float*>(nonvq) + (size_t)(-s - 1) * Dp)[part];
                v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
                e0 = part * 4;
                cnt = 4;
            }
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int e = e0 + k;
                if (k >= cnt) break;
                if (e < 3) {
                    s_dc[3 * g + e] = v[k];
                } else if (e < D) {
                    const int ch = (e - 3) / (M - 1), j = (e - 3) - ch * (M - 1);
                    s_rest[g * nrest + 3 * j + ch] = v[k];
                }
            }
        }
        return false;
    }
};

template <class Src>
__global__ void __launch_bounds__(256) preprocess_raw_kernel(RawArgs a, Src src, int* __restrict__ radii, GeometryState g)
{
    extern __shared__ __align__(128) unsigned char dyn_smem[];
    const int nrest = a.rest_stride;   // floats per staged row (the leaf's row stride)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* s_rest = reinterpret_cast<float*>(dyn_smem) + (size_t)warp * 32 * (nrest + 3);
    float* s_dc = s_rest + 32 * nrest;
    uint64_t* bars = reinterpret_cast<uint64_t*>(dyn_smem + (size_t)8 * 128 * (nrest + 3));
    float* s_cam = reinterpret_cast<float*>(bars + 8);
    if (threadIdx.x < 16) s_cam[threadIdx.x] = a.view[threadIdx.x];
    else if (threadIdx.x < 32) s_cam[threadIdx.x] = a.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_cam[threadIdx.x] = a.campos[threadIdx.x - 32];
    if (lane == 0) {
        mbar_init(&bars[warp], 1);
        fence_mbar_init();
    }
    __syncthreads();
    const float* view = s_cam;
    const float* proj = s_cam + 16;
    const float* cam = s_cam + 32;

    const int first = blockIdx.x * 256 + warp * 32;
    if (first >= a.P) return;
    const int n = min(32, a.P - first);
    const int i = first + lane;
    const bool valid = lane < n;

    float x = 0.f, y = 0.f, z = 0.f, cov[6];
    lgr::Geom geo;
    bool visible = false;
    if (valid) {
        x = a.xyz[3 * (size_t)i]; y = a.xyz[3 * (size_t)i + 1]; z = a.xyz[3 * (size_t)i + 2];
        visible = lgr::xform_row(view, 2, x, y, z) > 0.2f;
        if (visible) {
            const float s0 = act_exp(src.scaling(i, 0)), s1 = act_exp(src.scaling(i, 1)), s2 = act_exp(src.scaling(i, 2));
            float dn;
            const float4 q = act_normalize(src.rotation(i), dn);
            lgr::cov3d_from_scale_rot(s0, s1, s2, a.mod, q.x, q.y, q.z, q.w, cov);
#pragma unroll
            for (int k = 0; k < 6; k++) g.cov3D[6 * (size_t)i + k] = cov[k];
            visible = lgr::project_gaussian(x, y, z, view, proj, cov, a.fx, a.fy, a.tanx, a.tany, a.W, a.H, a.gx, a.gy, geo);
        } else if (a.prefiltered) {
            printf("Point is filtered although prefiltered is set. This shouldn't happen!");
            __trap();
        }
    }
    const unsigned vis_bits = __ballot_sync(FULL, visible);
    const bool any_vis = vis_bits != 0u;
    bool bulk = false;
    if (any_vis) bulk = src.stage(nrest, first, n, vis_bits, s_rest, s_dc, &bars[warp], lane);

    // everything that does not need the SH rows overlaps the copy
    const float op_act = visible ? act_sigmoid(src.opacity(i)) : 0.f;
    const unsigned long long keep_bits = warp_tile_keep_mask(visible, geo, make_float4(geo.conic_x, geo.conic_y, geo.conic_z, op_act), a.W, a.H, lane);
    if (valid) {
        if (!g.bin_rec) g.iota[i] = (uint32_t)i;
        if (!visible) {
            radii[i] = 0;
            g.tiles_touched[i] = 0;
            if (g.bin_rec) g.bin_rec[i] = make_uint4(0u, 0u, 0u, 0u);
            else g.tiles_kept[i] = 0;
            g.depth_keys[i] = 0xffffffffu;
            g.clamped[i] = 0;
        } else {
            radii[i] = geo.radius;
            g.depth[i] = geo.depth;
            g.depth_keys[i] = __float_as_uint(geo.depth);
            g.means2D[i] = make_float2(geo.px, geo.py);
            const float4 co = make_float4(geo.conic_x, geo.conic_y, geo.conic_z, op_act);
            g.conic_opacity[i] = co;
            const uint32_t area = (uint32_t)((geo.rect.y1 - geo.rect.y0) * (geo.rect.x1 - geo.rect.x0));
            g.tiles_touched[i] = area;
            const unsigned long long mask = keep_bits;
            const uint32_t kept = area > 64u ? area : (uint32_t)__popcll(mask);
            if (g.bin_rec) {
                g.bin_rec[i] = make_bin_rec(geo.rect.x0, geo.rect.y0, geo.rect.x1 - geo.rect.x0, geo.rect.y1 - geo.rect.y0, mask);
            } else {
                g.tiles_kept[i] = kept;
                g.keep_mask[i] = mask;
            }
        }
    }
    if (!any_vis) return;
    if (bulk) mbar_wait(&bars[warp], 0);
    else __syncwarp();
    if (visible) {
        const float* rr = s_rest + lane * nrest;
        const float* dd = s_dc + lane * 3;
        float rgb[3];
        unsigned clamp_bits;
        lgr::sh_to_rgb(a.D, [&](int k) { return k < 3 ? dd[k] : rr[k - 3]; }, x, y, z, cam, rgb, clamp_bits);
        g.rgb[i] = make_float4(rgb[0], rgb[1], rgb[2], 0.f);
        g.clamped[i] = (uint8_t)clamp_bits;
    }
}

struct RawBackArgs {
    int P, D, M, W, H;
    float fx, fy, tanx, tany, mod;
    const float* xyz;
    const float* dc;
    const float* rest;
    const float* scaling;
    const float* rotation;
    const float* cov3D;
    const float4* conic_opacity;
    const float* view;
    const float* proj;
    const float* campos;
    const int* radii;
    const uint8_t* clamped;
    const float* acc;
    float* d_xyz;
    float* d_dc;
    float* d_rest;
    float* d_scaling;
    float* d_rotation;
    float* d_opacity;
    float* dL_dmeans2D;
    int rest_stride;  // floats between consecutive rows of `rest` ((M-1)*3 when dense); gradients are always dense
    int block0;    // first 256-Gaussian block this launch covers (ranged launches of the view-parallel exchange)
    float* d_rgb;  // optional [P,3]: clamp-masked dL/dRGB (compact SH gradient factor); when set and d_rest == NULL the dense SH rows are not written
};

// The depth variant's extra K7+K8 input (lgr_backward_raw_depth): accumulator word 9 holds dL/d(depth value), the value being z
// (mode 1) or the forward's correctly rounded 1/z (mode 2); dL/dz reaches dL/dxyz through z = view[2] x + view[6] y + view[10] z + view[14].
struct RawDepth {
    const float* z;   // [P] view-space depth of the geometry blob
    int mode;         // 0 = alpha only (word 9 is zero), 1 = z, 2 = inverse
};

// dL/dz of Gaussian i from its accumulator record (word 9 = dL/d(depth value))
__device__ __forceinline__ float depth_grad_z(const RawDepth& dz, const float* __restrict__ rec, size_t i)
{
    float g = rec[9];
    if (dz.mode == 2) {
        const float r = __frcp_rn(dz.z[i]);
        g = -(g * r) * r;
    }
    return g;
}

__device__ __forceinline__ void depth_grad_to_mean(const RawDepth& dz, const float* __restrict__ rec, size_t i, const float* view, float* dmean)
{
    const float g = depth_grad_z(dz, rec, i);
    dmean[0] = fmaf(g, view[2], dmean[0]);
    dmean[1] = fmaf(g, view[6], dmean[1]);
    dmean[2] = fmaf(g, view[10], dmean[2]);
}

// ---- camera gradients (lgr_backward_raw_camera, DESIGN.md section 7) ----
// Each differentiated Gaussian contributes 27 live terms:
//   [3r + k]       dL/dV[4r + k]       r = 0..3, k = 0..2   (V = viewmatrix; V[4r + 3] is never read)
//   [12 + 3r + k]  dL/dPm[4r + c_k]    c = (0, 1, 3)        (Pm = projmatrix; Pm[4r + 2] is never read)
//   [24 + c]       dL/dcampos[c]
// A warp sums its lanes' terms with a fixed butterfly, the warps of a block add theirs in warp order in shared memory, and the block
// writes one 27-float row (entry k of block b at rows[k * gridDim.x + b]); camera_grad_finish_kernel adds the rows.  No float atomics.
constexpr int CAM_TERMS = 27;

// dcam: cov2d_backward's camera output (dL/dt incl. any depth-plane dL/dz, then the T = J W term); dh: mean2d_backward's; ddir:
// sh_backward's view-direction term.  p = (x, y, z, 1) is the world mean.
__device__ __forceinline__ void cam_terms(const float* dcam, const float* dh, const float* ddir, float x, float y, float z, float* t)
{
    const float p[4] = {x, y, z, 1.f};
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int k = 0; k < 3; k++) {
            t[3 * r + k] = r < 3 ? fmaf(p[r], dcam[k], dcam[3 + 3 * r + k]) : dcam[k];
            t[12 + 3 * r + k] = p[r] * dh[k];
        }
    t[24] = -ddir[0]; t[25] = -ddir[1]; t[26] = -ddir[2];
}

// the warp's sum of t[] into lane 0's `acc` row (acc += sum); every lane must call it
__device__ __forceinline__ void cam_warp_add(float* t, float* acc, int lane)
{
#pragma unroll
    for (int k = 0; k < CAM_TERMS; k++) {
        float s = t[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(FULL, s, off);
        if (lane == 0) acc[k] += s;
    }
}

// after a __syncthreads: entry k of this block's row = sum over the block's warps, in warp order
__device__ __forceinline__ void cam_block_row(const float* part, int nwarps, float* rows)
{
    if (threadIdx.x < CAM_TERMS) {
        float s = part[threadIdx.x];
        for (int w = 1; w < nwarps; w++) s += part[w * CAM_TERMS + threadIdx.x];
        rows[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = s;
    }
}

// dL/dviewmatrix [16], dL/dprojmatrix [16], dL/dcampos [3] from `nrows` block rows: warp k adds entry k, lane l the rows l, l + 32, ...
// in order, then a fixed butterfly -- the same order for every run with the same rows.  The eight unread entries are written as 0.
__global__ void __launch_bounds__(1024) camera_grad_finish_kernel(const float* __restrict__ rows, int nrows, float* __restrict__ dview,
                                                                  float* __restrict__ dproj, float* __restrict__ dcampos)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp < CAM_TERMS) {
        float s = 0.f;
        for (int b = lane; b < nrows; b += 32) s += rows[(size_t)warp * nrows + b];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(FULL, s, off);
        if (lane == 0) {
            if (warp < 12) dview[4 * (warp / 3) + warp % 3] = s;
            else if (warp < 24) dproj[4 * ((warp - 12) / 3) + ((warp - 12) % 3 == 2 ? 3 : (warp - 12) % 3)] = s;
            else dcampos[warp - 24] = s;
        }
    } else if (warp == CAM_TERMS && lane < 8) {
        if (lane < 4) dview[4 * lane + 3] = 0.f;
        else dproj[4 * (lane - 4) + 2] = 0.f;
    }
}

template <bool DEPTH, bool CAM = false>
__device__ __forceinline__ void preprocess_backward_raw_body(const RawBackArgs& a, const RawDepth& dz, float* cam_part = nullptr)
{
    extern __shared__ __align__(128) unsigned char dyn_smem[];
    const int nrest = (a.M - 1) * 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* s_rest = reinterpret_cast<float*>(dyn_smem) + (size_t)warp * 32 * (nrest + 3);
    float* s_dc = s_rest + 32 * nrest;
    uint64_t* bars = reinterpret_cast<uint64_t*>(dyn_smem + (size_t)8 * 128 * (nrest + 3));
    float* s_cam = reinterpret_cast<float*>(bars + 8);
    if (threadIdx.x < 16) s_cam[threadIdx.x] = a.view[threadIdx.x];
    else if (threadIdx.x < 32) s_cam[threadIdx.x] = a.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_cam[threadIdx.x] = a.campos[threadIdx.x - 32];
    if (CAM && threadIdx.x < 8 * CAM_TERMS) cam_part[threadIdx.x] = 0.f;   // warps that have no Gaussian add nothing
    if (lane == 0) {
        mbar_init(&bars[warp], 1);
        fence_mbar_init();
    }
    __syncthreads();
    const float* view = s_cam;
    const float* proj = s_cam + 16;
    const float* cam = s_cam + 32;

    const int first = (a.block0 + (int)blockIdx.x) * 256 + warp * 32;
    if (first >= a.P) return;
    const int n = min(32, a.P - first);
    const int i = first + lane;
    const size_t si = (size_t)i;
    const bool valid = lane < n;
    // A visible Gaussian whose blend-backward accumulators are all zero (measured: 87 % of them on the bench scene -- the pixels
    // saturate long before the deep Gaussians are reached) has exactly-zero gradients in every output: it is treated like a culled
    // one, i.e. only its 48-byte accumulator record is read and zero rows are written.
    bool vis = valid && a.radii[i] > 0;
    if (vis) {
        const float4* r4 = reinterpret_cast<const float4*>(a.acc + si * ACC_STRIDE);
        const float4 r0 = r4[0], r1 = r4[1];
        const float r2 = a.acc[si * ACC_STRIDE + 8];
        vis = r0.x != 0.f || r0.y != 0.f || r0.z != 0.f || r0.w != 0.f || r1.x != 0.f || r1.y != 0.f || r1.z != 0.f || r1.w != 0.f || r2 != 0.f;
        if (DEPTH) vis = vis || a.acc[si * ACC_STRIDE + 9] != 0.f;
    }
    const unsigned live = __ballot_sync(FULL, vis);
    const bool any_vis = live != 0;
    // The SH values are only needed for the view-direction term (degree >= 1).  The warp's rows are staged with one TMA bulk copy
    // only when enough of its lanes need them (>= 12 of 32: 6 KB of staging vs 192-byte rows read privately); otherwise -- and always
    // for a row-strided leaf (rest_stride != nrest), whose staging slice holds the DENSE gradient rows -- the lanes read their own
    // coefficients from global memory
    const bool strided = a.rest_stride != nrest || __popc(live) < 12;
    const bool need_sh = any_vis && a.D > 0 && !strided;
    bool bulk = false;
    if (need_sh) bulk = warp_stage_sh_begin(a.rest, a.dc, nrest, first, n, s_rest, s_dc, &bars[warp], lane);

    float dmean[3] = {0.f, 0.f, 0.f}, dscale[3] = {0.f, 0.f, 0.f}, dq[4] = {0.f, 0.f, 0.f, 0.f};
    float dop = 0.f, g2x = 0.f, g2y = 0.f, dRGB[3] = {0.f, 0.f, 0.f};
    float x = 0.f, y = 0.f, z = 0.f;
    float cin[CAM ? 18 : 1];   // CAM: cov2d_backward's 12 camera values, mean2d_backward's 3, sh_backward's 3 (zero when not differentiated)
#pragma unroll
    for (int k = 0; k < (CAM ? 18 : 1); k++) cin[k] = 0.f;
    if (vis) {
        const float4 co = a.conic_opacity[si];
        const Grad2D g2 = accum_to_grad2d(a.acc + si * ACC_STRIDE, co, a.W, a.H);
        x = a.xyz[3 * si]; y = a.xyz[3 * si + 1]; z = a.xyz[3 * si + 2];
        float c3[6], dcov[6];
#pragma unroll
        for (int k = 0; k < 6; k++) c3[k] = a.cov3D[6 * si + k];
        lgr::cov2d_backward(x, y, z, view, c3, a.fx, a.fy, a.tanx, a.tany, g2.dcx, g2.dcy, g2.dcw, dcov, dmean, CAM ? cin : nullptr);
        lgr::mean2d_backward(x, y, z, proj, g2.dm2x, g2.dm2y, dmean, CAM ? cin + 12 : nullptr);
        if (DEPTH) depth_grad_to_mean(dz, a.acc + si * ACC_STRIDE, si, view, dmean);
        if (CAM && DEPTH) cin[2] += depth_grad_z(dz, a.acc + si * ACC_STRIDE, si);   // z = t_2
        g2x = g2.dm2x; g2y = g2.dm2y;
        const unsigned cb = a.clamped[i];
        dRGB[0] = (cb & 1u) ? 0.f : g2.dcol[0]; dRGB[1] = (cb & 2u) ? 0.f : g2.dcol[1]; dRGB[2] = (cb & 4u) ? 0.f : g2.dcol[2];
        // scale / rotation chain: activations recomputed, then d/d(raw)
        const float s0 = act_exp(a.scaling[3 * si]), s1 = act_exp(a.scaling[3 * si + 1]), s2 = act_exp(a.scaling[3 * si + 2]);
        float dn;
        const float4 v = reinterpret_cast<const float4*>(a.rotation)[si];
        const float4 q = act_normalize(v, dn);
        float ds[3], dqn[4];
        lgr::cov3d_backward(s0, s1, s2, a.mod, q.x, q.y, q.z, q.w, dcov, ds, dqn);
        dscale[0] = ds[0] * s0; dscale[1] = ds[1] * s1; dscale[2] = ds[2] * s2;  // ExpBackward: grad * exp(x)
        // F.normalize backward: (g - q (q.g)) / max(||v||, eps)
        const float qg = q.x * dqn[0] + q.y * dqn[1] + q.z * dqn[2] + q.w * dqn[3];
        const float inv = 1.0f / dn;
        dq[0] = (dqn[0] - q.x * qg) * inv; dq[1] = (dqn[1] - q.y * qg) * inv;
        dq[2] = (dqn[2] - q.z * qg) * inv; dq[3] = (dqn[3] - q.w * qg) * inv;
        const float o = co.w;                    // sigmoid(raw), stored by the forward
        dop = (g2.dop * (1.0f - o)) * o;         // sigmoid_backward: grad * (1 - y) * y
    }
    if (need_sh) {
        if (bulk) mbar_wait(&bars[warp], 0);
        else __syncwarp();
    }
    // SH gradient rows are produced in place in the warp's slice (zeros for culled Gaussians / inactive degrees)
    float* rr = s_rest + lane * nrest;
    float* dd = s_dc + lane * 3;
    if (valid) {
        if (vis) {
            if (a.D > 0 && strided) {
                const float* gr = a.rest + si * a.rest_stride;
                const float* gd = a.dc + si * 3;
                lgr::sh_backward(a.D, [&](int k) { return k < 3 ? __ldg(gd + k) : __ldg(gr + k - 3); },
                                 [&](int k, int c, float val) {
                                     if (k == 0) dd[c] = val;
                                     else rr[3 * (k - 1) + c] = val;
                                 },
                                 x, y, z, cam, dRGB, dmean, CAM ? cin + 15 : nullptr);
            } else if (a.D > 0) {
                lgr::sh_backward(a.D, [&](int k) { return k < 3 ? dd[k] : rr[k - 3]; },
                                 [&](int k, int c, float val) {
                                     if (k == 0) dd[c] = val;
                                     else rr[3 * (k - 1) + c] = val;
                                 },
                                 x, y, z, cam, dRGB, dmean, CAM ? cin + 15 : nullptr);
            } else {
#pragma unroll
                for (int c = 0; c < 3; c++) dd[c] = LGR_C0 * dRGB[c];
            }
            const int nb = (a.D + 1) * (a.D + 1);
            for (int k = 3 * (nb - 1); k < nrest; k++) rr[k] = 0.f;
        } else {
            for (int k = 0; k < nrest; k++) rr[k] = 0.f;
            dd[0] = 0.f; dd[1] = 0.f; dd[2] = 0.f;
        }
        a.d_xyz[3 * si] = dmean[0]; a.d_xyz[3 * si + 1] = dmean[1]; a.d_xyz[3 * si + 2] = dmean[2];
        a.d_scaling[3 * si] = dscale[0]; a.d_scaling[3 * si + 1] = dscale[1]; a.d_scaling[3 * si + 2] = dscale[2];
        reinterpret_cast<float4*>(a.d_rotation)[si] = make_float4(dq[0], dq[1], dq[2], dq[3]);
        a.d_opacity[si] = dop;
        a.dL_dmeans2D[3 * si] = g2x; a.dL_dmeans2D[3 * si + 1] = g2y; a.dL_dmeans2D[3 * si + 2] = 0.f;
        if (a.d_rgb) {
            a.d_rgb[3 * si] = dRGB[0]; a.d_rgb[3 * si + 1] = dRGB[1]; a.d_rgb[3 * si + 2] = dRGB[2];
        }
    }
    if (CAM) {
        float t[CAM_TERMS];
        cam_terms(cin, cin + 12, cin + 15, x, y, z, t);
        cam_warp_add(t, cam_part + warp * CAM_TERMS, lane);
    }
    if (a.d_rest == nullptr) return;  // compact mode: the SH gradient is rebuilt from d_rgb (sh_grad_from_views_kernel)
    __syncwarp();
    if (n == 32) {
        fence_async_smem();  // generic-proxy writes above -> visible to the bulk (async-proxy) store
        __syncwarp();
        if (lane == 0) {
            bulk_s2g(a.d_rest + (size_t)first * nrest, s_rest, 128u * (uint32_t)nrest);
            bulk_s2g(a.d_dc + (size_t)first * 3, s_dc, 384u);
            bulk_commit();
            bulk_wait_read_all();  // shared memory must stay valid until the copy engine has read it
        }
    } else {
        for (int k = lane; k < n * nrest; k += 32) a.d_rest[(size_t)first * nrest + k] = s_rest[k];
        for (int k = lane; k < n * 3; k += 32) a.d_dc[(size_t)first * 3 + k] = s_dc[k];
    }
}

__global__ void __launch_bounds__(256) preprocess_backward_raw_kernel(RawBackArgs a) { preprocess_backward_raw_body<false>(a, RawDepth{}); }
__global__ void __launch_bounds__(256) preprocess_backward_raw_depth_kernel(RawBackArgs a, RawDepth dz) { preprocess_backward_raw_body<true>(a, dz); }

// the dense kernels plus one camera-gradient row per block (rows: [27][gridDim.x])
template <bool DEPTH>
__device__ __forceinline__ void preprocess_backward_raw_cam_body(const RawBackArgs& a, const RawDepth& dz, float* __restrict__ cam_rows)
{
    __shared__ float part[8 * CAM_TERMS];
    preprocess_backward_raw_body<DEPTH, true>(a, dz, part);
    __syncthreads();
    cam_block_row(part, 8, cam_rows);
}
__global__ void __launch_bounds__(256) preprocess_backward_raw_cam_kernel(RawBackArgs a, float* cam_rows)
{
    preprocess_backward_raw_cam_body<false>(a, RawDepth{}, cam_rows);
}
__global__ void __launch_bounds__(256) preprocess_backward_raw_depth_cam_kernel(RawBackArgs a, RawDepth dz, float* cam_rows)
{
    preprocess_backward_raw_cam_body<true>(a, dz, cam_rows);
}

// ------------------------------------------------------------------------------------------------------------------
// View-parallel SH gradient.  For one view dL/dSH[k][c] = basis_k(dir) * dRGB[c] is rank-1 per Gaussian
// (RAST/cuda_rasterizer/backward.cu:44-97), so ranks exchange the 3-float factor dRGB (all-gather, 12 B/Gaussian/view)
// instead of all-reducing 12*M B/Gaussian, and every rank rebuilds  sum_v basis(dir_v) (x) dRGB_v  here.
// dir_v = normalize(xyz - campos_v).  Rows are staged in shared memory and written with one bulk store per warp.
// ------------------------------------------------------------------------------------------------------------------
struct ShGradArgs {
    int P, D, M, n_views;
    const float* xyz;
    const float* campos;  // [n_views,3]
    const float* d_rgb;   // [n_views,P,3]
    float* d_dc;          // [P,3]
    float* d_rest;        // [P,(M-1)*3]
};

__global__ void __launch_bounds__(256) sh_grad_from_views_kernel(ShGradArgs a)
{
    extern __shared__ __align__(128) unsigned char dyn_smem[];
    const int nrest = (a.M - 1) * 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* s_rest = reinterpret_cast<float*>(dyn_smem) + (size_t)warp * 32 * (nrest + 3);
    float* s_dc = s_rest + 32 * nrest;
    const int first = blockIdx.x * 256 + warp * 32;
    if (first >= a.P) return;
    const int n = min(32, a.P - first);
    const int i = first + lane;
    const size_t si = (size_t)i;
    float* rr = s_rest + lane * nrest;
    float* dd = s_dc + lane * 3;
    if (lane < n) {
        const float x = a.xyz[3 * si], y = a.xyz[3 * si + 1], z = a.xyz[3 * si + 2];
        float acc[48];
#pragma unroll
        for (int k = 0; k < 48; k++) acc[k] = 0.f;
        for (int v = 0; v < a.n_views; v++) {
            const float* g = a.d_rgb + ((size_t)v * a.P + si) * 3;
            const float dRGB[3] = {g[0], g[1], g[2]};
            if (dRGB[0] == 0.f && dRGB[1] == 0.f && dRGB[2] == 0.f) continue;  // culled / fully clamped in this view
            float unused[3] = {0.f, 0.f, 0.f};
            const float cam[3] = {a.campos[3 * v], a.campos[3 * v + 1], a.campos[3 * v + 2]};
            lgr::sh_backward(a.D, [&](int) { return 0.f; }, [&](int k, int c, float val) { acc[3 * k + c] += val; }, x, y, z, cam, dRGB,
                             unused);
        }
        dd[0] = acc[0]; dd[1] = acc[1]; dd[2] = acc[2];
#pragma unroll
        for (int k = 3; k < 48; k++)
            if (k - 3 < nrest) rr[k - 3] = acc[k];
    }
    __syncwarp();
    if (n == 32) {
        fence_async_smem();
        __syncwarp();
        if (lane == 0) {
            bulk_s2g(a.d_rest + (size_t)first * nrest, s_rest, 128u * (uint32_t)nrest);
            bulk_s2g(a.d_dc + (size_t)first * 3, s_dc, 384u);
            bulk_commit();
            bulk_wait_read_all();
        }
    } else {
        for (int k = lane; k < n * nrest; k += 32) a.d_rest[(size_t)first * nrest + k] = s_rest[k];
        for (int k = lane; k < n * 3; k += 32) a.d_dc[(size_t)first * 3 + k] = s_dc[k];
    }
}

// dL/dRGB of this view straight from the blend-backward accumulators (clamp-masked, zero for culled Gaussians), so that the
// all-gather of the compact SH factor can start BEFORE the per-Gaussian backward kernel runs.
__global__ void __launch_bounds__(256) extract_drgb_kernel(int P, const int* __restrict__ radii, const uint8_t* __restrict__ clamped,
                                                           const float* __restrict__ acc, float* __restrict__ d_rgb)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float r = 0.f, g = 0.f, b = 0.f;
    if (radii[i] > 0) {
        const float4 r0 = *reinterpret_cast<const float4*>(acc + (size_t)i * ACC_STRIDE);
        const unsigned cb = clamped[i];
        r = (cb & 1u) ? 0.f : r0.x;
        g = (cb & 2u) ? 0.f : r0.y;
        b = (cb & 4u) ? 0.f : r0.z;
    }
    d_rgb[3 * (size_t)i] = r; d_rgb[3 * (size_t)i + 1] = g; d_rgb[3 * (size_t)i + 2] = b;
}

// ------------------------------------------------------------------------------------------------------------------
// All-reduce (sum) over NVLink peer memory for the view-parallel gradient exchange.  Every rank holds a buffer of n floats
// mapped into all peers (symmetric memory).  Rank r owns slice r: it loads that slice from ALL ranks with 128-bit P2P
// loads, adds in rank order (so every rank computes bit-identical sums), and stores the result into ALL ranks' buffers.
// Slice r of any buffer is read and written only by rank r, and each element is read before it is written by the same
// thread, so one kernel between two cross-GPU barriers is enough (reduce-scatter + all-gather in one pass):
// per GPU (N-1)/N * n floats in and out over NVLink, vs. 2x that through a ring.
// ------------------------------------------------------------------------------------------------------------------
struct PeerPtrs {
    float* p[8];
};

__global__ void __launch_bounds__(512) peer_allreduce_kernel(PeerPtrs bufs, int rank, int world, size_t n_vec4)
{
    const size_t per = (n_vec4 + world - 1) / world;
    const size_t lo = per * rank, hi = min(n_vec4, lo + per);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    constexpr int U = 4;  // independent 128-bit peer loads in flight per thread and peer (NVLink latency ~2 us)
    for (size_t base = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; base < hi; base += stride * U) {
        float4 acc[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const size_t i = base + u * stride;
            acc[u] = i < hi ? reinterpret_cast<const float4*>(bufs.p[0])[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int r = 1; r < world; r++) {
            float4 v[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const size_t i = base + u * stride;
                v[u] = i < hi ? reinterpret_cast<const float4*>(bufs.p[r])[i] : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                acc[u].x += v[u].x; acc[u].y += v[u].y; acc[u].z += v[u].z; acc[u].w += v[u].w;
            }
        }
        for (int r = 0; r < world; r++) {
#pragma unroll
            for (int u = 0; u < U; u++) {
                const size_t i = base + u * stride;
                if (i < hi) reinterpret_cast<float4*>(bufs.p[r])[i] = acc[u];
            }
        }
    }
}

// The same all-reduce with the reduction done IN the NVSwitch (NVLS): `mc` is the multicast mapping of the symmetric buffer.
// multimem.ld_reduce returns the sum over all ranks of the addressed 16 bytes (one response crosses this GPU's link instead
// of world-1), multimem.st writes it to every rank.  Per GPU: n/world floats reduced in + n/world floats broadcast out, plus
// serving the other ranks' reads -- ~1.5x (N=4) to ~1.75x (N=8) less NVLink traffic than the peer-pointer two-shot.
__global__ void __launch_bounds__(512) multimem_allreduce_kernel(float* mc, int rank, int world, size_t n_vec4)
{
    const size_t per = (n_vec4 + world - 1) / world;
    const size_t lo = per * rank, hi = min(n_vec4, lo + per);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    constexpr int U = 4;
    for (size_t base = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; base < hi; base += stride * U) {
        float4 acc[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const size_t i = base + u * stride;
            if (i < hi)
                asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                             : "=f"(acc[u].x), "=f"(acc[u].y), "=f"(acc[u].z), "=f"(acc[u].w)
                             : "l"(reinterpret_cast<float4*>(mc) + i)
                             : "memory");
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const size_t i = base + u * stride;
            if (i < hi)
                asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(reinterpret_cast<float4*>(mc) + i),
                             "f"(acc[u].x), "f"(acc[u].y), "f"(acc[u].z), "f"(acc[u].w)
                             : "memory");
        }
    }
}

// important_score for the raw path: the activated opacity lives in conic_opacity.w (rows of culled Gaussians are unwritten)
__global__ void __launch_bounds__(256) score_from_geom_kernel(int P, const int* __restrict__ count, const float4* __restrict__ conic_opacity,
                                                              float* __restrict__ score)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int c = count[i];
    score[i] = c ? conic_opacity[i].w * (float)c : 0.f;
}

}  // namespace
