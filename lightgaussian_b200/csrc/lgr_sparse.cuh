// lgr_sparse.cuh -- sparse view-parallel gradient exchange over NVLink peer memory.
//
// Measured on the 3M-Gaussian / 1080p bench scene (scripts/exp_grad_density.py): 92 % of the Gaussians are visible in a view but only
// 12-13 % receive a NON-ZERO gradient from it -- the pixels saturate (T < 1e-4) long before the deep Gaussians are reached, and
// everything behind gets exact zeros.  The dense exchange (all-gather of dRGB 12 B/Gaussian/view + all-reduce of 44 B/Gaussian)
// therefore moves ~7x more bytes over NVLink than the gradients contain, and is what limited 8-GPU scaling to 65 %.
//
// Here every rank publishes ONE buffer in symmetric (peer-mapped) memory per step:
//     header (campos of its view, row count) | bitmap[P/32] of Gaussians with a non-zero gradient | prefix[P/32] (exclusive popcount)
//     | rows[nnz][16 floats] = dRGB(3) dxyz(3) dscaling(3) drotation(4) dopacity(1) pad(2), in ascending Gaussian order
// produced by K7+K8 run on the COMPACTED list of non-zero Gaussians (sparse_pack: flag -> scan -> index -> per-Gaussian backward with
// the activation chain rules, 13 % of the dense kernel's work).  After one cross-GPU barrier every rank runs sparse_accumulate_kernel:
// one thread per Gaussian walks the views that hold a row for it, in rank order, finds its row in view v with  prefix_v[i/32] + popc(bitmap_v[i/32] & lanes below)
// -- the bitmap word and prefix of a warp's 32 Gaussians are ONE word each per view -- loads the 64-byte row straight from the peer's
// memory (P2P loads over NVLink; no all-gather, no host-side size exchange), adds the small leaves and rebuilds the SH gradient
// basis(dir_v) (x) dRGB_v in registers, and writes every dense output row once.  All ranks add the views in the same order, so the
// summed gradients are bit-identical on every rank (replicas cannot drift).  Per rank and step the NVLink traffic is
// (world-1) * (nnz * 64 B + P/4 B) instead of (world-1) * 12 B * P + ~2 * 44 B * P.
//
// Densification statistics (view-parallel add_densification_stats, opt-in): the slot then also carries, for free or nearly so,
//   * word 14 of every row (a zero pad otherwise) = den_norm2(dL/dmeans2D) of the row's Gaussian in this view -- the same bits as the
//     local dL/dmeans2D the pack writes, and exactly what GaussianModel.add_densification_stats adds for it;
//   * vis[w32a] after the rows: bit i = radii[i] > 0 in this view (the visibility filter every training loop passes), P/8 bytes;
//   * header words 4-6: SPX_STATS_MAGIC, the host's step serial, P.
// densify_stats_exchanged_kernel then adds every rank's view to accum / denom in rank order, bit-identically on every rank.
#pragma once

namespace {

constexpr int SPX_ROW = 16;  // floats per exchanged row
constexpr int SPX_NORM = 14; // row word holding the densification norm (stats slots only)
constexpr uint32_t SPX_STATS_MAGIC = 0x53544154u;   // header word 4 of a slot packed with densification statistics

struct SparseLayout {
    size_t hdr, bitmap, prefix, rows, total;  // offsets in 4-byte words
    size_t vis, total_stats;                  // visibility bitmap of a stats slot (after the rows), and that slot's size
};
__host__ __device__ inline SparseLayout sparse_layout(int P)
{
    const size_t w32 = ((size_t)P + 31) / 32;
    const size_t w32a = (w32 + 63) / 64 * 64;
    SparseLayout l;
    l.hdr = 0;
    l.bitmap = 64;
    l.prefix = l.bitmap + w32a;
    l.rows = l.prefix + w32a;
    l.total = l.rows + (size_t)P * SPX_ROW;
    l.vis = l.total;
    l.total_stats = l.vis + w32a;
    return l;
}

// bit i of bitmap = Gaussian i is visible and its blend-backward accumulators are not all zero (=> its gradients may be non-zero);
// STATS: bit i of vis = Gaussian i is visible
template <bool STATS>
__global__ void __launch_bounds__(256) sparse_flag_kernel(int P, const int* __restrict__ radii, const float* __restrict__ acc,
                                                          uint32_t* __restrict__ bitmap, uint32_t* __restrict__ popc, uint32_t* __restrict__ vis)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    bool nz = false;
    const bool visible = i < P && radii[i] > 0;
    if (visible) {
        const float4* r = reinterpret_cast<const float4*>(acc + (size_t)i * ACC_STRIDE);
        const float4 a = r[0], b = r[1];
        const float c = acc[(size_t)i * ACC_STRIDE + 8];
        nz = a.x != 0.f || a.y != 0.f || a.z != 0.f || a.w != 0.f || b.x != 0.f || b.y != 0.f || b.z != 0.f || b.w != 0.f || c != 0.f;
    }
    const unsigned word = __ballot_sync(FULL, nz);
    unsigned vword = 0;
    if (STATS) vword = __ballot_sync(FULL, visible);
    if ((threadIdx.x & 31) == 0 && i < P) {
        bitmap[i >> 5] = word;
        popc[i >> 5] = __popc(word);
        if (STATS) vis[i >> 5] = vword;
    }
}

__global__ void __launch_bounds__(256) sparse_index_kernel(int P, const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ prefix,
                                                           int* __restrict__ idx, uint32_t* __restrict__ hdr, const float* __restrict__ campos,
                                                           int stats, uint32_t serial)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const uint32_t word = bitmap[i >> 5];
    const int lane = i & 31;
    if ((word >> lane) & 1u) idx[prefix[i >> 5] + __popc(word & ((1u << lane) - 1u))] = i;
    if (i == P - 1) {
        hdr[3] = prefix[i >> 5] + __popc(word);
        hdr[0] = __float_as_uint(campos[0]); hdr[1] = __float_as_uint(campos[1]); hdr[2] = __float_as_uint(campos[2]);
        if (stats) {
            hdr[4] = SPX_STATS_MAGIC; hdr[5] = serial; hdr[6] = (uint32_t)P;
        }
    }
}

// K7+K8 with the activation chain rules (the `vis` branch of preprocess_backward_raw_kernel, same arithmetic) for the t-th Gaussian of the
// compacted list; SH coefficients come straight from global memory (the rows are scattered, there is no contiguous run to bulk-copy)
// where a rank's packed view goes: its slot in its own exchange buffer (always) and -- push mode -- the same slot of every peer's
// buffer, written with plain stores over NVLink while the kernel computes (posted writes: no round-trip latency on the critical path,
// and the fast ranks' traffic overlaps the slow ranks' blend backward)
struct SparsePush {
    uint32_t* dst[8];  // slot base of this rank in the buffer of rank r (dst[self] = the local slot); unused entries NULL
    int n;             // number of destinations (1 = local only)
};

// header + bitmap + prefix of the local slot -> the peers' slots (small: ~P/4 bytes per peer); with statistics also the words
// [extra_off, extra_off + extra_words) (the visibility bitmap, P/8 bytes)
__global__ void __launch_bounds__(256) sparse_publish_kernel(SparsePush push, int self, size_t words, size_t extra_off, size_t extra_words)
{
    const uint32_t* src = push.dst[self];
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < words + extra_words; j += (size_t)gridDim.x * blockDim.x) {
        const size_t i = j < words ? j : extra_off + (j - words);
        const uint32_t v = src[i];
        for (int r = 0; r < push.n; r++)
            if (r != self) push.dst[r][i] = v;
    }
}

constexpr int SPK_THREADS = 128;
constexpr int SPK_ROW = 49;   // floats per staged SH row (48 + 1: conflict-free at one row per lane)

// STATS: word SPX_NORM of every row = den_norm2 of the dL/dmeans2D written for it (a zero pad otherwise)
template <bool STATS>
__global__ void __launch_bounds__(SPK_THREADS) preprocess_backward_sparse_kernel(RawBackArgs a, const int* __restrict__ idx, const uint32_t* __restrict__ hdr,
                                                                                 SparsePush push, size_t rows_off)
{
    __shared__ float s_cam[36];
    __shared__ __align__(16) float s_sh[SPK_THREADS / 32][32 * SPK_ROW];   // 6272 B per warp: a multiple of 16
    if (threadIdx.x < 16) s_cam[threadIdx.x] = a.view[threadIdx.x];
    else if (threadIdx.x < 32) s_cam[threadIdx.x] = a.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_cam[threadIdx.x] = a.campos[threadIdx.x - 32];
    __syncthreads();
    const float* view = s_cam;
    const float* proj = s_cam + 16;
    const float* cam = s_cam + 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int count = (int)hdr[3];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t - lane >= count) return;   // whole warp past the list
    const bool valid = t < count;
    const int i = valid ? idx[t] : -1;
    const size_t si = (size_t)(valid ? i : 0);
    // the SH coefficients feed only the view-direction term of dL/dmean3D (degree >= 1): the warp's 32 scattered rows are staged through
    // shared memory with row-contiguous loads (3 instructions per row, eight rows in flight) instead of 48 strided loads per lane
    float* rows = s_sh[warp];
    const int nrest_act = 3 * ((a.D + 1) * (a.D + 1) - 1);
    if (a.D > 0) {
#pragma unroll 1
        for (int r0 = 0; r0 < 32; r0 += 8) {
            float v0[8], v1[8], v2[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int ir = __shfl_sync(FULL, i, r0 + u);
                v0[u] = v1[u] = v2[u] = 0.f;
                if (ir >= 0) {
                    const float* src = a.rest + (size_t)ir * a.rest_stride;
                    if (lane < 3) v0[u] = __ldg(a.dc + (size_t)ir * 3 + lane);
                    if (lane < nrest_act) v1[u] = __ldg(src + lane);
                    if (lane + 32 < nrest_act) v2[u] = __ldg(src + 32 + lane);
                }
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                float* dst = rows + (r0 + u) * SPK_ROW;
                if (lane < 3) dst[lane] = v0[u];
                if (lane < nrest_act) dst[3 + lane] = v1[u];
                if (lane + 32 < nrest_act) dst[3 + 32 + lane] = v2[u];
            }
        }
        __syncwarp();
    }
    const float* mine = rows + lane * SPK_ROW;
    float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0, v2 = v0, v3 = v0;
    if (valid) {
        float dmean[3] = {0.f, 0.f, 0.f}, dscale[3], dq[4], dRGB[3];
        const float4 co = a.conic_opacity[si];
        const Grad2D g2 = accum_to_grad2d(a.acc + si * ACC_STRIDE, co, a.W, a.H);
        const float x = a.xyz[3 * si], y = a.xyz[3 * si + 1], z = a.xyz[3 * si + 2];
        float c3[6], dcov[6];
#pragma unroll
        for (int k = 0; k < 6; k++) c3[k] = a.cov3D[6 * si + k];
        lgr::cov2d_backward(x, y, z, view, c3, a.fx, a.fy, a.tanx, a.tany, g2.dcx, g2.dcy, g2.dcw, dcov, dmean);
        lgr::mean2d_backward(x, y, z, proj, g2.dm2x, g2.dm2y, dmean);
        const unsigned cb = a.clamped[i];
        dRGB[0] = (cb & 1u) ? 0.f : g2.dcol[0]; dRGB[1] = (cb & 2u) ? 0.f : g2.dcol[1]; dRGB[2] = (cb & 4u) ? 0.f : g2.dcol[2];
        const float s0 = act_exp(a.scaling[3 * si]), s1 = act_exp(a.scaling[3 * si + 1]), s2 = act_exp(a.scaling[3 * si + 2]);
        float dn;
        const float4 v = reinterpret_cast<const float4*>(a.rotation)[si];
        const float4 q = act_normalize(v, dn);
        float ds[3], dqn[4];
        lgr::cov3d_backward(s0, s1, s2, a.mod, q.x, q.y, q.z, q.w, dcov, ds, dqn);
        dscale[0] = ds[0] * s0; dscale[1] = ds[1] * s1; dscale[2] = ds[2] * s2;
        const float qg = q.x * dqn[0] + q.y * dqn[1] + q.z * dqn[2] + q.w * dqn[3];
        const float inv = 1.0f / dn;
        dq[0] = (dqn[0] - q.x * qg) * inv; dq[1] = (dqn[1] - q.y * qg) * inv;
        dq[2] = (dqn[2] - q.z * qg) * inv; dq[3] = (dqn[3] - q.w * qg) * inv;
        const float o = co.w;
        const float dop = (g2.dop * (1.0f - o)) * o;
        if (a.D > 0)   // view-direction term of dL/dmean3D; the SH gradient itself is rebuilt from dRGB by the accumulate kernel
            lgr::sh_backward(a.D, [&](int k) { return mine[k]; }, [](int, int, float) {}, x, y, z, cam, dRGB, dmean);
        v0 = make_float4(dRGB[0], dRGB[1], dRGB[2], dmean[0]);
        v1 = make_float4(dmean[1], dmean[2], dscale[0], dscale[1]);
        v2 = make_float4(dscale[2], dq[0], dq[1], dq[2]);
        v3 = make_float4(dq[3], dop, STATS ? lgr::den_norm2(g2.dm2x, g2.dm2y) : 0.f, 0.f);
        a.dL_dmeans2D[3 * si] = g2.dm2x; a.dL_dmeans2D[3 * si + 1] = g2.dm2y;   // dense [P,3], zero-filled by the caller; local view only
    }
    // The warp's rows are consecutive in every destination slot (row t at t * 64 bytes): they are staged in shared memory (reusing the
    // SH staging slice) and leave with ONE TMA bulk store per destination rank -- 2 KB packets over NVLink instead of 16-byte posted
    // stores (measured at 8 GPUs: the per-lane stores made this kernel 0.95 ms, 5x its 2-GPU time).
    __syncwarp();
    float4* stage = reinterpret_cast<float4*>(rows);
    stage[4 * lane + 0] = v0; stage[4 * lane + 1] = v1; stage[4 * lane + 2] = v2; stage[4 * lane + 3] = v3;
    fence_async_smem();
    __syncwarp();
    if (lane == 0) {
        const int t0 = t;                                   // lane 0's list slot
        const int nvalid = min(32, count - t0);
        for (int r = 0; r < push.n; r++)
            bulk_s2g(reinterpret_cast<float*>(push.dst[r]) + rows_off + (size_t)t0 * SPX_ROW, stage, (uint32_t)nvalid * SPX_ROW * 4u);
        bulk_commit();
        bulk_wait_read_all();
    }
}

struct SparseAccArgs {
    int P, D, M, world;
    const uint32_t* peer[8];  // each rank's exchange buffer (peer-mapped)
    const float* xyz;
    float* d_xyz;
    float* d_dc;
    float* d_rest;
    float* d_scaling;
    float* d_rotation;
    float* d_opacity;
};

__global__ void __launch_bounds__(256) sparse_accumulate_kernel(SparseAccArgs a)
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
    const SparseLayout L = sparse_layout(a.P);
    // lane v fetches view v's bitmap word, prefix and camera position for this warp's 32 Gaussians
    uint32_t my_word = 0, my_pre = 0;
    float my_cx = 0.f, my_cy = 0.f, my_cz = 0.f;
    if (lane < a.world) {
        const uint32_t* base = a.peer[lane];
        my_word = base[L.bitmap + (first >> 5)];
        my_pre = base[L.prefix + (first >> 5)];
        my_cx = __uint_as_float(base[L.hdr + 0]); my_cy = __uint_as_float(base[L.hdr + 1]); my_cz = __uint_as_float(base[L.hdr + 2]);
    }
    float x = 0.f, y = 0.f, z = 0.f;
    if (lane < n) { x = a.xyz[3 * si]; y = a.xyz[3 * si + 1]; z = a.xyz[3 * si + 2]; }
    float acc[48];
#pragma unroll
    for (int k = 0; k < 48; k++) acc[k] = 0.f;
    float gx = 0.f, gy = 0.f, gz = 0.f, gs0 = 0.f, gs1 = 0.f, gs2 = 0.f, gq0 = 0.f, gq1 = 0.f, gq2 = 0.f, gq3 = 0.f, gop = 0.f;
    // which views have a row for THIS lane's Gaussian (bit v of `views`), then every lane walks ITS OWN views in ascending order: the warp
    // runs max-popcount iterations (3-4 of 8 views at 13 % density) instead of one lock-step pass per view with 13 % of the lanes busy
    unsigned views = 0;
    for (int v = 0; v < a.world; v++) {
        const uint32_t word = __shfl_sync(FULL, my_word, v);
        if ((word >> lane) & 1u) views |= 1u << v;
    }
    const int iters = __reduce_max_sync(FULL, __popc(views));
    for (int it = 0; it < iters; it++) {
        const bool active = views != 0;
        const int v = active ? (__ffs(views) - 1) : 0;
        views &= views - 1;
        const uint32_t word = __shfl_sync(FULL, my_word, v);
        const uint32_t pre = __shfl_sync(FULL, my_pre, v);
        const float cam[3] = {__shfl_sync(FULL, my_cx, v), __shfl_sync(FULL, my_cy, v), __shfl_sync(FULL, my_cz, v)};
        if (!active) continue;
        const size_t r = (size_t)pre + __popc(word & ((1u << lane) - 1u));
        const float4* row = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.peer[v]) + L.rows + r * SPX_ROW);
        const float4 r0 = row[0], r1 = row[1], r2 = row[2], r3 = row[3];
        gx += r0.w; gy += r1.x; gz += r1.y;
        gs0 += r1.z; gs1 += r1.w; gs2 += r2.x;
        gq0 += r2.y; gq1 += r2.z; gq2 += r2.w; gq3 += r3.x;
        gop += r3.y;
        const float dRGB[3] = {r0.x, r0.y, r0.z};
        if (dRGB[0] == 0.f && dRGB[1] == 0.f && dRGB[2] == 0.f) continue;  // fully clamped in this view
        float unused[3] = {0.f, 0.f, 0.f};
        lgr::sh_backward(a.D, [&](int) { return 0.f; }, [&](int k, int c, float val) { acc[3 * k + c] += val; }, x, y, z, cam, dRGB, unused);
    }
    float* rr = s_rest + lane * nrest;
    float* dd = s_dc + lane * 3;
    if (lane < n) {
        dd[0] = acc[0]; dd[1] = acc[1]; dd[2] = acc[2];
#pragma unroll
        for (int k = 3; k < 48; k++)
            if (k - 3 < nrest) rr[k - 3] = acc[k];
        a.d_xyz[3 * si] = gx; a.d_xyz[3 * si + 1] = gy; a.d_xyz[3 * si + 2] = gz;
        a.d_scaling[3 * si] = gs0; a.d_scaling[3 * si + 1] = gs1; a.d_scaling[3 * si + 2] = gs2;
        reinterpret_cast<float4*>(a.d_rotation)[si] = make_float4(gq0, gq1, gq2, gq3);
        a.d_opacity[si] = gop;
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

// ------------------------------------------------------------------------------------------------------------------
// View-parallel add_densification_stats from the step's stats slots.  One thread per Gaussian, lane v of a warp fetches view v's bitmap
// word, prefix, visibility word and header; every thread walks the views 0..world-1 in order and, where view v saw its Gaussian, adds
// word SPX_NORM of its row (flagged) or +0.0f (visible with no row: its dL/dmeans2D is zero, so the serial call adds den_norm2(0, 0) = +0)
// to accum and 1 to denom -- the arithmetic of densify_stats_kernel called once per view in rank order.
// The same pass checks the caller against its own slot and ORs into *err:
//   SPX_ERR_HEADER  a slot without statistics, from another step (serial) or for another P: the warp adds nothing (its prefix words
//                   cannot be trusted to address rows)
//   SPX_ERR_FILTER  update_filter[i] != the published radii[i] > 0
//   SPX_ERR_GRAD    den_norm2(grad[i, 0:2]) != the published norm (0 for a visible row without one)
// ------------------------------------------------------------------------------------------------------------------
constexpr uint32_t SPX_ERR_HEADER = 1u, SPX_ERR_FILTER = 2u, SPX_ERR_GRAD = 4u;

struct DensifyExchArgs {
    int P, world, self;
    uint32_t serial;
    const uint32_t* slot[8];   // view v's slot, as the accumulate kernel reads it
    const float* grad;         // this rank's dL/dmeans2D rows
    int grad_stride;
    const uint8_t* filter;     // this rank's update filter
    float* accum;
    float* denom;
    uint32_t* err;
};

__global__ void __launch_bounds__(256) densify_stats_exchanged_kernel(DensifyExchArgs a)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int first = blockIdx.x * 256 + warp * 32;
    if (first >= a.P) return;
    const int i = first + lane;
    const bool in = i < a.P;
    const SparseLayout L = sparse_layout(a.P);
    uint32_t my_word = 0, my_pre = 0, my_vis = 0;
    unsigned long long my_base = 0;
    bool bad = false;
    if (lane < a.world) {
        const uint32_t* base = a.slot[lane];
        my_base = reinterpret_cast<unsigned long long>(base);
        bad = base[L.hdr + 4] != SPX_STATS_MAGIC || base[L.hdr + 5] != a.serial || base[L.hdr + 6] != (uint32_t)a.P;
        if (!bad) {
            my_word = base[L.bitmap + (first >> 5)];
            my_pre = base[L.prefix + (first >> 5)];
            my_vis = base[L.vis + (first >> 5)];
        }
    }
    if (__any_sync(FULL, bad)) {
        if (lane == 0) atomicOr(a.err, SPX_ERR_HEADER);
        return;
    }
    uint32_t err = 0;
    float acc = 0.f, den = 0.f;
    if (in) { acc = a.accum[i]; den = a.denom[i]; }
    const unsigned below = (1u << lane) - 1u;
    for (int v = 0; v < a.world; v++) {
        const uint32_t word = __shfl_sync(FULL, my_word, v);
        const uint32_t pre = __shfl_sync(FULL, my_pre, v);
        const uint32_t vis = __shfl_sync(FULL, my_vis, v);
        const uint32_t* base = reinterpret_cast<const uint32_t*>(__shfl_sync(FULL, my_base, v));
        if (!in) continue;
        const bool visible = (vis >> lane) & 1u, flagged = (word >> lane) & 1u;
        float nrm = 0.f;
        if (flagged) nrm = __uint_as_float(base[L.rows + ((size_t)pre + __popc(word & below)) * SPX_ROW + SPX_NORM]);
        if (visible) {
            acc = __fadd_rn(acc, nrm);
            den = __fadd_rn(den, 1.0f);
        }
        if (v == a.self) {
            if ((a.filter[i] != 0) != visible) err |= SPX_ERR_FILTER;
            const float* g = a.grad + (size_t)i * a.grad_stride;
            if (visible && __float_as_uint(lgr::den_norm2(g[0], g[1])) != __float_as_uint(nrm)) err |= SPX_ERR_GRAD;
        }
    }
    if (in) { a.accum[i] = acc; a.denom[i] = den; }
    err = __reduce_or_sync(FULL, err);
    if (lane == 0 && err) atomicOr(a.err, err);
}

// ------------------------------------------------------------------------------------------------------------------
// Single-GPU K7+K8 on the compacted list (the dense kernel spends a full warp pass on every 32 Gaussians that hold even ONE
// non-zero gradient -- 99 % of the warps at 13 % density -- and re-reads 0.7 GB of parameters for rows that come out as zeros).
//
//   zero-fill                 EVERY dense output row is cleared with TMA bulk stores from one shared page of zeros (cp.async.bulk S2G,
//                             issued by one thread; no per-lane store instructions) -- by default from inside the blend backward
//                             (lgr_blend.cuh: its producer thread clears the tile's share of the rows while the kernel, which is
//                             instruction-issue-bound and leaves HBM idle, does its work), else by kback_zero_flag_kernel<true>.
//   kback_zero_flag_kernel    one pass over the 48-byte accumulator records: flags the Gaussians with a non-zero gradient and
//                             appends their ids to a list (one atomicAdd per warp).
//   preprocess_backward_compact_kernel   K7+K8 with the activation chain rules for the listed Gaussians only (all 32 lanes busy),
//                             SH rows staged through shared memory row by row, results written over the zeros.  Grid-stride over
//                             the device-side count: no host synchronisation.
// ------------------------------------------------------------------------------------------------------------------
// DEPTH: word 9 (dL/d(depth value)) counts too, so a Gaussian whose only gradient comes from the depth plane is listed
template <bool ZERO, bool DEPTH>
__device__ __forceinline__ void kback_zero_flag_body(const KbackZeroArgs& a)
{
    __shared__ __align__(128) float zero_page[ZERO ? KB_ZERO_BYTES / 4 : 4];
    if (ZERO) {
        for (int k = threadIdx.x; k < KB_ZERO_BYTES / 4; k += 256) zero_page[k] = 0.f;
        fence_async_smem();
        __syncthreads();
    }
    const int first = blockIdx.x * 256;
    const int n = min(256, a.P - first);
    if (ZERO && threadIdx.x == 0) {
        if (n == 256) {   // every run starts 16-byte aligned and is a multiple of 16 bytes
            bulk_zero(a.d_rest + (size_t)first * a.nrest, (size_t)256 * a.nrest, zero_page);
            bulk_zero(a.d_dc + (size_t)first * 3, 768, zero_page);
            bulk_zero(a.d_xyz + (size_t)first * 3, 768, zero_page);
            bulk_zero(a.d_scaling + (size_t)first * 3, 768, zero_page);
            bulk_zero(a.d_rotation + (size_t)first * 4, 1024, zero_page);
            bulk_zero(a.d_opacity + (size_t)first, 256, zero_page);
            bulk_zero(a.dL_dmeans2D + (size_t)first * 3, 768, zero_page);
            bulk_commit();
        }
    }
    if (ZERO && n < 256) {   // ragged last block: plain stores
        for (int k = threadIdx.x; k < n * a.nrest; k += 256) a.d_rest[(size_t)first * a.nrest + k] = 0.f;
        for (int k = threadIdx.x; k < n * 3; k += 256) {
            a.d_dc[(size_t)first * 3 + k] = 0.f; a.d_xyz[(size_t)first * 3 + k] = 0.f; a.d_scaling[(size_t)first * 3 + k] = 0.f;
            a.dL_dmeans2D[(size_t)first * 3 + k] = 0.f;
        }
        for (int k = threadIdx.x; k < n * 4; k += 256) a.d_rotation[(size_t)first * 4 + k] = 0.f;
        for (int k = threadIdx.x; k < n; k += 256) a.d_opacity[(size_t)first + k] = 0.f;
    }
    const int i = first + threadIdx.x;
    bool nz = false;
    if (i < a.P && a.radii[i] > 0) {
        const float4* r = reinterpret_cast<const float4*>(a.acc + (size_t)i * ACC_STRIDE);
        const float4 u = r[0], w = r[1];
        const float c = a.acc[(size_t)i * ACC_STRIDE + 8];
        nz = u.x != 0.f || u.y != 0.f || u.z != 0.f || u.w != 0.f || w.x != 0.f || w.y != 0.f || w.z != 0.f || w.w != 0.f || c != 0.f;
        if (DEPTH) nz = nz || a.acc[(size_t)i * ACC_STRIDE + 9] != 0.f;
    }
    const unsigned word = __ballot_sync(FULL, nz);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // ONE atomicAdd per block on the list length (a per-warp atomic would queue ~90 000 updates of the same address in L2)
    __shared__ int wpop[8];
    __shared__ int block_base;
    if (lane == 0) wpop[warp] = __popc(word);
    __syncthreads();
    if (threadIdx.x == 0) {
        int tot = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) { const int c = wpop[w]; wpop[w] = tot; tot += c; }
        block_base = tot ? atomicAdd(a.counter, tot) : 0;
    }
    __syncthreads();
    if (nz) a.idx[block_base + wpop[warp] + __popc(word & ((1u << lane) - 1u))] = i;
    if (ZERO && threadIdx.x == 0 && n == 256) bulk_wait_read_all();   // the zero page must outlive the copies that read it
}

template <bool ZERO>
__global__ void __launch_bounds__(256) kback_zero_flag_kernel(KbackZeroArgs a) { kback_zero_flag_body<ZERO, false>(a); }
template <bool ZERO>
__global__ void __launch_bounds__(256) kback_zero_flag_depth_kernel(KbackZeroArgs a) { kback_zero_flag_body<ZERO, true>(a); }

constexpr int KC_THREADS = 128;   // compacted K7+K8: 4 warps per block
constexpr int KC_ROW = 49;        // floats per staged SH row (48 + 1: conflict-free at one row per lane)

// CAM: also the camera-gradient terms (lgr_raw.cuh, cam_terms); each warp adds its per-iteration sums into its own row of the shared
// cam_acc ([4][27]) across the grid-stride loop, not in 27 more registers per lane
template <bool DEPTH, bool CAM = false>
__device__ __forceinline__ void preprocess_backward_compact_body(const RawBackArgs& a, const int* __restrict__ idx, const int* __restrict__ counter,
                                                                 const RawDepth& dz, float* cam_acc = nullptr)
{
    // SH rows (48 floats per Gaussian) are scattered in memory: each warp moves its 32 rows through shared memory with row-contiguous
    // accesses (2 + 1 instructions per row) instead of 48 strided ones per lane -- 8x fewer sectors touched for the loads and the stores
    __shared__ float s_cam[36];
    __shared__ float s_sh[KC_THREADS / 32][32 * KC_ROW];
    if (threadIdx.x < 16) s_cam[threadIdx.x] = a.view[threadIdx.x];
    else if (threadIdx.x < 32) s_cam[threadIdx.x] = a.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_cam[threadIdx.x] = a.campos[threadIdx.x - 32];
    if (CAM && threadIdx.x < KC_THREADS / 32 * CAM_TERMS) cam_acc[threadIdx.x] = 0.f;
    __syncthreads();
    const float* view = s_cam;
    const float* proj = s_cam + 16;
    const float* cam = s_cam + 32;
    const int count = *counter;
    const int nrest = (a.M - 1) * 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* rows = s_sh[warp];
    const int nb = (a.D + 1) * (a.D + 1);
    const int nrest_act = 3 * (nb - 1);   // floats of the rest row that belong to active degrees
    for (int t0 = (blockIdx.x * (KC_THREADS / 32) + warp) * 32; t0 < count; t0 += gridDim.x * KC_THREADS) {
        const int t = t0 + lane;
        const bool valid = t < count;
        const int i = valid ? idx[t] : -1;
        const size_t si = (size_t)(valid ? i : 0);
        // stage the warp's SH coefficient rows (only needed for the view-direction term, degree >= 1)
        if (a.D > 0) {
#pragma unroll 1
            for (int r0 = 0; r0 < 32; r0 += 8) {   // eight rows' loads in flight, then their shared-memory stores
                float v0[8], v1[8], v2[8];
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    const int ir = __shfl_sync(FULL, i, r0 + u);
                    v0[u] = v1[u] = v2[u] = 0.f;
                    if (ir >= 0) {
                        const float* src = a.rest + (size_t)ir * a.rest_stride;
                        if (lane < 3) v0[u] = __ldg(a.dc + (size_t)ir * 3 + lane);
                        if (lane < nrest_act) v1[u] = __ldg(src + lane);
                        if (lane + 32 < nrest_act) v2[u] = __ldg(src + 32 + lane);
                    }
                }
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    float* dst = rows + (r0 + u) * KC_ROW;
                    if (lane < 3) dst[lane] = v0[u];
                    if (lane < nrest_act) dst[3 + lane] = v1[u];
                    if (lane + 32 < nrest_act) dst[3 + 32 + lane] = v2[u];
                }
            }
            __syncwarp();
        }
        float* mine = rows + lane * KC_ROW;
        float cin[CAM ? 18 : 1];   // as in preprocess_backward_raw_body
        float px = 0.f, py = 0.f, pz = 0.f;
#pragma unroll
        for (int k = 0; k < (CAM ? 18 : 1); k++) cin[k] = 0.f;
        if (valid) {
            float dmean[3] = {0.f, 0.f, 0.f}, dscale[3], dq[4], dRGB[3];
            const float4 co = a.conic_opacity[si];
            const Grad2D g2 = accum_to_grad2d(a.acc + si * ACC_STRIDE, co, a.W, a.H);
            const float x = a.xyz[3 * si], y = a.xyz[3 * si + 1], z = a.xyz[3 * si + 2];
            if (CAM) { px = x; py = y; pz = z; }
            float c3[6], dcov[6];
#pragma unroll
            for (int k = 0; k < 6; k++) c3[k] = a.cov3D[6 * si + k];
            lgr::cov2d_backward(x, y, z, view, c3, a.fx, a.fy, a.tanx, a.tany, g2.dcx, g2.dcy, g2.dcw, dcov, dmean, CAM ? cin : nullptr);
            lgr::mean2d_backward(x, y, z, proj, g2.dm2x, g2.dm2y, dmean, CAM ? cin + 12 : nullptr);
            if (DEPTH) depth_grad_to_mean(dz, a.acc + si * ACC_STRIDE, si, view, dmean);
            if (CAM && DEPTH) cin[2] += depth_grad_z(dz, a.acc + si * ACC_STRIDE, si);
            const unsigned cb = a.clamped[i];
            dRGB[0] = (cb & 1u) ? 0.f : g2.dcol[0]; dRGB[1] = (cb & 2u) ? 0.f : g2.dcol[1]; dRGB[2] = (cb & 4u) ? 0.f : g2.dcol[2];
            const float s0 = act_exp(a.scaling[3 * si]), s1 = act_exp(a.scaling[3 * si + 1]), s2 = act_exp(a.scaling[3 * si + 2]);
            float dn;
            const float4 v = reinterpret_cast<const float4*>(a.rotation)[si];
            const float4 q = act_normalize(v, dn);
            float ds[3], dqn[4];
            lgr::cov3d_backward(s0, s1, s2, a.mod, q.x, q.y, q.z, q.w, dcov, ds, dqn);
            dscale[0] = ds[0] * s0; dscale[1] = ds[1] * s1; dscale[2] = ds[2] * s2;
            const float qg = q.x * dqn[0] + q.y * dqn[1] + q.z * dqn[2] + q.w * dqn[3];
            const float inv = 1.0f / dn;
            dq[0] = (dqn[0] - q.x * qg) * inv; dq[1] = (dqn[1] - q.y * qg) * inv;
            dq[2] = (dqn[2] - q.z * qg) * inv; dq[3] = (dqn[3] - q.w * qg) * inv;
            const float o = co.w;
            const float dop = (g2.dop * (1.0f - o)) * o;
            if (a.D > 0) {   // coefficients in, gradient out, in place in the lane's staged row
                lgr::sh_backward(a.D, [&](int k) { return mine[k]; }, [&](int k, int c, float val) { mine[3 * k + c] = val; }, x, y, z, cam, dRGB, dmean,
                                 CAM ? cin + 15 : nullptr);
            } else {
#pragma unroll
                for (int c = 0; c < 3; c++) mine[c] = LGR_C0 * dRGB[c];
            }
            a.d_xyz[3 * si] = dmean[0]; a.d_xyz[3 * si + 1] = dmean[1]; a.d_xyz[3 * si + 2] = dmean[2];
            a.d_scaling[3 * si] = dscale[0]; a.d_scaling[3 * si + 1] = dscale[1]; a.d_scaling[3 * si + 2] = dscale[2];
            reinterpret_cast<float4*>(a.d_rotation)[si] = make_float4(dq[0], dq[1], dq[2], dq[3]);
            a.d_opacity[si] = dop;
            a.dL_dmeans2D[3 * si] = g2.dm2x; a.dL_dmeans2D[3 * si + 1] = g2.dm2y;
            if (a.d_rgb) {
                a.d_rgb[3 * si] = dRGB[0]; a.d_rgb[3 * si + 1] = dRGB[1]; a.d_rgb[3 * si + 2] = dRGB[2];
            }
        }
        if (CAM) {
            float t[CAM_TERMS];
            cam_terms(cin, cin + 12, cin + 15, px, py, pz, t);
            cam_warp_add(t, cam_acc + warp * CAM_TERMS, lane);
        }
        __syncwarp();
        // gradient rows out (the rows were zero-filled: only the active degrees are written)
        for (int r = 0; r < 32; r++) {
            const int ir = __shfl_sync(FULL, i, r);
            if (ir < 0) continue;
            const float* srow = rows + r * KC_ROW;
            float* dst = a.d_rest + (size_t)ir * nrest;
            if (lane < 3) a.d_dc[(size_t)ir * 3 + lane] = srow[lane];
            if (lane < nrest_act) dst[lane] = srow[3 + lane];
            if (lane + 32 < nrest_act) dst[32 + lane] = srow[3 + 32 + lane];
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(KC_THREADS) preprocess_backward_compact_kernel(RawBackArgs a, const int* __restrict__ idx, const int* __restrict__ counter)
{
    preprocess_backward_compact_body<false>(a, idx, counter, RawDepth{});
}
__global__ void __launch_bounds__(KC_THREADS) preprocess_backward_compact_depth_kernel(RawBackArgs a, const int* __restrict__ idx,
                                                                                        const int* __restrict__ counter, RawDepth dz)
{
    preprocess_backward_compact_body<true>(a, idx, counter, dz);
}
// the compacted kernels plus one camera-gradient row per block (cam_rows: [27][gridDim.x])
template <bool DEPTH>
__device__ __forceinline__ void preprocess_backward_compact_cam_body(const RawBackArgs& a, const int* __restrict__ idx, const int* __restrict__ counter,
                                                                     const RawDepth& dz, float* __restrict__ cam_rows)
{
    __shared__ float acc[KC_THREADS / 32 * CAM_TERMS];
    preprocess_backward_compact_body<DEPTH, true>(a, idx, counter, dz, acc);
    __syncthreads();
    cam_block_row(acc, KC_THREADS / 32, cam_rows);
}
__global__ void __launch_bounds__(KC_THREADS) preprocess_backward_compact_cam_kernel(RawBackArgs a, const int* __restrict__ idx,
                                                                                      const int* __restrict__ counter, float* __restrict__ cam_rows)
{
    preprocess_backward_compact_cam_body<false>(a, idx, counter, RawDepth{}, cam_rows);
}
__global__ void __launch_bounds__(KC_THREADS) preprocess_backward_compact_depth_cam_kernel(RawBackArgs a, const int* __restrict__ idx,
                                                                                            const int* __restrict__ counter, RawDepth dz,
                                                                                            float* __restrict__ cam_rows)
{
    preprocess_backward_compact_cam_body<true>(a, idx, counter, dz, cam_rows);
}

}  // namespace
