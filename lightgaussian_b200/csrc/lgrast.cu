// lgrast.cu -- sm_90a kernels and the C-ABI (include/lgrast.h) of the H100 rasterizer.
//
// Pipeline per view (reference call order: RAST/cuda_rasterizer/rasterizer_impl.cu:198-337):
//
//   preprocess_kernel     per Gaussian: cull, EWA projection, SH->RGB, tile rectangle        (K1)
//   depth sort            CUB radix sort of P 32-bit depth keys                               (replaces part of L2)
//   scan                  CUB inclusive sum of tiles_touched in depth order                   (L1)
//   emit_kernel           one (tile, id) instance per overlapped tile, in depth order          (K2)
//   tile sort             CUB radix sort on the <=16-bit tile key only (2 passes, stable)     (replaces L2)
//   ranges_kernel         per-tile [start,end)                                                 (K3)
//   blend_forward_kernel  one warp per 8x4 pixel sub-tile, lane-parallel exact culling         (K4/K5)
//
// The reference sorts R (tile<<32|depth) 64-bit keys in ~6 radix passes.  Sorting the P Gaussians by
// depth once and then stably bucketing the R instances by tile gives the IDENTICAL order (tile, depth
// bits, ascending id) with ~6x less sort traffic.
//
// Backward (RAST/cuda_rasterizer/rasterizer_impl.cu:341-435):
//   blend_backward_kernel       back-to-front re-walk, butterfly warp reduction, 9 atomics per
//                               (warp, Gaussian) instead of 9 per (pixel, Gaussian)              (K6)
//   preprocess_backward_kernel  conic/mean2D/colour gradients -> all dense per-Gaussian outputs  (K7+K8 fused)
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>
#include <thrust/iterator/counting_iterator.h>
#include <cfloat>
#include <cmath>
#include <algorithm>
#include <atomic>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/lgrast.h"
#include "lgr_math.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int LGR_SMS = 132;    // streaming multiprocessors of an H100 SXM: grid sizes of the grid-stride kernels
constexpr int ACC_STRIDE = 12;  // floats per Gaussian in the backward accumulator record
constexpr int DET_ROW = 9;      // floats per partial row of the deterministic blend backward: the record without its pad
// record layout: 0..2 dL/dcolor rgb | 3 S0 | 4,5 S1x,S1y | 6,7,8 S2xx,S2xy,S2yy | 9..11 pad
// with w = G * dL/dalpha per (pixel, Gaussian) pair and d = mean2D - pixel:  S0 = sum w, S1 = sum w*d, S2 = sum w*d*d^T.
// The per-Gaussian factors (conic, opacity, viewport) are applied once per Gaussian in K8 (accum_to_grad2d).

thread_local std::string g_last_error;
int g_blend_mode = 0;   // 0 = ring kernels (lgr_blend.cuh), 1 = round-1 kernels (kept for A/B measurements and as a cross-check in the tests)
// binning: 2 = library radix sorts + scan, binning blob sized from a running estimate, no GPU idle on the host (default: the fastest path
// measured, DESIGN.md section 4; deterministic mode sizes the blob exactly after a host synchronisation); 0 = hand-written kernels
// (lgr_bin.cuh), the same estimate (0.76 ms: correct and library-free, but its serial tile-ranking warp is slower than two library radix
// passes -- DESIGN.md section 9); 1 = hand-written kernels, blob sized exactly after a stream synchronisation
int g_bin_mode = 2;
std::atomic<size_t> g_bin_hint{0};   // running estimate of the listed instances per view (modes 0 and 2)
int g_vq_mode = 0;      // VecTree nearest-code search: 0 = tensor-core coarse pass + exact FP32 rescore (d <= 32), 1 = FP32 FFMA kernel only
// deterministic mode (lgr_set_deterministic): fixed-order reductions in place of the float atomics of the blend backward and the VecTree
// accumulation; needs library binning and the ring blend kernels
int g_det = 0;
int g_kback_mode = 0;   // single-GPU K7+K8: 0 = rows cleared inside the blend backward + compacted list (lgr_sparse.cuh), 1 = dense kernel, 2 = separate zero-fill kernel + compacted list (A/B)
std::atomic<uint64_t> g_launches{0};

// ---- optional per-stage device timing (CUDA events on the launch stream), used by bench.py's roofline ----
enum StageId { ST_PREPROCESS = 0, ST_DEPTH_SORT, ST_SCAN, ST_EMIT, ST_TILE_SORT, ST_RANGES, ST_BLEND_FWD, ST_BLEND_FWD_COUNT,
               ST_SCORE, ST_BLEND_BWD, ST_PREPROCESS_BWD, ST_MEMSET, ST_SH_GRAD, ST_PEER_ALLREDUCE, ST_LOSS_FWD, ST_LOSS_BWD, ST_ADAMW, ST_COMPACT, ST_VQ_ASSIGN, ST_VQ_UPDATE, ST_SPARSE_PACK, ST_SPARSE_ACC, ST_BIN_DSORT, ST_BIN_COUNT, ST_BIN_SCATTER, ST_DET_GATHER, ST_ADAMW_SELECTIVE, ST_CAMERA_FINISH, ST_COUNT };
const char* const kStageNames[ST_COUNT] = {"preprocess_kernel", "depth_sort(cub)", "scan(cub)", "emit_kernel", "tile_sort(cub)",
                                           "ranges_kernel", "blend_forward_kernel", "blend_forward_kernel<count>", "score_kernel",
                                           "blend_backward_kernel", "preprocess_backward_kernel", "memset", "sh_grad_from_views_kernel",
                                           "peer_allreduce_kernel", "image_loss_forward_kernel", "image_loss_backward_kernel", "adamw_multi_kernel",
                                           "compact_gather_kernel", "vq_assign_kernel", "vq_ema_kernels", "sparse_pack(flag+scan+index+K8)",
                                           "sparse_accumulate_kernel", "depth_sort(dsort_count+bin_scan+dsort_scatter x3)", "tile_count_kernel+bin_scan_kernel",
                                           "tile_scatter_kernel", "det_gather_kernel", "adamw_selective_kernel",
                                           "camera_grad_finish_kernel"};
struct ProfRecord { int stage; cudaEvent_t a, b; };
bool g_prof_on = false;
std::vector<ProfRecord> g_prof_records;
std::vector<cudaEvent_t> g_prof_pool;
double g_prof_ms[ST_COUNT] = {0};
uint64_t g_prof_n[ST_COUNT] = {0};
std::mutex g_prof_mutex;

cudaEvent_t prof_event()
{
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
struct ProfScope {
    int stage; cudaStream_t s; cudaEvent_t a = nullptr, b = nullptr; bool on;
    ProfScope(int stage_, cudaStream_t s_) : stage(stage_), s(s_), on(g_prof_on)
    {
        if (on) { std::lock_guard<std::mutex> l(g_prof_mutex); a = prof_event(); b = prof_event(); cudaEventRecord(a, s); }
    }
    ~ProfScope()
    {
        if (on) { cudaEventRecord(b, s); std::lock_guard<std::mutex> l(g_prof_mutex); g_prof_records.push_back({stage, a, b}); }
    }
};

#define LGR_CUDA_TRY(expr)                                                                          \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            g_last_error = std::string(#expr) + ": " + cudaGetErrorString(_e);                      \
            return LGR_ERR_CUDA;                                                                    \
        }                                                                                           \
    } while (0)

#define LGR_LAUNCH_CHECK(name, debug, stream)                                                       \
    do {                                                                                            \
        g_launches.fetch_add(1, std::memory_order_relaxed);                                         \
        cudaError_t _e = cudaGetLastError();                                                        \
        if (_e == cudaSuccess && (debug)) _e = cudaStreamSynchronize(stream);                       \
        if (_e != cudaSuccess) {                                                                    \
            g_last_error = std::string(name) + ": " + cudaGetErrorString(_e);                       \
            return LGR_ERR_CUDA;                                                                    \
        }                                                                                           \
    } while (0)

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace
#include "lgr_bin.cuh"
namespace {

// Sub-allocation of one opaque blob (the role of obtain()/required() in
// RAST/cuda_rasterizer/rasterizer_impl.h:21-73).  With base == nullptr it only measures.
struct Carver {
    char* base;
    size_t off = 0;
    explicit Carver(char* b) : base(b) {}
    template <typename T>
    T* take(size_t count, size_t* offset_out = nullptr)
    {
        off = align_up(off, 256);
        if (offset_out) *offset_out = off;
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * sizeof(T);
        return p;
    }
};

struct GeometryState {
    float* depth;              // [P] view-space z (valid where radii > 0)
    float2* means2D;           // [P]
    float4* conic_opacity;     // [P]
    float4* rgb;               // [P] xyz = colour fed to the blend
    float* cov3D;              // [6P]
    uint8_t* clamped;          // [P] bit c = channel c clamped
    uint32_t* tiles_touched;   // [P] tile-rectangle area (the reference's definition)
    uint32_t* sorted_ids;      // [P] Gaussian ids in (depth bits, id) order; culled ones last
    float* grad_acc;           // [12P] backward accumulator records
    // forward-only binning scratch.  Hand-written binning (g_bin_mode 0/1): aliased INSIDE the grad_acc region (dead before the
    // backward clears it): bin_rec, depth_keys, depth_keys_sorted, iota (= second id buffer of the depth sort).
    uint4* bin_rec;            // [P] tile rectangle + exact 64-bit keep mask (lgr_bin.cuh); NULL on the library path
    uint32_t* depth_keys;      // [P]
    uint32_t* depth_keys_sorted;  // [P]
    uint32_t* iota;            // [P]
    // library path only (g_bin_mode 2), behind grad_acc
    uint32_t* tiles_kept;      // [P] instances actually emitted after exact tile culling (<= tiles_touched)
    unsigned long long* keep_mask;  // [P] bit b set = rectangle tile b (row-major) is kept; all ones when the rectangle has > 64 tiles
    unsigned long long* offsets;  // [P] inclusive scan in sorted order: low word kept instances, high word rectangle areas
    int* num_rendered;         // header (64 ints): [0] instances listed, [1] the reference's num_rendered (sum of tiles_touched),
                               //   [2] capacity of the binning blob, [3] capacity overflow flag, [8] scan kernels' arrival counter
    char* cub_temp;
    size_t cub_temp_bytes;
    size_t offs[8];
    size_t total;
};

// scan input in depth order: low 32 bits = instances kept, high 32 bits = tile-rectangle area, so ONE inclusive scan yields
// the emit offsets (low) and the reference's num_rendered (high word of the last element)
struct TilesTouchedOp {
    const uint32_t* kept;
    const uint32_t* touched;
    __host__ __device__ __forceinline__ unsigned long long operator()(const uint32_t& id) const
    {
        return (unsigned long long)kept[id] | ((unsigned long long)touched[id] << 32);
    }
};

// The part the backward reads (everything up to and including grad_acc) has the same layout in every binning mode.
GeometryState carve_geometry(char* base, size_t P, bool library_binning)
{
    GeometryState g;
    Carver c(base);
    g.num_rendered = c.take<int>(64);
    g.depth = c.take<float>(P, &g.offs[0]);
    g.means2D = c.take<float2>(P, &g.offs[1]);
    g.conic_opacity = c.take<float4>(P, &g.offs[2]);
    g.rgb = c.take<float4>(P, &g.offs[3]);
    g.cov3D = c.take<float>(6 * P, &g.offs[4]);
    g.clamped = c.take<uint8_t>(P, &g.offs[5]);
    g.tiles_touched = c.take<uint32_t>(P, &g.offs[6]);
    g.sorted_ids = c.take<uint32_t>(P, &g.offs[7]);
    const size_t acc_bytes = sizeof(float) * ACC_STRIDE * P, scratch_bytes = 28 * P + 4 * 256;
    size_t acc_off = 0;
    char* region = c.take<char>(std::max(acc_bytes, scratch_bytes), &acc_off);
    g.grad_acc = reinterpret_cast<float*>(region);
    g.bin_rec = nullptr;
    g.tiles_kept = nullptr; g.keep_mask = nullptr; g.offsets = nullptr;
    g.cub_temp = nullptr; g.cub_temp_bytes = 0;
    if (!library_binning) {
        Carver a(region);   // aliases grad_acc
        g.bin_rec = a.take<uint4>(P);
        g.depth_keys = a.take<uint32_t>(P);
        g.depth_keys_sorted = a.take<uint32_t>(P);
        g.iota = a.take<uint32_t>(P);
    } else {
        g.tiles_kept = c.take<uint32_t>(P);
        g.keep_mask = c.take<unsigned long long>(P);
        g.depth_keys = c.take<uint32_t>(P);
        g.depth_keys_sorted = c.take<uint32_t>(P);
        g.iota = c.take<uint32_t>(P);
        g.offsets = c.take<unsigned long long>(P);
        size_t sort_bytes = 0, scan_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, (int)P, 0, 32);
        auto it = thrust::make_transform_iterator((const uint32_t*)nullptr, TilesTouchedOp{nullptr, nullptr});
        cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, it, (unsigned long long*)nullptr, (int)P);
        g.cub_temp_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
        g.cub_temp = c.take<char>(g.cub_temp_bytes);
    }
    g.total = align_up(c.off, 256);
    return g;
}

struct ImageState {
    float* final_T;       // [N]
    uint32_t* n_contrib;  // [N]
    uint2* ranges;        // [tiles]
    // forward-only scratch of the hand-written binning (lgr_bin.cuh); NULL on the library path
    uint32_t* bin_M;      // [BIN_V][max(DS_BINS, tiles_pad)] count matrix
    uint32_t* bin_total;  // [max(DS_BINS, tiles_pad)]
    uint32_t* bin_base;   // [max(DS_BINS, tiles_pad)]
    size_t offs[3];
    size_t total;
};

// the part the backward reads (final_T, n_contrib, ranges) has the same layout in every binning mode
ImageState carve_image(char* base, int W, int H, bool library_binning)
{
    ImageState s;
    const size_t N = (size_t)W * H;
    const size_t tiles = (size_t)((W + LGR_TILE - 1) / LGR_TILE) * ((H + LGR_TILE - 1) / LGR_TILE);
    Carver c(base);
    s.final_T = c.take<float>(N, &s.offs[0]);
    s.n_contrib = c.take<uint32_t>(N, &s.offs[1]);
    s.ranges = c.take<uint2>(tiles, &s.offs[2]);
    s.bin_M = s.bin_total = s.bin_base = nullptr;
    if (!library_binning) {
        const size_t pad = std::max((size_t)DS_BINS, (size_t)bin_pad((int)tiles));
        s.bin_M = c.take<uint32_t>((size_t)BIN_V * pad);
        s.bin_total = c.take<uint32_t>(pad);
        s.bin_base = c.take<uint32_t>(pad);
    }
    s.total = align_up(c.off, 256);
    return s;
}

// bits of the tile sort's keys: 2^bits > tiles, so that the pad key (all ones, emit_kernel) lies strictly above every tile index
inline int tile_key_bits(int W, int H)
{
    const uint32_t tiles = (uint32_t)((W + LGR_TILE - 1) / LGR_TILE) * ((H + LGR_TILE - 1) / LGR_TILE);
    int bits = 1;
    while ((1u << bits) <= tiles) bits++;
    return bits;
}

struct BinningState {
    uint32_t* point_list;       // [R] sorted ids
    uint32_t* ids_unsorted;     // [R]
    void* keys_unsorted;        // [R] u16 or u32 tile index
    void* keys_sorted;          // [R]
    char* cub_temp;
    size_t cub_temp_bytes;
    float* records;             // [R][12] per-instance records in list order, written by the forward blend for the chunks it visits
    float* det_partial;         // deterministic mode: [R][9] partial rows by unsorted index (forward: [R] sorted -> unsorted permutation)
    uint32_t* det_reached;      // deterministic mode: [ceil(R/32)] bit u = the backward wrote partial row u
    bool wide_keys;
    size_t offs[1];
    size_t total;
};

// R = instances the blob holds: the listed count on the library path and in mode 1, the capacity estimate in mode 0
// det (deterministic mode, library binning only): the per-instance partial rows of the backward ([R][9] floats, which hold the sort's
// permutation during the forward) and a bitmap of the instances the backward reached follow the records; det_*_offset (lgr_blend.cuh)
// recompute these offsets on the device
BinningState carve_binning(char* base, size_t R, int W, int H, bool library_binning, bool det = false)
{
    BinningState b;
    const int bits = tile_key_bits(W, H);
    b.wide_keys = bits > 16;
    const size_t Rn = R ? R : 1;
    Carver c(base);
    b.point_list = c.take<uint32_t>(Rn, &b.offs[0]);
    b.records = c.take<float>(Rn * 12);   // second region: its offset, align_up(4*max(R,1), 256), is recomputed ON THE DEVICE by the backward
    b.ids_unsorted = nullptr; b.keys_unsorted = b.keys_sorted = nullptr; b.cub_temp = nullptr; b.cub_temp_bytes = 0;
    b.det_partial = nullptr; b.det_reached = nullptr;
    if (!library_binning) {
        b.total = align_up(c.off, 256);
        return b;
    }
    if (det) {
        b.det_partial = c.take<float>(Rn * DET_ROW);
        b.det_reached = c.take<uint32_t>((Rn + 31) / 32);
    }
    b.ids_unsorted = c.take<uint32_t>(Rn);
    const size_t ksz = b.wide_keys ? 4 : 2;
    b.keys_unsorted = c.take<char>(Rn * ksz);
    b.keys_sorted = c.take<char>(Rn * ksz);
    size_t bytes = 0;
    if (b.wide_keys)
        cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, (int)Rn, 0, bits);
    else
        cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint16_t*)nullptr, (uint16_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, (int)Rn, 0, bits);
    b.cub_temp_bytes = bytes;
    b.cub_temp = c.take<char>(bytes);
    b.total = align_up(c.off, 256);
    return b;
}

// ------------------------------------------------------------------------------------------------
// Exact, conservative sub-tile culling.  Returns true when NO pixel centre in [rx0,rx1]x[ry0,ry1] can
// reach alpha >= 1/255 for this Gaussian, i.e. when the reference would skip every pair at
// RAST/cuda_rasterizer/forward.cu:345-347.  The margins are lgr::rect_culled's (DESIGN.md section 4).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool subtile_cull(float gxp, float gyp, float4 co, float rx0, float rx1, float ry0, float ry1)
{
    const float A = co.x, B = co.y, Cc = co.z;
    const float t = 257.55f * co.w;  // 255 * 1.01 * opacity
    if (t <= 1.0f) return true;      // alpha <= opacity < 1/255 everywhere
    if (!(A > 0.f && Cc > 0.f && A * Cc - B * B > 0.f)) return false;  // not positive definite: never cull
    return lgr::rect_culled(0.5f * A, 0.5f * Cc, B, __fdividef(-B, A), __fdividef(-B, Cc), __logf(t), gxp - rx1, gxp - rx0, gyp - ry1,
                            gyp - ry0);
}

// Exact tile-level culling at binning time: tile b of a Gaussian's rectangle is dropped when no pixel centre inside
// it can reach alpha >= 1/255 -- every (pixel, Gaussian) pair of such an instance is skipped by the reference
// (forward.cu:345-347), so the image is unchanged while the instance list, its sort and the per-tile walks shrink.
// Rectangles above 64 tiles (huge splats) are kept whole.
__device__ bool g_tile_cull_enabled = true;

__device__ __forceinline__ void tile_keep_mask(const lgr::Geom& geo, float4 co, int W, int H, unsigned long long& mask, uint32_t& kept)
{
    const int w = geo.rect.x1 - geo.rect.x0, h = geo.rect.y1 - geo.rect.y0;
    const int area = w * h;
    mask = ~0ull;
    kept = (uint32_t)area;
    if (area > 64) return;
    if (area < 64) mask = (1ull << area) - 1ull;   // bits >= area stay clear: popcount(mask) = instances listed
    if (!g_tile_cull_enabled) return;
    // lgr::rect_culled per tile, with everything that does not depend on the tile hoisted out of the loop
    const float A = co.x, B = co.y, Cc = co.z;
    const float t = 257.55f * co.w;
    if (t <= 1.0f) {  // alpha <= opacity < 1/255 everywhere: the Gaussian is listed nowhere
        mask = 0ull;
        kept = 0;
        return;
    }
    if (!(A > 0.f && Cc > 0.f && A * Cc - B * B > 0.f)) return;
    const float thr = __logf(t);
    const float nbc = __fdividef(-B, Cc), nba = __fdividef(-B, A), hA = 0.5f * A, hC = 0.5f * Cc;
    unsigned long long m = 0ull;
    int b = 0;
    for (int ty = geo.rect.y0; ty < geo.rect.y1; ty++) {
        const float dy_lo = geo.py - (float)min(ty * LGR_TILE + LGR_TILE - 1, H - 1), dy_hi = geo.py - (float)(ty * LGR_TILE);
        for (int tx = geo.rect.x0; tx < geo.rect.x1; tx++, b++) {
            const float dx_lo = geo.px - (float)min(tx * LGR_TILE + LGR_TILE - 1, W - 1), dx_hi = geo.px - (float)(tx * LGR_TILE);
            if (!lgr::rect_culled(hA, hC, B, nba, nbc, thr, dx_lo, dx_hi, dy_lo, dy_hi)) m |= 1ull << b;
        }
    }
    mask = m;
    kept = (uint32_t)__popcll(m);
}

// The same mask for the 32 Gaussians of a warp, evaluated warp-cooperatively: the (Gaussian, tile) candidates of the warp are laid
// out back to back, lane L tests candidates L, L+32, ... (owner found with a 5-step shuffle search, its hoisted coefficients fetched by
// shuffle), one ballot per step returns the keep bits and every owner cuts its own bits out of it.  ~6 steps per warp instead of a
// per-lane loop as long as the largest rectangle in the warp (thread efficiency 17/32 in the per-lane version, profiles/r01c).
// All 32 lanes must call it; `visible` lanes get their mask, the others 0.  Same arithmetic as tile_keep_mask() => same masks.
__device__ __forceinline__ unsigned long long warp_tile_keep_mask(bool visible, const lgr::Geom& geo, float4 co, int W, int H, int lane)
{
    const int w = visible ? geo.rect.x1 - geo.rect.x0 : 0, h = visible ? geo.rect.y1 - geo.rect.y0 : 0;
    const int area = w * h;
    unsigned long long mask = area >= 64 ? ~0ull : ((1ull << area) - 1ull);
    const float A = co.x, B = co.y, Cc = co.z;
    const float t = 257.55f * co.w;
    uint32_t need = 0;
    if (visible && area <= 64 && g_tile_cull_enabled) {
        if (t <= 1.0f) mask = 0ull;
        else if (A > 0.f && Cc > 0.f && A * Cc - B * B > 0.f) need = (uint32_t)area;
    }
    uint32_t incl = need;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += v;
    }
    const uint32_t off = incl - need, total = __shfl_sync(FULL, incl, 31);
    if (total == 0) return mask;
    const float thr = __logf(fmaxf(t, 1.0f));
    const float nbc = __fdividef(-B, Cc), nba = __fdividef(-B, A), hA = 0.5f * A, hC = 0.5f * Cc;
    // the rectangle's origin and width travel unpacked, so any tile index works; idle lanes get width 1 (never a division by 0)
    const int x0 = visible ? geo.rect.x0 : 0, y0 = visible ? geo.rect.y0 : 0, width = visible ? w : 1;
    const float px = visible ? geo.px : 0.f, py = visible ? geo.py : 0.f;
    unsigned long long kept = 0ull;
    for (uint32_t base = 0; base < total; base += 32) {
        const uint32_t j = base + lane;
        int lo = 0, hi = 31;   // largest lane m with off[m] <= j
#pragma unroll
        for (int it = 0; it < 5; it++) {
            const int mid = (lo + hi + 1) >> 1;
            const uint32_t v = __shfl_sync(FULL, off, mid);
            if (v <= j) lo = mid;
            else hi = mid - 1;
        }
        const uint32_t o_off = __shfl_sync(FULL, off, lo);
        const int o_x0 = __shfl_sync(FULL, x0, lo), o_y0 = __shfl_sync(FULL, y0, lo), o_w = __shfl_sync(FULL, width, lo);
        const float o_px = __shfl_sync(FULL, px, lo), o_py = __shfl_sync(FULL, py, lo);
        const float o_hA = __shfl_sync(FULL, hA, lo), o_hC = __shfl_sync(FULL, hC, lo), o_B = __shfl_sync(FULL, B, lo);
        const float o_nbc = __shfl_sync(FULL, nbc, lo), o_nba = __shfl_sync(FULL, nba, lo), o_thr = __shfl_sync(FULL, thr, lo);
        bool keep = false;
        if (j < total) {
            const int local = (int)(j - o_off);
            const int ry = (int)__fdividef((float)local + 0.5f, (float)o_w), rx = local - ry * o_w;
            const int tx = o_x0 + rx, ty = o_y0 + ry;
            const float dy_lo = o_py - (float)min(ty * LGR_TILE + LGR_TILE - 1, H - 1), dy_hi = o_py - (float)(ty * LGR_TILE);
            const float dx_lo = o_px - (float)min(tx * LGR_TILE + LGR_TILE - 1, W - 1), dx_hi = o_px - (float)(tx * LGR_TILE);
            keep = !lgr::rect_culled(o_hA, o_hC, o_B, o_nba, o_nbc, o_thr, dx_lo, dx_hi, dy_lo, dy_hi);
        }
        const unsigned bal = __ballot_sync(FULL, keep);
        // my candidates inside [base, base + 32)
        const uint32_t s0 = max(off, base), s1 = min(off + need, base + 32u);
        if (s0 < s1) {
            const uint32_t len = s1 - s0;
            const uint32_t seg = (bal >> (s0 - base)) & (len == 32u ? 0xffffffffu : ((1u << len) - 1u));
            kept |= (unsigned long long)seg << (s0 - off);
        }
    }
    return need ? kept : mask;
}

// ------------------------------------------------------------------------------------------------
// K1  preprocess
// ------------------------------------------------------------------------------------------------
struct PreprocessArgs {
    int P, D, M, W, H, gx, gy;
    float fx, fy, tanx, tany, mod;
    const float* means3D;
    const float* scales;
    const float* rotations;
    const float* opacities;
    const float* shs;
    const float* cov3D_precomp;
    const float* colors_precomp;
    const float* view;
    const float* proj;
    const float* campos;
    int prefiltered;
};

__global__ void __launch_bounds__(256) preprocess_kernel(PreprocessArgs a, int* __restrict__ radii, GeometryState g)
{
    __shared__ float s_cam[36];  // view 16 | proj 16 | campos 3
    if (threadIdx.x < 16) s_cam[threadIdx.x] = a.view[threadIdx.x];
    else if (threadIdx.x < 32) s_cam[threadIdx.x] = a.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_cam[threadIdx.x] = a.campos[threadIdx.x - 32];
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    const float* view = s_cam;
    const float* proj = s_cam + 16;
    const float* cam = s_cam + 32;

    const float x = a.means3D[3 * i], y = a.means3D[3 * i + 1], z = a.means3D[3 * i + 2];
    float cov[6];
    bool have_cov = false;
    // the cull test needs only the position; do it before touching scale/rot
    const float depth0 = lgr::xform_row(view, 2, x, y, z);
    bool visible = depth0 > 0.2f;
    lgr::Geom geo;
    if (visible) {
        if (a.cov3D_precomp) {
#pragma unroll
            for (int k = 0; k < 6; k++) cov[k] = a.cov3D_precomp[6 * (size_t)i + k];
        } else {
            const float4 q = reinterpret_cast<const float4*>(a.rotations)[i];
            lgr::cov3d_from_scale_rot(a.scales[3 * i], a.scales[3 * i + 1], a.scales[3 * i + 2], a.mod, q.x, q.y, q.z, q.w, cov);
            have_cov = true;
        }
        visible = lgr::project_gaussian(x, y, z, view, proj, cov, a.fx, a.fy, a.tanx, a.tany, a.W, a.H, a.gx, a.gy, geo);
    } else if (a.prefiltered) {
        printf("Point is filtered although prefiltered is set. This shouldn't happen!");
        __trap();
    }
    if (!g.bin_rec) g.iota[i] = (uint32_t)i;
    if (have_cov) {  // the reference stores cov3D before the later culls (forward.cu:213)
#pragma unroll
        for (int k = 0; k < 6; k++) g.cov3D[6 * (size_t)i + k] = cov[k];
    }
    if (!visible) {
        radii[i] = 0;
        g.tiles_touched[i] = 0;
        if (g.bin_rec) g.bin_rec[i] = make_uint4(0u, 0u, 0u, 0u);
        else g.tiles_kept[i] = 0;
        g.depth_keys[i] = 0xffffffffu;
        g.clamped[i] = 0;
        return;
    }
    float rgb[3];
    unsigned clamp_bits = 0;
    if (a.colors_precomp) {
        rgb[0] = a.colors_precomp[3 * (size_t)i];
        rgb[1] = a.colors_precomp[3 * (size_t)i + 1];
        rgb[2] = a.colors_precomp[3 * (size_t)i + 2];
    } else {
        const float* sh = a.shs + (size_t)i * a.M * 3;
        if (a.M == 16) {  // 192 B per Gaussian, 16 B aligned: 128-bit loads of the active prefix only
            float v[48];
            const int nfl = 3 * (a.D + 1) * (a.D + 1);
            const float4* s4 = reinterpret_cast<const float4*>(sh);
#pragma unroll
            for (int j = 0; j < 12; j++) {
                float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
                if (4 * j < nfl) t = __ldg(s4 + j);
                v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
            }
            lgr::sh_to_rgb(a.D, [&](int k) { return v[k]; }, x, y, z, cam, rgb, clamp_bits);
        } else {
            lgr::sh_to_rgb(a.D, [&](int k) { return __ldg(sh + k); }, x, y, z, cam, rgb, clamp_bits);
        }
    }
    radii[i] = geo.radius;
    g.depth[i] = geo.depth;
    g.depth_keys[i] = __float_as_uint(geo.depth);
    g.means2D[i] = make_float2(geo.px, geo.py);
    g.conic_opacity[i] = make_float4(geo.conic_x, geo.conic_y, geo.conic_z, a.opacities[i]);
    g.rgb[i] = make_float4(rgb[0], rgb[1], rgb[2], 0.f);
    g.clamped[i] = (uint8_t)clamp_bits;
    const uint32_t area = (uint32_t)((geo.rect.y1 - geo.rect.y0) * (geo.rect.x1 - geo.rect.x0));
    g.tiles_touched[i] = area;
    unsigned long long mask;
    uint32_t kept;
    tile_keep_mask(geo, make_float4(geo.conic_x, geo.conic_y, geo.conic_z, a.opacities[i]), a.W, a.H, mask, kept);
    if (g.bin_rec) {
        g.bin_rec[i] = make_bin_rec(geo.rect.x0, geo.rect.y0, geo.rect.x1 - geo.rect.x0, geo.rect.y1 - geo.rect.y0, mask);
    } else {
        g.tiles_kept[i] = kept;
        g.keep_mask[i] = mask;
    }
}

// ------------------------------------------------------------------------------------------------
// K2  emit (tile, id) instances in depth order     (RAST/cuda_rasterizer/rasterizer_impl.cu:70-111)
// ------------------------------------------------------------------------------------------------
// Warp-cooperative: the 32 Gaussians of a warp own one contiguous span of the instance list; lane L writes
// instances span_begin+L, +32, ... and finds each instance's owner with a 5-step shuffle binary search over the
// warp's run offsets, so key/id stores are fully coalesced whatever the splat sizes are (the reference's one thread
// per Gaussian loop is serial in the splat area, rasterizer_impl.cu:98-109).
// The blob holds `capacity` instances, sized before the count R was known: instances at or past it are not written and R > capacity
// raises HDR_OVERFLOW (the host repeats with an exact blob); slots [R, capacity) get the pad key ~0, which lies above every tile index
// in the sort's key bits (tile_key_bits), so the pads sort last and no range reaches them.
template <typename KeyT>
__global__ void __launch_bounds__(256) emit_kernel(int P, const uint32_t* __restrict__ sorted_ids, const unsigned long long* __restrict__ offsets,
                                                   const unsigned long long* __restrict__ keep_mask, const float2* __restrict__ means2D,
                                                   const int* __restrict__ radii, int gx, int gy, uint32_t capacity, KeyT* __restrict__ keys,
                                                   uint32_t* __restrict__ ids, int* __restrict__ header)
{
    const int lane = threadIdx.x & 31;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t id = 0, cnt = 0, off = 0;
    int x0 = 0, y0 = 0, w = 1;
    unsigned long long mask = ~0ull;
    if (k < P) {
        // low word of the inclusive scan = kept instances up to and including k: the count comes from two adjacent (coalesced) scan
        // words rather than a gather of tiles_kept by id, and Gaussians listed nowhere gather nothing
        off = k > 0 ? (uint32_t)offsets[k - 1] : 0u;
        cnt = (uint32_t)offsets[k] - off;
        if (cnt) {
            id = sorted_ids[k];
            const float2 p = means2D[id];
            const lgr::TileRect r = lgr::tile_rect(p.x, p.y, radii[id], gx, gy);
            x0 = r.x0; y0 = r.y0; w = r.x1 - r.x0;
            mask = keep_mask[id];
        }
    }
    // lanes past P inherit the running offset so that `off` stays non-decreasing across the warp
    const uint32_t end_mine = off + cnt;
    uint32_t run_end = end_mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(FULL, run_end, d);
        if (lane >= d) run_end = max(run_end, t);
    }
    if (k >= P) off = run_end;
    const uint32_t span_begin = __shfl_sync(FULL, off, 0);
    const uint32_t span_end = min(__shfl_sync(FULL, run_end, 31), capacity);
    for (uint32_t base = span_begin; base < span_end; base += 32) {
        const uint32_t j = base + lane;
        int lo = 0, hi = 31;  // largest lane m with off[m] <= j
#pragma unroll
        for (int it = 0; it < 5; it++) {
            const int mid = (lo + hi + 1) >> 1;
            const uint32_t v = __shfl_sync(FULL, off, mid);
            if (v <= j) lo = mid;
            else hi = mid - 1;
        }
        const uint32_t o_off = __shfl_sync(FULL, off, lo);
        const uint32_t o_id = __shfl_sync(FULL, id, lo);
        const int o_x0 = __shfl_sync(FULL, x0, lo), o_y0 = __shfl_sync(FULL, y0, lo), o_w = __shfl_sync(FULL, w, lo);
        const unsigned long long o_mask = __shfl_sync(FULL, mask, lo);
        if (j < span_end) {
            int local = (int)(j - o_off);
            if (o_mask != ~0ull) {  // local-th kept tile of the rectangle
                const uint32_t mlo = (uint32_t)o_mask;
                const int clo = __popc(mlo);
                local = local < clo ? (int)__fns(mlo, 0, local + 1) : 32 + (int)__fns((uint32_t)(o_mask >> 32), 0, local - clo + 1);
            }
            const int ry = local / o_w, rx = local - ry * o_w;
            keys[j] = (KeyT)((o_y0 + ry) * gx + (o_x0 + rx));
            ids[j] = o_id;
        }
    }
    const uint32_t R = (uint32_t)offsets[P - 1];
    if (R > capacity) {
        if (k == 0) header[HDR_OVERFLOW] = 1;
    } else {
        for (uint32_t j = R + (uint32_t)k; j < capacity; j += gridDim.x * blockDim.x) keys[j] = (KeyT)~0u;
    }
}

// K3  per-tile ranges: two binary searches per tile in the sorted tile keys (the reference scans all R keys,
// RAST/cuda_rasterizer/rasterizer_impl.cu:116-138).  Empty tiles get (0,0) like the reference's memset.
template <typename KeyT>
__global__ void __launch_bounds__(256) ranges_kernel(int R, int tiles, const KeyT* __restrict__ keys, uint2* __restrict__ ranges)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= tiles) return;
    auto lower = [&](uint32_t key) {
        int lo = 0, hi = R;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((uint32_t)keys[mid] < key) lo = mid + 1;
            else hi = mid;
        }
        return (uint32_t)lo;
    };
    const uint32_t a = lower((uint32_t)t), b = lower((uint32_t)t + 1u);
    ranges[t] = (b > a) ? make_uint2(a, b) : make_uint2(0u, 0u);
}

// ------------------------------------------------------------------------------------------------
// K4/K5  forward blend.  Block = one 16x16 tile, 8 warps; warp w owns the 8x4 pixel sub-tile
// (w&1, w>>1).  Warps never synchronise with each other: each walks the tile's depth-sorted list in
// batches of 32 (lane-parallel gather + cull), then broadcasts the survivors through its private
// shared-memory slice.  Per-pixel arithmetic is the reference's, operation for operation.
// ------------------------------------------------------------------------------------------------
template <bool COUNT>
__global__ void __launch_bounds__(256)
blend_forward_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H, int tiles_x,
                     const float2* __restrict__ means2D, const float4* __restrict__ conic_opacity, const float4* __restrict__ rgb,
                     const float* __restrict__ bg, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                     float* __restrict__ out_color, int* __restrict__ count, const int* __restrict__ header)
{
    if (header[HDR_OVERFLOW]) return;   // binning blob too small: the host repeats scatter + blend (lgr_bin.cuh)
    __shared__ float2 s_xy[8][32];
    __shared__ float4 s_co[8][32];
    __shared__ float4 s_rgb[8][32];
    __shared__ uint32_t s_id[8][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int sx0 = tx * LGR_TILE + (warp & 1) * 8, sy0 = ty * LGR_TILE + (warp >> 1) * 4;
    const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
    const bool inside = px < W && py < H;
    const float pxf = (float)px, pyf = (float)py;
    const float rx0 = (float)sx0, rx1 = (float)min(sx0 + 7, W - 1), ry0 = (float)sy0, ry1 = (float)min(sy0 + 3, H - 1);
    const uint2 range = ranges[tile];

    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f;
    uint32_t last = 0;
    bool done = !inside;

    for (uint32_t base = range.x; base < range.y; base += 32) {
        if (__all_sync(FULL, done)) break;
        const uint32_t idx = base + lane;
        const bool valid = idx < range.y;
        const uint32_t id = valid ? point_list[idx] : 0u;
        const float2 xy = means2D[id];
        const float4 co = conic_opacity[id];
        const bool keep = valid && !subtile_cull(xy.x, xy.y, co, rx0, rx1, ry0, ry1);
        unsigned mask = __ballot_sync(FULL, keep);
        if (mask == 0) continue;
        float4 col = make_float4(0.f, 0.f, 0.f, 0.f);
        if (keep) col = rgb[id];
        __syncwarp();
        s_xy[warp][lane] = xy;
        s_co[warp][lane] = co;
        s_rgb[warp][lane] = col;
        if (COUNT) s_id[warp][lane] = id;
        __syncwarp();
        while (mask) {
            const int j = __ffs(mask) - 1;
            mask &= mask - 1;
            bool contrib = false;
            if (!done) {
                const float2 g = s_xy[warp][j];
                const float4 c = s_co[warp][j];
                const float dx = LGR_SUB(g.x, pxf), dy = LGR_SUB(g.y, pyf);
                const float power = lgr::pair_power(dx, dy, c.x, c.y, c.z);
                if (!(power > 0.0f)) {
                    const float alpha = fminf(0.99f, LGR_MUL(c.w, expf(power)));
                    if (!(alpha < 1.0f / 255.0f)) {
                        const float test_T = LGR_MUL(T, LGR_SUB(1.0f, alpha));
                        if (test_T < 0.0001f) {
                            done = true;
                        } else {
                            const float4 f = s_rgb[warp][j];
                            C0 = LGR_FMA(T, LGR_MUL(alpha, f.x), C0);
                            C1 = LGR_FMA(T, LGR_MUL(alpha, f.y), C1);
                            C2 = LGR_FMA(T, LGR_MUL(alpha, f.z), C2);
                            T = test_T;
                            last = (base - range.x) + (uint32_t)j + 1u;
                            contrib = true;
                        }
                    }
                }
            }
            if (COUNT) {
                const unsigned cm = __ballot_sync(FULL, contrib);
                if (cm != 0 && lane == 0) atomicAdd(&count[s_id[warp][j]], __popc(cm));
            }
            if (__all_sync(FULL, done)) mask = 0;
        }
    }
    if (inside) {
        const size_t pix = (size_t)py * W + px;
        const size_t plane = (size_t)H * W;
        final_T[pix] = T;
        n_contrib[pix] = last;
        out_color[pix] = LGR_FMA(bg[0], T, C0);
        out_color[plane + pix] = LGR_FMA(bg[1], T, C1);
        out_color[2 * plane + pix] = LGR_FMA(bg[2], T, C2);
    }
}

__global__ void __launch_bounds__(256) score_kernel(int P, const int* __restrict__ count, const float* __restrict__ opacities,
                                                    float* __restrict__ score)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P) score[i] = opacities[i] * (float)count[i];
}

__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ view,
                                                           uint8_t* __restrict__ present)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float v[16];
#pragma unroll
    for (int k = 0; k < 16; k++) v[k] = view[k];
    present[i] = lgr::xform_row(v, 2, means3D[3 * i], means3D[3 * i + 1], means3D[3 * i + 2]) > 0.2f;
}

// ------------------------------------------------------------------------------------------------
// K6  backward blend (RAST/cuda_rasterizer/backward.cu:399-557).
// Per (warp, Gaussian) the nine per-lane partial sums are parked in a per-warp shared-memory matrix
// [column = (buffered Gaussian, component)][lane]; every RED_K Gaussians the matrix is summed with one lane per
// column (8 conflict-free LDS.128 each) and ONE vector of atomics -- instead of a 14-shuffle butterfly per Gaussian.
// ------------------------------------------------------------------------------------------------
constexpr int RED_K = 3;                 // Gaussians buffered between flushes (27 columns <= 32 lanes)
constexpr int RED_STRIDE = 36;           // floats per column: 32 lanes + 4 pad => 16-byte units stride 9 == 1 (mod 8)

__device__ __forceinline__ void red_flush(float* __restrict__ red, const uint32_t* __restrict__ rid, int nbuf, int lane, int col_g,
                                          int col_c, float* __restrict__ acc)
{
    __syncwarp();
    if (lane < nbuf * 9) {
        const float4* p = reinterpret_cast<const float4*>(red + lane * RED_STRIDE);
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const float4 t = p[q];
            s += (t.x + t.y) + (t.z + t.w);
        }
        atomicAdd(acc + (size_t)rid[col_g] * ACC_STRIDE + col_c, s);
    }
    __syncwarp();
}

__global__ void __launch_bounds__(256, 5)
blend_backward_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H, int tiles_x,
                      const float2* __restrict__ means2D, const float4* __restrict__ conic_opacity, const float4* __restrict__ rgb,
                      const float* __restrict__ bg, const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
                      const float* __restrict__ dL_dpix, float* __restrict__ acc)
{
    __shared__ float2 s_xy[8][32];
    __shared__ float4 s_co[8][32];
    __shared__ float4 s_rgb[8][32];
    __shared__ uint32_t s_id[8][32];
    __shared__ __align__(16) float s_red[8][RED_K * 9 * RED_STRIDE];
    __shared__ uint32_t s_rid[8][4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int sx0 = tx * LGR_TILE + (warp & 1) * 8, sy0 = ty * LGR_TILE + (warp >> 1) * 4;
    const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
    const bool inside = px < W && py < H;
    const float pxf = (float)px, pyf = (float)py;
    const float rx0 = (float)sx0, rx1 = (float)min(sx0 + 7, W - 1), ry0 = (float)sy0, ry1 = (float)min(sy0 + 3, H - 1);
    const uint2 range = ranges[tile];
    const size_t pix = (size_t)py * W + px;
    const size_t plane = (size_t)H * W;

    const float T_final = inside ? final_T[pix] : 0.f;
    float T = T_final;
    const uint32_t last = inside ? n_contrib[pix] : 0u;
    float d0 = 0.f, d1 = 0.f, d2 = 0.f;
    if (inside) {
        d0 = dL_dpix[pix];
        d1 = dL_dpix[plane + pix];
        d2 = dL_dpix[2 * plane + pix];
    }
    const float bg_dot = bg[0] * d0 + bg[1] * d1 + bg[2] * d2;
    const uint32_t max_last = __reduce_max_sync(FULL, last);
    if (max_last == 0) return;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;       // accum_rec
    float lc0 = 0.f, lc1 = 0.f, lc2 = 0.f;    // last colour
    float last_alpha = 0.f;
    float* red = s_red[warp];
    uint32_t* rid = s_rid[warp];
    const int col_g = lane / 9, col_c = lane - 9 * (lane / 9);
    int nbuf = 0;

    for (int b = (int)((max_last - 1) >> 5); b >= 0; --b) {
        const uint32_t pos = (uint32_t)b * 32u + lane;
        const bool valid = pos < max_last;
        const uint32_t id = valid ? point_list[range.x + pos] : 0u;
        const float2 xy = means2D[id];
        const float4 co = conic_opacity[id];
        const bool keep = valid && !subtile_cull(xy.x, xy.y, co, rx0, rx1, ry0, ry1);
        unsigned mask = __ballot_sync(FULL, keep);
        if (mask == 0) continue;
        float4 col = make_float4(0.f, 0.f, 0.f, 0.f);
        if (keep) col = rgb[id];
        __syncwarp();
        s_xy[warp][lane] = xy;
        s_co[warp][lane] = co;
        s_rgb[warp][lane] = col;
        s_id[warp][lane] = id;
        __syncwarp();
        while (mask) {
            const int j = 31 - __clz(mask);  // back to front
            mask &= ~(1u << j);
            const uint32_t pj = (uint32_t)b * 32u + (uint32_t)j;
            const float2 g = s_xy[warp][j];
            const float4 c = s_co[warp][j];
            const float dx = LGR_SUB(g.x, pxf), dy = LGR_SUB(g.y, pyf);
            const float power = lgr::pair_power(dx, dy, c.x, c.y, c.z);
            float G = 0.f, alpha = 0.f;
            bool on = (pj < last) && !(power > 0.0f);
            if (on) {
                G = expf(power);
                alpha = fminf(0.99f, LGR_MUL(c.w, G));
                on = !(alpha < 1.0f / 255.0f);
            }
            if (!__any_sync(FULL, on)) continue;
            float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f, v5 = 0.f, v6 = 0.f, v7 = 0.f, v8 = 0.f;
            if (on) {
                const float4 f = s_rgb[warp][j];
                // 1/(1-alpha): 1-alpha is in [0.01, 0.996], so MUFU.RCP + one Newton step is within 1 ulp and needs no
                // range fix-up (the two IEEE divisions of the reference cost ~25 instructions here)
                const float one_m_a = 1.0f - alpha;
                float rcp;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rcp) : "f"(one_m_a));
                rcp = fmaf(rcp, fmaf(-one_m_a, rcp, 1.0f), rcp);
                T = T * rcp;
                const float w = alpha * T;
                const float oml = 1.f - last_alpha;
                a0 = fmaf(last_alpha, lc0, oml * a0);
                a1 = fmaf(last_alpha, lc1, oml * a1);
                a2 = fmaf(last_alpha, lc2, oml * a2);
                lc0 = f.x; lc1 = f.y; lc2 = f.z;
                float dL_dalpha = (f.x - a0) * d0 + (f.y - a1) * d1 + (f.z - a2) * d2;
                v0 = w * d0; v1 = w * d1; v2 = w * d2;
                last_alpha = alpha;
                dL_dalpha = fmaf(dL_dalpha, T, (-T_final * rcp) * bg_dot);
                const float wg = G * dL_dalpha;   // S0 term (= dL/dopacity contribution)
                const float wdx = wg * dx, wdy = wg * dy;
                v3 = wg; v4 = wdx; v5 = wdy;
                v6 = wdx * dx; v7 = wdx * dy; v8 = wdy * dy;
            }
            float* colp = red + nbuf * 9 * RED_STRIDE + lane;
            colp[0 * RED_STRIDE] = v0; colp[1 * RED_STRIDE] = v1; colp[2 * RED_STRIDE] = v2;
            colp[3 * RED_STRIDE] = v3; colp[4 * RED_STRIDE] = v4; colp[5 * RED_STRIDE] = v5;
            colp[6 * RED_STRIDE] = v6; colp[7 * RED_STRIDE] = v7; colp[8 * RED_STRIDE] = v8;
            if (lane == 0) rid[nbuf] = s_id[warp][j];
            if (++nbuf == RED_K) {
                red_flush(red, rid, nbuf, lane, col_g, col_c, acc);
                nbuf = 0;
            }
        }
    }
    if (nbuf) red_flush(red, rid, nbuf, lane, col_g, col_c, acc);
}

// accumulator record -> dL/dmean2D (x,y), dL/dconic (x,y,w), dL/dopacity  (RAST/cuda_rasterizer/backward.cu:538-554)
struct Grad2D {
    float dcol[3], dop, dm2x, dm2y, dcx, dcy, dcw;
};
__device__ __forceinline__ Grad2D accum_to_grad2d(const float* __restrict__ rec, float4 co, int W, int H)
{
    const float4* rec4 = reinterpret_cast<const float4*>(rec);
    const float4 r0 = rec4[0], r1 = rec4[1], r2 = rec4[2];
    Grad2D g;
    g.dcol[0] = r0.x; g.dcol[1] = r0.y; g.dcol[2] = r0.z;
    g.dop = r0.w;
    const float o = co.w;
    g.dm2x = -o * (0.5f * W) * (co.x * r1.x + co.y * r1.y);
    g.dm2y = -o * (0.5f * H) * (co.z * r1.y + co.y * r1.x);
    g.dcx = -0.5f * o * r1.z;
    g.dcy = -0.5f * o * r1.w;
    g.dcw = -0.5f * o * r2.x;
    return g;
}

// ------------------------------------------------------------------------------------------------
// K7+K8 fused  (RAST/cuda_rasterizer/backward.cu:144-396).  One thread per Gaussian; writes EVERY dense
// output row (zeros for culled Gaussians) so the caller never has to clear them.
// ------------------------------------------------------------------------------------------------
struct PreBackArgs {
    int P, D, M, W, H;
    float fx, fy, tanx, tany, mod;
    const float* means3D;
    const float* scales;
    const float* rotations;
    const float* shs;
    const float* cov3D;  // precomputed by the caller, or the forward's geometry cov3D
    const float* view;
    const float* proj;
    const float* campos;
    const int* radii;
    const uint8_t* clamped;
    const float* acc;
    const float4* conic_opacity;
    float* dL_dmeans2D;
    float* dL_dcolors;
    float* dL_dopacity;
    float* dL_dmeans3D;
    float* dL_dcov3D;
    float* dL_dsh;
    float* dL_dscales;
    float* dL_drot;
};

__global__ void __launch_bounds__(256) preprocess_backward_kernel(PreBackArgs a)
{
    __shared__ float s_cam[36];
    if (threadIdx.x < 16) s_cam[threadIdx.x] = a.view[threadIdx.x];
    else if (threadIdx.x < 32) s_cam[threadIdx.x] = a.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_cam[threadIdx.x] = a.campos[threadIdx.x - 32];
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    const size_t si = (size_t)i;
    const bool vis = a.radii[i] > 0;
    float4* dsh4 = a.M == 16 ? reinterpret_cast<float4*>(a.dL_dsh + si * 48) : nullptr;
    if (!vis) {
        a.dL_dmeans2D[3 * si] = 0.f; a.dL_dmeans2D[3 * si + 1] = 0.f; a.dL_dmeans2D[3 * si + 2] = 0.f;
        a.dL_dcolors[3 * si] = 0.f; a.dL_dcolors[3 * si + 1] = 0.f; a.dL_dcolors[3 * si + 2] = 0.f;
        a.dL_dopacity[si] = 0.f;
        a.dL_dmeans3D[3 * si] = 0.f; a.dL_dmeans3D[3 * si + 1] = 0.f; a.dL_dmeans3D[3 * si + 2] = 0.f;
#pragma unroll
        for (int k = 0; k < 6; k++) a.dL_dcov3D[6 * si + k] = 0.f;
        a.dL_dscales[3 * si] = 0.f; a.dL_dscales[3 * si + 1] = 0.f; a.dL_dscales[3 * si + 2] = 0.f;
        reinterpret_cast<float4*>(a.dL_drot)[si] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a.dL_dsh) {
            if (dsh4) {
#pragma unroll
                for (int j = 0; j < 12; j++) dsh4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            } else {
                for (int k = 0; k < 3 * a.M; k++) a.dL_dsh[si * 3 * a.M + k] = 0.f;
            }
        }
        return;
    }
    const float* view = s_cam;
    const float* proj = s_cam + 16;
    const float* cam = s_cam + 32;
    const Grad2D g2 = accum_to_grad2d(a.acc + si * ACC_STRIDE, a.conic_opacity[si], a.W, a.H);
    const float x = a.means3D[3 * si], y = a.means3D[3 * si + 1], z = a.means3D[3 * si + 2];
    float c3[6];
#pragma unroll
    for (int k = 0; k < 6; k++) c3[k] = a.cov3D[6 * si + k];
    float dcov[6], dmean[3];
    lgr::cov2d_backward(x, y, z, view, c3, a.fx, a.fy, a.tanx, a.tany, g2.dcx, g2.dcy, g2.dcw, dcov, dmean);
    lgr::mean2d_backward(x, y, z, proj, g2.dm2x, g2.dm2y, dmean);
    a.dL_dmeans2D[3 * si] = g2.dm2x; a.dL_dmeans2D[3 * si + 1] = g2.dm2y; a.dL_dmeans2D[3 * si + 2] = 0.f;
    a.dL_dcolors[3 * si] = g2.dcol[0]; a.dL_dcolors[3 * si + 1] = g2.dcol[1]; a.dL_dcolors[3 * si + 2] = g2.dcol[2];
    a.dL_dopacity[si] = g2.dop;
#pragma unroll
    for (int k = 0; k < 6; k++) a.dL_dcov3D[6 * si + k] = dcov[k];

    if (a.shs) {
        const unsigned cb = a.clamped[i];
        const float dRGB[3] = {(cb & 1u) ? 0.f : g2.dcol[0], (cb & 2u) ? 0.f : g2.dcol[1], (cb & 4u) ? 0.f : g2.dcol[2]};
        const float* sh = a.shs + si * a.M * 3;
        if (a.M == 16) {
            float v[48], o[48];
            const int nfl = 3 * (a.D + 1) * (a.D + 1);
            const float4* s4 = reinterpret_cast<const float4*>(sh);
#pragma unroll
            for (int j = 0; j < 12; j++) {
                float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
                if (4 * j < nfl) t = __ldg(s4 + j);
                v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
            }
#pragma unroll
            for (int k = 0; k < 48; k++) o[k] = 0.f;
            lgr::sh_backward(a.D, [&](int k) { return v[k]; }, [&](int k, int c, float val) { o[3 * k + c] = val; }, x, y, z, cam,
                             dRGB, dmean);
#pragma unroll
            for (int j = 0; j < 12; j++) dsh4[j] = make_float4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
        } else {
            float* out = a.dL_dsh + si * 3 * a.M;
            const int nb = (a.D + 1) * (a.D + 1);
            for (int k = 3 * nb; k < 3 * a.M; k++) out[k] = 0.f;
            lgr::sh_backward(a.D, [&](int k) { return __ldg(sh + k); }, [&](int k, int c, float val) { out[3 * k + c] = val; }, x, y, z,
                             cam, dRGB, dmean);
        }
    } else if (a.dL_dsh) {
        for (int k = 0; k < 3 * a.M; k++) a.dL_dsh[si * 3 * a.M + k] = 0.f;
    }
    a.dL_dmeans3D[3 * si] = dmean[0]; a.dL_dmeans3D[3 * si + 1] = dmean[1]; a.dL_dmeans3D[3 * si + 2] = dmean[2];
    if (a.scales) {
        const float4 q = reinterpret_cast<const float4*>(a.rotations)[si];
        float dscale[3], dq[4];
        lgr::cov3d_backward(a.scales[3 * si], a.scales[3 * si + 1], a.scales[3 * si + 2], a.mod, q.x, q.y, q.z, q.w, dcov, dscale, dq);
        a.dL_dscales[3 * si] = dscale[0]; a.dL_dscales[3 * si + 1] = dscale[1]; a.dL_dscales[3 * si + 2] = dscale[2];
        reinterpret_cast<float4*>(a.dL_drot)[si] = make_float4(dq[0], dq[1], dq[2], dq[3]);
    } else {
        a.dL_dscales[3 * si] = 0.f; a.dL_dscales[3 * si + 1] = 0.f; a.dL_dscales[3 * si + 2] = 0.f;
        reinterpret_cast<float4*>(a.dL_drot)[si] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

}  // namespace
#include "lgr_raw.cuh"
#include "lgr_blend.cuh"
#include "lgr_sparse.cuh"
#include "lgr_loss.cuh"
#include "lgr_optim.cuh"
#include "lgr_vq.cuh"
#include "lgr_vq_tc.cuh"
#include "lgr_knn.cuh"
#include "lgr_densify.cuh"
namespace {

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// row stride (floats) of the features_rest leaf: 0 in the struct means dense
inline int raw_rest_stride(const lgr_raw_params* raw, int M) { return raw->features_rest_row_stride > 0 ? raw->features_rest_row_stride : (M - 1) * 3; }
inline bool raw_rest_stride_ok(const lgr_raw_params* raw, int M)
{
    const int s = raw->features_rest_row_stride;
    return s == 0 || (s >= (M - 1) * 3 && s <= 256);
}

struct PinnedInt {
    int* p = nullptr;
    ~PinnedInt() { if (p) cudaFreeHost(p); }
    int* get()
    {
        if (!p) cudaMallocHost(&p, 64);
        return p;
    }
};
thread_local PinnedInt t_pinned;

struct SyncEvent {
    cudaEvent_t e = nullptr;
    ~SyncEvent() { if (e) cudaEventDestroy(e); }
    cudaEvent_t get()
    {
        if (!e) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
        return e;
    }
};
thread_local SyncEvent t_event;
std::atomic<uint64_t> g_bin_overflows{0};
std::atomic<uint64_t> g_forward_syncs{0};   // stream synchronisations of the forwards (exactly sized binning blobs)

// LGR_BINNING_SYNC=1: the library binning sizes its blob exactly after a stream synchronisation, as deterministic mode does (tests
// compare the default's estimated, padded lists against it)
bool binning_sync_requested()
{
    const char* e = std::getenv("LGR_BINNING_SYNC");
    return e && e[0] == '1';
}

__global__ void set_capacity_kernel(int* header, int capacity, int det)
{
    if (threadIdx.x == 0) {
        header[HDR_CAPACITY] = capacity;
        header[HDR_OVERFLOW] = 0;
        header[HDR_DET] = det;
    }
}

// the geometry fields of the raw-leaf / resident preprocess, from the plain preprocess arguments
inline RawArgs raw_args(const PreprocessArgs& a, int gx, int gy)
{
    RawArgs ra;
    ra.P = a.P; ra.D = a.D; ra.M = a.M; ra.W = a.W; ra.H = a.H; ra.gx = gx; ra.gy = gy;
    ra.fx = a.fx; ra.fy = a.fy; ra.tanx = a.tanx; ra.tany = a.tany; ra.mod = a.mod;
    ra.xyz = nullptr; ra.view = a.view; ra.proj = a.proj; ra.campos = a.campos;
    ra.prefiltered = a.prefiltered;
    ra.rest_stride = 0;
    return ra;
}

// deterministic mode: the binning's helpers (iota as sort values, point_list by gather through the permutation)
__global__ void __launch_bounds__(256) det_iota_kernel(int R, uint32_t* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R) out[i] = (uint32_t)i;
}
__global__ void __launch_bounds__(256) det_point_list_kernel(int R, const uint32_t* __restrict__ perm, const uint32_t* __restrict__ ids_unsorted,
                                                             uint32_t* __restrict__ point_list)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < R) point_list[i] = ids_unsorted[perm[i]];
}

// Deterministic mode's tile sort: the values are the unsorted instance indices, so the stable sort yields the permutation (sorted ->
// unsorted), which the forward blend stores in the records for the deterministic backward; the ids follow by one gather, the same list
// as sorting the ids themselves.  The permutation lives in the partial-row region until the backward overwrites it.  Also clears the
// bitmap of instances the backward reaches.
template <typename KeyT>
int det_tile_sort(const BinningState& bin, int R, int bits, bool debug, cudaStream_t stream)
{
    uint32_t* perm = reinterpret_cast<uint32_t*>(bin.det_partial);
    det_iota_kernel<<<(R + 255) / 256, 256, 0, stream>>>(R, bin.point_list);
    LGR_LAUNCH_CHECK("det_iota_kernel", debug, stream);
    size_t tmp = bin.cub_temp_bytes;
    LGR_CUDA_TRY(cub::DeviceRadixSort::SortPairs(bin.cub_temp, tmp, (const KeyT*)bin.keys_unsorted, (KeyT*)bin.keys_sorted,
                                                  (const uint32_t*)bin.point_list, perm, R, 0, bits, stream));
    det_point_list_kernel<<<(R + 255) / 256, 256, 0, stream>>>(R, perm, bin.ids_unsorted, bin.point_list);
    LGR_LAUNCH_CHECK("det_point_list_kernel", debug, stream);
    LGR_CUDA_TRY(cudaMemsetAsync(bin.det_reached, 0, sizeof(uint32_t) * (((size_t)R + 31) / 32), stream));
    return LGR_OK;
}

// K2 + tile sort + K3 of the library binning over `items` instances of a blob that holds `capacity` (items == capacity, or the exact
// count R <= capacity): emit (pads and overflow flag, see emit_kernel), stable radix sort by tile, per-tile ranges
template <typename KeyT>
int tile_binning(const GeometryState& geo, const BinningState& bin, const ImageState& img, const int32_t* radii, int P, int items,
                 int capacity, int gx, int gy, int bits, bool det, bool debug, cudaStream_t stream)
{
    {
        ProfScope ps(ST_EMIT, stream);
        emit_kernel<KeyT><<<(P + 255) / 256, 256, 0, stream>>>(P, geo.sorted_ids, geo.offsets, geo.keep_mask, geo.means2D,
                                                                 radii, gx, gy, (uint32_t)capacity, (KeyT*)bin.keys_unsorted,
                                                                 bin.ids_unsorted, geo.num_rendered);
    }
    LGR_LAUNCH_CHECK("emit_kernel", debug, stream);
    {
        ProfScope ps(ST_TILE_SORT, stream);
        if (det) {
            const int st = det_tile_sort<KeyT>(bin, items, bits, debug, stream);
            if (st != LGR_OK) return st;
        } else {
            size_t tmp = bin.cub_temp_bytes;
            LGR_CUDA_TRY(cub::DeviceRadixSort::SortPairs(bin.cub_temp, tmp, (const KeyT*)bin.keys_unsorted, (KeyT*)bin.keys_sorted,
                                                          (const uint32_t*)bin.ids_unsorted, bin.point_list, items, 0, bits, stream));
        }
    }
    {
        ProfScope ps(ST_RANGES, stream);
        ranges_kernel<KeyT><<<(gx * gy + 255) / 256, 256, 0, stream>>>(items, gx * gy, (const KeyT*)bin.keys_sorted, img.ranges);
    }
    LGR_LAUNCH_CHECK("ranges_kernel", debug, stream);
    return LGR_OK;
}

// deterministic mode has no implementation for the hand-written binning or the round-1 blend kernels: refuse before any launch
bool det_supported(const char* what)
{
    if (g_bin_mode != 2) {
        g_last_error = std::string(what) + ": deterministic mode needs library binning; lgr_set_binning_mode(" + std::to_string(g_bin_mode) +
                       ") has no deterministic implementation";
        return false;
    }
    if (g_blend_mode != 0) {
        g_last_error = std::string(what) + ": deterministic mode needs the ring blend kernels; lgr_set_blend_mode(1) has no deterministic implementation";
        return false;
    }
    return true;
}

int forward_impl(const lgr_view* v, int P, int M, const float* means3D, const float* shs, const float* colors_precomp,
                 const float* opacities, const float* scales, const float* rotations, const float* cov3D_precomp,
                 lgr_alloc_fn geometry_alloc, void* geometry_user, lgr_alloc_fn binning_alloc, void* binning_user,
                 lgr_alloc_fn image_alloc, void* image_user, float* out_color, int32_t* gaussians_count, float* important_score,
                 int32_t* radii, int32_t* num_rendered, void* cuda_stream, bool count_mode, const lgr_raw_params* raw = nullptr,
                 const lgr_vq_resident_params* vq = nullptr, int64_t* blend_weight = nullptr, const BlendDepth* depth_out = nullptr)
{
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    if (vq) {  // resident VQ model: attributes and colour rows come from the compressed arrays (validated by lgr_forward_vq)
        means3D = vq->xyz;
        opacities = scales = static_cast<const float*>(vq->attr);
        rotations = static_cast<const float*>(vq->attr);
        shs = static_cast<const float*>(vq->codebook);
    }
    if (raw) {  // fused-activation path: the six leaves replace the activated tensors
        means3D = raw->xyz;
        opacities = raw->opacity;
        scales = raw->scaling;
        rotations = raw->rotation;
        shs = raw->features_dc;
        if (P > 0 && (!raw->xyz || !raw->opacity || !raw->scaling || !raw->rotation || !raw->features_dc || (M > 1 && !raw->features_rest))) {
            g_last_error = "lgr_forward_raw: a parameter leaf is NULL";
            return LGR_ERR_INVALID_ARG;
        }
        if (((uintptr_t)raw->features_rest & 15) || ((uintptr_t)raw->features_dc & 15)) {
            g_last_error = "lgr_forward_raw: features_dc / features_rest must be 16-byte aligned";
            return LGR_ERR_INVALID_ARG;
        }
        if (!raw_rest_stride_ok(raw, M)) {
            g_last_error = "lgr_forward_raw: features_rest_row_stride must be 0 (dense) or in [(M-1)*3, 256]";
            return LGR_ERR_INVALID_ARG;
        }
    }
    if (!v || P < 0 || M < 0 || !num_rendered || !out_color || !geometry_alloc || !binning_alloc || !image_alloc) {
        g_last_error = "lgr_forward: missing required argument";
        return LGR_ERR_INVALID_ARG;
    }
    const int W = v->image_width, H = v->image_height;
    if (W <= 0 || H <= 0 || v->sh_degree < 0 || v->sh_degree > 3) {
        g_last_error = "lgr_forward: bad image size or sh_degree";
        return LGR_ERR_INVALID_ARG;
    }
    if (P > 0) {
        if (!means3D || !opacities || !radii || (!shs && !colors_precomp) || (!cov3D_precomp && (!scales || !rotations))) {
            g_last_error = "lgr_forward: need means3D, opacities, radii, one of shs/colors_precomp and one of scales+rotations/cov3D_precomp";
            return LGR_ERR_INVALID_ARG;
        }
        if (shs && !colors_precomp && (v->sh_degree + 1) * (v->sh_degree + 1) > M) {
            g_last_error = "lgr_forward: sh_degree needs more coefficients than M";
            return LGR_ERR_INVALID_ARG;
        }
        if (count_mode && (!gaussians_count || !important_score)) {
            g_last_error = "lgr_forward_count: gaussians_count / important_score missing";
            return LGR_ERR_INVALID_ARG;
        }
    }
    if (g_det && !det_supported("lgr_forward")) return LGR_ERR_INVALID_ARG;
    if (blend_weight && (!count_mode || g_blend_mode != 0)) {
        g_last_error = g_blend_mode != 0 ? "lgr_forward_*_weight: the blending weight needs the ring blend kernels; lgr_set_blend_mode(1) has no weight output"
                                         : "lgr_forward_*_weight: the blending weight is a count-mode output";
        return LGR_ERR_INVALID_ARG;
    }
    if (depth_out && (count_mode || g_det || g_blend_mode != 0)) {
        g_last_error = count_mode ? "lgr_forward_raw_depth: depth and alpha are not count-mode outputs"
                       : g_det    ? "lgr_forward_raw_depth: deterministic mode has no depth or alpha output"
                                  : "lgr_forward_raw_depth: depth and alpha need the ring blend kernels; lgr_set_blend_mode(1) has no depth output";
        return LGR_ERR_INVALID_ARG;
    }
    const bool debug = v->debug != 0;
    *num_rendered = 0;
    const int gx = (W + LGR_TILE - 1) / LGR_TILE, gy = (H + LGR_TILE - 1) / LGR_TILE;
    const size_t N = (size_t)W * H;

    if (P == 0) {  // the reference returns an all-zero image and empty blobs (rasterize_points.cu:79-93)
        LGR_CUDA_TRY(cudaMemsetAsync(out_color, 0, sizeof(float) * 3 * N, stream));
        if (depth_out && depth_out->depth) LGR_CUDA_TRY(cudaMemsetAsync(depth_out->depth, 0, sizeof(float) * N, stream));
        if (depth_out && depth_out->alpha) LGR_CUDA_TRY(cudaMemsetAsync(depth_out->alpha, 0, sizeof(float) * N, stream));
        return LGR_OK;
    }
    if (((uintptr_t)rotations & 15) || ((uintptr_t)shs & 15)) {
        g_last_error = "lgr_forward: rotations and shs must be 16-byte aligned";
        return LGR_ERR_INVALID_ARG;
    }
    const int tiles = gx * gy;
    const bool lib_bin = g_bin_mode == 2 || tiles > BIN_MAX_TILES || gx > 0xffff || gy > 0xffff || bin_per_block(P) > 65535;
    GeometryState geo = carve_geometry(nullptr, (size_t)P, lib_bin);
    char* geo_blob = geometry_alloc(geometry_user, geo.total);
    if (!geo_blob) { g_last_error = "geometry allocator returned NULL"; return LGR_ERR_ALLOC; }
    geo = carve_geometry(geo_blob, (size_t)P, lib_bin);

    ImageState img = carve_image(nullptr, W, H, lib_bin);
    char* img_blob = image_alloc(image_user, img.total);
    if (!img_blob) { g_last_error = "image allocator returned NULL"; return LGR_ERR_ALLOC; }
    img = carve_image(img_blob, W, H, lib_bin);

    {
        PreprocessArgs a;
        a.P = P; a.D = v->sh_degree; a.M = M; a.W = W; a.H = H; a.gx = gx; a.gy = gy;
        a.fy = H / (2.0f * v->tan_fovy);   // rasterizer_impl.cu:223-224
        a.fx = W / (2.0f * v->tan_fovx);
        a.tanx = v->tan_fovx; a.tany = v->tan_fovy; a.mod = v->scale_modifier;
        a.means3D = means3D; a.scales = scales; a.rotations = rotations; a.opacities = opacities; a.shs = shs;
        a.cov3D_precomp = cov3D_precomp; a.colors_precomp = colors_precomp;
        a.view = v->viewmatrix; a.proj = v->projmatrix; a.campos = v->campos; a.prefiltered = v->prefiltered;
        const int blocks = (P + 255) / 256;
        if (raw) {
            RawArgs ra = raw_args(a, gx, gy);
            ra.xyz = raw->xyz;
            ra.rest_stride = raw_rest_stride(raw, M);
            const LeafSource src = {raw->features_dc, raw->features_rest, raw->scaling, raw->rotation, raw->opacity};
            const size_t smem = raw_smem_bytes_stride(ra.rest_stride);
            LGR_CUDA_TRY(cudaFuncSetAttribute(preprocess_raw_kernel<LeafSource>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ProfScope ps(ST_PREPROCESS, stream);
            preprocess_raw_kernel<<<blocks, 256, smem, stream>>>(ra, src, radii, geo);
        } else if (vq) {
            RawArgs ra = raw_args(a, gx, gy);
            ra.xyz = vq->xyz;
            ra.rest_stride = (M - 1) * 3;
            const VqSource src = {vq->attr, vq->slot, static_cast<const __half*>(vq->codebook), vq->nonvq, vq->attr_half, vq->nonvq_half,
                                  vq->D, vq->Dp, M};
            const size_t smem = raw_smem_bytes_stride(ra.rest_stride);
            LGR_CUDA_TRY(cudaFuncSetAttribute(preprocess_raw_kernel<VqSource>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ProfScope ps(ST_PREPROCESS, stream);
            preprocess_raw_kernel<<<blocks, 256, smem, stream>>>(ra, src, radii, geo);
        } else {
            ProfScope ps(ST_PREPROCESS, stream);
            preprocess_kernel<<<blocks, 256, 0, stream>>>(a, radii, geo);
        }
        LGR_LAUNCH_CHECK("preprocess_kernel", debug, stream);
    }

    int R = 0, R_ref = 0;
    BinningState bin = {};
    const bool det = g_det != 0;   // lib_bin holds: det_supported() refused the hand-written binning
    int* host_hdr = t_pinned.get();

    // K4/K5 -- and everything of it that has to be repeated when the binning blob turns out too small
    auto launch_blend = [&]() -> int {
        if (count_mode) LGR_CUDA_TRY(cudaMemsetAsync(gaussians_count, 0, sizeof(int) * (size_t)P, stream));
        if (blend_weight) LGR_CUDA_TRY(cudaMemsetAsync(blend_weight, 0, sizeof(int64_t) * (size_t)P, stream));
        ProfScope ps(count_mode ? ST_BLEND_FWD_COUNT : ST_BLEND_FWD, stream);
        if (depth_out) {   // refused above unless g_blend_mode == 0, not count mode and not deterministic
            BlendDepth dz = *depth_out;
            dz.z = geo.depth;
            dz.header = geo.num_rendered;
            blend_forward_ring_kernel<false, true, false, false, true><<<tiles, BL_THREADS, 0, stream>>>(
                img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity, geo.rgb, v->background, img.final_T, img.n_contrib,
                out_color, nullptr, bin.records, geo.num_rendered, nullptr, nullptr, dz);
        } else if (blend_weight)   // refused above unless g_blend_mode == 0 and count_mode
            blend_forward_ring_kernel<true, false, false, true><<<tiles, BL_THREADS, 0, stream>>>(
                img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity, geo.rgb, v->background, img.final_T, img.n_contrib,
                out_color, gaussians_count, nullptr, geo.num_rendered, nullptr, reinterpret_cast<unsigned long long*>(blend_weight));
        else if (g_blend_mode == 0 && count_mode)
            blend_forward_ring_kernel<true, false><<<tiles, BL_THREADS, 0, stream>>>(img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity,
                                                                                      geo.rgb, v->background, img.final_T, img.n_contrib, out_color,
                                                                                      gaussians_count, nullptr, geo.num_rendered);
        else if (g_blend_mode == 0 && det)
            blend_forward_ring_kernel<false, true, true><<<tiles, BL_THREADS, 0, stream>>>(img.ranges, bin.point_list, W, H, gx, geo.means2D,
                                                                                            geo.conic_opacity, geo.rgb, v->background, img.final_T,
                                                                                            img.n_contrib, out_color, nullptr, bin.records,
                                                                                            geo.num_rendered, reinterpret_cast<const uint32_t*>(bin.det_partial));
        else if (g_blend_mode == 0)
            blend_forward_ring_kernel<false, true><<<tiles, BL_THREADS, 0, stream>>>(img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity,
                                                                                      geo.rgb, v->background, img.final_T, img.n_contrib, out_color,
                                                                                      nullptr, bin.records, geo.num_rendered);
        else if (count_mode)
            blend_forward_kernel<true><<<tiles, 256, 0, stream>>>(img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity,
                                                                   geo.rgb, v->background, img.final_T, img.n_contrib, out_color,
                                                                   gaussians_count, geo.num_rendered);
        else
            blend_forward_kernel<false><<<tiles, 256, 0, stream>>>(img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity,
                                                                    geo.rgb, v->background, img.final_T, img.n_contrib, out_color,
                                                                    nullptr, geo.num_rendered);
        LGR_LAUNCH_CHECK("blend_forward_kernel", debug, stream);
        return LGR_OK;
    };

    if (!lib_bin) {
        // ---------------- hand-written binning (lgr_bin.cuh) ----------------
        const int per_block = bin_per_block(P);
        const int tiles_pad = bin_pad(tiles);
        {
            ProfScope ps(ST_BIN_DSORT, stream);
            BinScanArgs sa;
            sa.M = img.bin_M; sa.V = BIN_V; sa.bins = DS_BINS; sa.bins_pad = DS_BINS; sa.bin_total = img.bin_total; sa.bin_base = img.bin_base;
            sa.header = geo.num_rendered; sa.ranges = nullptr; sa.capacity = 0;
            // 11 + 11 + 10 bits: depth_keys -> (depth_keys_sorted, sorted_ids) -> (depth_keys, iota) -> sorted_ids
            dsort_count_kernel<0, true><<<BIN_V, 256, 0, stream>>>(geo.depth_keys, P, per_block, img.bin_M, geo.num_rendered);
            bin_scan_kernel<false><<<DS_BINS / 32, SCAN_THREADS, 0, stream>>>(sa);
            dsort_scatter_kernel<0, true, false><<<BIN_V, DS_THREADS, 0, stream>>>(geo.depth_keys, nullptr, geo.depth_keys_sorted, geo.sorted_ids, img.bin_M,
                                                                           img.bin_base, P, per_block);
            dsort_count_kernel<DS_BITS, false><<<BIN_V, 256, 0, stream>>>(geo.depth_keys_sorted, P, per_block, img.bin_M, geo.num_rendered);
            bin_scan_kernel<false><<<DS_BINS / 32, SCAN_THREADS, 0, stream>>>(sa);
            dsort_scatter_kernel<DS_BITS, false, false><<<BIN_V, DS_THREADS, 0, stream>>>(geo.depth_keys_sorted, geo.sorted_ids, geo.depth_keys, geo.iota,
                                                                                  img.bin_M, img.bin_base, P, per_block);
            dsort_count_kernel<2 * DS_BITS, false><<<BIN_V, 256, 0, stream>>>(geo.depth_keys, P, per_block, img.bin_M, geo.num_rendered);
            bin_scan_kernel<false><<<DS_BINS / 32, SCAN_THREADS, 0, stream>>>(sa);
            dsort_scatter_kernel<2 * DS_BITS, false, true><<<BIN_V, DS_THREADS, 0, stream>>>(geo.depth_keys, geo.iota, nullptr, geo.sorted_ids, img.bin_M,
                                                                                      img.bin_base, P, per_block);
            g_launches.fetch_add(8, std::memory_order_relaxed);
            LGR_LAUNCH_CHECK("depth sort kernels", debug, stream);
        }
        const size_t tb_smem = sizeof(uint32_t) * (size_t)tiles_pad, ts_smem = tile_scatter_smem(tiles_pad);
        // always: static + dynamic shared memory together may pass 48 KB even when the dynamic part alone does not
        LGR_CUDA_TRY(cudaFuncSetAttribute(tile_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(tb_smem, (size_t)48 * 1024)));
        LGR_CUDA_TRY(cudaFuncSetAttribute(tile_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(ts_smem, (size_t)48 * 1024)));
        const bool exact = g_bin_mode == 1;
        size_t capacity = 0;
        if (!exact) {   // size the blob now, from the running estimate
            capacity = std::max(g_bin_hint.load(std::memory_order_relaxed), (size_t)4096);
            bin = carve_binning(nullptr, capacity, W, H, false);
            char* bin_blob = binning_alloc(binning_user, bin.total);
            if (!bin_blob) { g_last_error = "binning allocator returned NULL"; return LGR_ERR_ALLOC; }
            bin = carve_binning(bin_blob, capacity, W, H, false);
        }
        {
            ProfScope ps(ST_BIN_COUNT, stream);
            tile_count_kernel<<<BIN_V, TC_THREADS, tb_smem, stream>>>(geo.sorted_ids, geo.bin_rec, P, per_block, gx, tiles_pad, img.bin_M, geo.num_rendered);
            BinScanArgs sa;
            sa.M = img.bin_M; sa.V = BIN_V; sa.bins = tiles; sa.bins_pad = tiles_pad; sa.bin_total = img.bin_total; sa.bin_base = img.bin_base;
            sa.header = geo.num_rendered; sa.ranges = img.ranges;
            sa.capacity = exact ? 0xffffffffu : (uint32_t)std::min(capacity, (size_t)0x7fffffff);
            bin_scan_kernel<true><<<tiles_pad / 32, SCAN_THREADS, 0, stream>>>(sa);
            g_launches.fetch_add(1, std::memory_order_relaxed);
            LGR_LAUNCH_CHECK("tile_count_kernel", debug, stream);
        }
        LGR_CUDA_TRY(cudaMemcpyAsync(host_hdr, geo.num_rendered, 4 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        auto launch_scatter = [&]() -> int {
            ProfScope ps(ST_BIN_SCATTER, stream);
            tile_scatter_kernel<<<BIN_V, TB_THREADS, ts_smem, stream>>>(geo.sorted_ids, geo.bin_rec, P, per_block, gx, tiles_pad, img.bin_M, img.bin_base,
                                                                        geo.num_rendered, bin.point_list);
            LGR_LAUNCH_CHECK("tile_scatter_kernel", debug, stream);
            return LGR_OK;
        };
        auto exact_blob = [&]() -> int {   // (re)allocate for exactly R instances and tell the device
            bin = carve_binning(nullptr, (size_t)R, W, H, false);
            char* bin_blob = binning_alloc(binning_user, bin.total);
            if (!bin_blob) { g_last_error = "binning allocator returned NULL"; return LGR_ERR_ALLOC; }
            bin = carve_binning(bin_blob, (size_t)R, W, H, false);
            set_capacity_kernel<<<1, 32, 0, stream>>>(geo.num_rendered, R > 0 ? R : 1, 0);
            LGR_LAUNCH_CHECK("set_capacity_kernel", debug, stream);
            return LGR_OK;
        };
        if (exact) {
            LGR_CUDA_TRY(cudaStreamSynchronize(stream));
            g_forward_syncs.fetch_add(1, std::memory_order_relaxed);
            R = host_hdr[HDR_LISTED];
            R_ref = host_hdr[HDR_RENDERED];
            int st = exact_blob();
            if (st != LGR_OK) return st;
            if ((st = launch_scatter()) != LGR_OK) return st;
            if ((st = launch_blend()) != LGR_OK) return st;
        } else {
            // the count is on its way to the host; scatter and blend are queued behind it right away, so the GPU keeps working while the
            // host waits for those 16 bytes
            cudaEvent_t ev = t_event.get();
            LGR_CUDA_TRY(cudaEventRecord(ev, stream));
            int st = launch_scatter();
            if (st != LGR_OK) return st;
            if ((st = launch_blend()) != LGR_OK) return st;
            LGR_CUDA_TRY(cudaEventSynchronize(ev));
            R = host_hdr[HDR_LISTED];
            R_ref = host_hdr[HDR_RENDERED];
            if ((size_t)R > capacity) {   // estimate too small (first view, or a jump between views): both kernels returned early; repeat
                if ((st = exact_blob()) != LGR_OK) return st;
                if ((st = launch_scatter()) != LGR_OK) return st;
                if ((st = launch_blend()) != LGR_OK) return st;
                g_bin_overflows.fetch_add(1, std::memory_order_relaxed);
            }
            // next estimate: 25 % above this view, never dropping by more than 2 % per view
            const size_t want = (size_t)R + (size_t)R / 4 + 4096, keep = g_bin_hint.load(std::memory_order_relaxed) / 50 * 49;
            g_bin_hint.store(std::max(want, keep), std::memory_order_relaxed);
        }
    } else {
        // ---------------- library radix sorts and scan ----------------
        // Default: the binning blob is sized from the running estimate before the count is known, and emit, tile sort, ranges and blend
        // are queued behind the count's copy to the host, so the GPU never waits for the host (the scheme of the hand-written binning
        // above).  Deterministic mode, and LGR_BINNING_SYNC=1, size the blob exactly after a stream synchronisation.
        const bool exact = det || binning_sync_requested();
        size_t capacity = 0;
        auto carve = [&](size_t instances) -> int {   // (re)allocate the blob for `instances` and tell the device
            bin = carve_binning(nullptr, instances, W, H, true, det);
            char* bin_blob = binning_alloc(binning_user, bin.total);
            if (!bin_blob) { g_last_error = "binning allocator returned NULL"; return LGR_ERR_ALLOC; }
            bin = carve_binning(bin_blob, instances, W, H, true, det);
            set_capacity_kernel<<<1, 32, 0, stream>>>(geo.num_rendered, instances > 0 ? (int)instances : 1, det ? 1 : 0);
            LGR_LAUNCH_CHECK("set_capacity_kernel", debug, stream);
            return LGR_OK;
        };
        const int bits = tile_key_bits(W, H);
        auto binning = [&](int items, int cap) -> int {
            return bin.wide_keys ? tile_binning<uint32_t>(geo, bin, img, radii, P, items, cap, gx, gy, bits, det, debug, stream)
                                 : tile_binning<uint16_t>(geo, bin, img, radii, P, items, cap, gx, gy, bits, det, debug, stream);
        };
        LGR_CUDA_TRY(cudaMemsetAsync(geo.num_rendered, 0, 64 * sizeof(int), stream));
        LGR_CUDA_TRY(cudaMemsetAsync(img.ranges, 0, sizeof(uint2) * (size_t)gx * gy, stream));
        if (!exact) {
            capacity = std::min(std::max(g_bin_hint.load(std::memory_order_relaxed), (size_t)4096), (size_t)INT_MAX);
            const int st = carve(capacity);
            if (st != LGR_OK) return st;
        }
        size_t tmp = geo.cub_temp_bytes;
        {
            ProfScope ps(ST_DEPTH_SORT, stream);
            LGR_CUDA_TRY(cub::DeviceRadixSort::SortPairs(geo.cub_temp, tmp, (const uint32_t*)geo.depth_keys, geo.depth_keys_sorted,
                                                          (const uint32_t*)geo.iota, geo.sorted_ids, P, 0, 32, stream));
        }
        auto it = thrust::make_transform_iterator((const uint32_t*)geo.sorted_ids, TilesTouchedOp{geo.tiles_kept, geo.tiles_touched});
        tmp = geo.cub_temp_bytes;
        {
            ProfScope ps(ST_SCAN, stream);
            LGR_CUDA_TRY(cub::DeviceScan::InclusiveSum(geo.cub_temp, tmp, it, geo.offsets, P, stream));
        }
        LGR_CUDA_TRY(cudaMemcpyAsync(geo.num_rendered, geo.offsets + (P - 1), 2 * sizeof(int), cudaMemcpyDeviceToDevice, stream));
        LGR_CUDA_TRY(cudaMemcpyAsync(host_hdr, geo.offsets + (P - 1), 2 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        int st = LGR_OK;
        if (exact) {
            LGR_CUDA_TRY(cudaStreamSynchronize(stream));
            g_forward_syncs.fetch_add(1, std::memory_order_relaxed);
            R = host_hdr[0];       // instances actually emitted (after exact tile culling)
            R_ref = host_hdr[1];   // the reference's num_rendered: sum of the tile-rectangle areas
            if ((st = carve((size_t)R)) != LGR_OK) return st;
            if (R > 0 && (st = binning(R, R)) != LGR_OK) return st;
            if ((st = launch_blend()) != LGR_OK) return st;
        } else {
            // all `capacity` slots are sorted: the pads past R sort last and no range reaches them (emit_kernel)
            cudaEvent_t ev = t_event.get();
            LGR_CUDA_TRY(cudaEventRecord(ev, stream));
            if ((st = binning((int)capacity, (int)capacity)) != LGR_OK) return st;
            if ((st = launch_blend()) != LGR_OK) return st;
            LGR_CUDA_TRY(cudaEventSynchronize(ev));
            R = host_hdr[0];
            R_ref = host_hdr[1];
            if ((size_t)R > capacity) {   // estimate too small (first view, or a jump between views): the blend returned early; repeat
                if ((st = carve((size_t)R)) != LGR_OK) return st;
                if ((st = binning(R, R)) != LGR_OK) return st;
                if ((st = launch_blend()) != LGR_OK) return st;
                g_bin_overflows.fetch_add(1, std::memory_order_relaxed);
            }
            // next estimate: 25 % above this view, never dropping by more than 2 % per view (as the hand-written binning's)
            const size_t want = (size_t)R + (size_t)R / 4 + 4096, keep = g_bin_hint.load(std::memory_order_relaxed) / 50 * 49;
            g_bin_hint.store(std::max(want, keep), std::memory_order_relaxed);
        }
    }
    if (count_mode && P > 0) {
        ProfScope ps(ST_SCORE, stream);
        if (raw || vq) score_from_geom_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, gaussians_count, geo.conic_opacity, important_score);
        else score_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, gaussians_count, opacities, important_score);
        LGR_LAUNCH_CHECK("score_kernel", debug, stream);
    }
    (void)N;
    *num_rendered = R_ref;
    return LGR_OK;
}

// Deterministic stage 1 of every backward: blend backward with fixed-order sums into per-instance partial rows, then one pass per
// Gaussian that writes every accumulator record (no memset, no float atomics).  zr.P > 0: the blend backward also clears the dense
// gradient rows, exactly as the default kernel does for kback mode 0.
int blend_backward_det(const GeometryState& geo, const ImageState& img, char* binning_blob, int P, int W, int H, const float* background,
                       const float* dL_dout_color, const KbackZeroArgs& zr, bool debug, cudaStream_t stream)
{
    const int gx = (W + LGR_TILE - 1) / LGR_TILE, gy = (H + LGR_TILE - 1) / LGR_TILE;
    {
        ProfScope ps(ST_BLEND_BWD, stream);
        const size_t bsmem = blend_back_smem_bytes(zr.P > 0, true);
        LGR_CUDA_TRY(cudaFuncSetAttribute(blend_backward_ring_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)blend_back_smem_bytes(true, true)));
        blend_backward_ring_kernel<true><<<gx * gy, BL_THREADS, bsmem, stream>>>(img.ranges, binning_blob, geo.num_rendered, W, H, gx, background,
                                                                                  img.final_T, img.n_contrib, dL_dout_color, geo.grad_acc, zr);
        LGR_LAUNCH_CHECK("blend_backward_ring_kernel<det>", debug, stream);
    }
    {
        ProfScope ps(ST_DET_GATHER, stream);
        det_gather_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, geo.tiles_kept, geo.offsets, binning_blob, geo.num_rendered, geo.grad_acc);
        LGR_LAUNCH_CHECK("det_gather_kernel", debug, stream);
    }
    return LGR_OK;
}

}  // namespace

extern "C" {

int lgr_abi_version(void) { return LGR_ABI_VERSION; }
const char* lgr_last_error(void) { return g_last_error.c_str(); }
uint64_t lgr_launch_count(void) { return g_launches.load(); }

int lgr_set_blend_mode(int mode)
{
    if (mode != 0 && mode != 1) {
        g_last_error = "lgr_set_blend_mode: 0 = ring kernels (default), 1 = round-1 kernels";
        return LGR_ERR_INVALID_ARG;
    }
    g_blend_mode = mode;
    return LGR_OK;
}

int lgr_set_binning_mode(int mode)
{
    if (mode < 0 || mode > 2) {
        g_last_error = "lgr_set_binning_mode: 0 = hand-written kernels, estimated blob size, 1 = hand-written kernels, exact blob size, 2 = library sorts (default)";
        return LGR_ERR_INVALID_ARG;
    }
    g_bin_mode = mode;
    return LGR_OK;
}

int lgr_set_deterministic(int on)
{
    g_det = on != 0;
    return LGR_OK;
}

int lgr_set_kback_mode(int mode)
{
    if (mode < 0 || mode > 2) {
        g_last_error = "lgr_set_kback_mode: 0 = rows cleared inside the blend backward + compacted K7+K8 (default), 1 = dense K7+K8 kernel, 2 = separate zero-fill kernel + compacted K7+K8";
        return LGR_ERR_INVALID_ARG;
    }
    g_kback_mode = mode;
    return LGR_OK;
}

int lgr_set_vq_mode(int mode)
{
    if (mode != 0 && mode != 1) {
        g_last_error = "lgr_set_vq_mode: 0 = tensor-core coarse pass + exact FP32 rescore (default), 1 = FP32 kernel only";
        return LGR_ERR_INVALID_ARG;
    }
    g_vq_mode = mode;
    return LGR_OK;
}

uint64_t lgr_binning_overflows(void) { return g_bin_overflows.load(); }
uint64_t lgr_forward_stream_syncs(void) { return g_forward_syncs.load(); }
void lgr_set_binning_estimate(uint64_t instances) { g_bin_hint.store((size_t)instances); }

int lgr_set_tile_culling(int on)
{
    const bool v = on != 0;
    LGR_CUDA_TRY(cudaMemcpyToSymbol(g_tile_cull_enabled, &v, sizeof(bool)));
    return LGR_OK;
}

int lgr_profile_enable(int on)
{
    std::lock_guard<std::mutex> l(g_prof_mutex);
    g_prof_on = on != 0;
    return LGR_OK;
}

int lgr_profile_stage_count(void) { return ST_COUNT; }
const char* lgr_profile_stage_name(int k) { return (k >= 0 && k < ST_COUNT) ? kStageNames[k] : ""; }

int lgr_profile_collect(double* ms_out, uint64_t* launches_out, int n)
{
    LGR_CUDA_TRY(cudaDeviceSynchronize());
    std::lock_guard<std::mutex> l(g_prof_mutex);
    for (const ProfRecord& r : g_prof_records) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
            g_prof_ms[r.stage] += ms;
            g_prof_n[r.stage] += 1;
        }
        g_prof_pool.push_back(r.a);
        g_prof_pool.push_back(r.b);
    }
    g_prof_records.clear();
    for (int k = 0; k < n && k < ST_COUNT; k++) {
        if (ms_out) ms_out[k] = g_prof_ms[k];
        if (launches_out) launches_out[k] = g_prof_n[k];
        g_prof_ms[k] = 0;
        g_prof_n[k] = 0;
    }
    return LGR_OK;
}

size_t lgr_geometry_layout(int P, size_t* out, int n_out)
{
    GeometryState g = carve_geometry(nullptr, (size_t)(P > 0 ? P : 1), g_bin_mode == 2);
    for (int k = 0; k < n_out && k < 8; k++) out[k] = g.offs[k];
    return g.total;
}

size_t lgr_image_layout(int width, int height, size_t* out, int n_out)
{
    ImageState s = carve_image(nullptr, width, height, g_bin_mode == 2);
    for (int k = 0; k < n_out && k < 3; k++) out[k] = s.offs[k];
    return s.total;
}

size_t lgr_binning_layout(int num_rendered, int width, int height, size_t* out, int n_out)
{
    BinningState b = carve_binning(nullptr, (size_t)(num_rendered > 0 ? num_rendered : 0), width, height, g_bin_mode == 2);
    for (int k = 0; k < n_out && k < 1; k++) out[k] = b.offs[k];
    return b.total;
}

int lgr_forward(const lgr_view* view, int P, int M, const float* means3D, const float* shs, const float* colors_precomp,
                const float* opacities, const float* scales, const float* rotations, const float* cov3D_precomp,
                lgr_alloc_fn geometry_alloc, void* geometry_user, lgr_alloc_fn binning_alloc, void* binning_user,
                lgr_alloc_fn image_alloc, void* image_user, float* out_color, int32_t* radii, int32_t* num_rendered, void* cuda_stream)
{
    return forward_impl(view, P, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, geometry_alloc,
                        geometry_user, binning_alloc, binning_user, image_alloc, image_user, out_color, nullptr, nullptr, radii,
                        num_rendered, cuda_stream, false);
}

int lgr_forward_count(const lgr_view* view, int P, int M, const float* means3D, const float* shs, const float* colors_precomp,
                      const float* opacities, const float* scales, const float* rotations, const float* cov3D_precomp,
                      lgr_alloc_fn geometry_alloc, void* geometry_user, lgr_alloc_fn binning_alloc, void* binning_user,
                      lgr_alloc_fn image_alloc, void* image_user, float* out_color, int32_t* gaussians_count, float* important_score,
                      int32_t* radii, int32_t* num_rendered, void* cuda_stream)
{
    return forward_impl(view, P, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, geometry_alloc,
                        geometry_user, binning_alloc, binning_user, image_alloc, image_user, out_color, gaussians_count,
                        important_score, radii, num_rendered, cuda_stream, true);
}

// the *_weight entry points: their sibling's contract plus blend_weight [P], which they require
static bool weight_present(const char* what, int P, const int64_t* blend_weight)
{
    if (P > 0 && !blend_weight) {
        g_last_error = std::string(what) + ": blend_weight missing";
        return false;
    }
    return true;
}

int lgr_forward_count_weight(const lgr_view* view, int P, int M, const float* means3D, const float* shs, const float* colors_precomp,
                             const float* opacities, const float* scales, const float* rotations, const float* cov3D_precomp,
                             lgr_alloc_fn geometry_alloc, void* geometry_user, lgr_alloc_fn binning_alloc, void* binning_user,
                             lgr_alloc_fn image_alloc, void* image_user, float* out_color, int32_t* gaussians_count, float* important_score,
                             int64_t* blend_weight, int32_t* radii, int32_t* num_rendered, void* cuda_stream)
{
    if (!weight_present("lgr_forward_count_weight", P, blend_weight)) return LGR_ERR_INVALID_ARG;
    return forward_impl(view, P, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, geometry_alloc,
                        geometry_user, binning_alloc, binning_user, image_alloc, image_user, out_color, gaussians_count,
                        important_score, radii, num_rendered, cuda_stream, true, nullptr, nullptr, blend_weight);
}

int lgr_backward(const lgr_view* v, int P, int M, int num_rendered, const float* means3D, const float* shs,
                 const float* colors_precomp, const float* scales, const float* rotations, const float* cov3D_precomp,
                 const int32_t* radii, char* geometry_blob, char* binning_blob, char* image_blob, const float* dL_dout_color,
                 float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity, float* dL_dmeans3D, float* dL_dcov3D, float* dL_dsh,
                 float* dL_dscales, float* dL_drotations, void* cuda_stream)
{
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    if (P == 0) return LGR_OK;
    if (!v || P < 0 || !means3D || !radii || !geometry_blob || !binning_blob || !image_blob || !dL_dout_color || !dL_dmeans2D ||
        !dL_dcolors || !dL_dopacity || !dL_dmeans3D || !dL_dcov3D || !dL_dscales || !dL_drotations || (M > 0 && !dL_dsh)) {
        g_last_error = "lgr_backward: missing required argument";
        return LGR_ERR_INVALID_ARG;
    }
    (void)colors_precomp;
    if (((uintptr_t)rotations & 15) || ((uintptr_t)shs & 15) || ((uintptr_t)dL_dsh & 15) || ((uintptr_t)dL_drotations & 15)) {
        g_last_error = "lgr_backward: rotations, shs, dL_dsh and dL_drotations must be 16-byte aligned";
        return LGR_ERR_INVALID_ARG;
    }
    if (g_det && !det_supported("lgr_backward")) return LGR_ERR_INVALID_ARG;
    const bool debug = v->debug != 0;
    const int W = v->image_width, H = v->image_height;
    const int gx = (W + LGR_TILE - 1) / LGR_TILE, gy = (H + LGR_TILE - 1) / LGR_TILE;
    GeometryState geo = carve_geometry(geometry_blob, (size_t)P, g_det != 0);
    ImageState img = carve_image(image_blob, W, H, false);
    BinningState bin = carve_binning(binning_blob, (size_t)(num_rendered > 0 ? num_rendered : 0), W, H, false);

    if (g_det) {
        const int st = blend_backward_det(geo, img, binning_blob, P, W, H, v->background, dL_dout_color, KbackZeroArgs{}, debug, stream);
        if (st != LGR_OK) return st;
    } else {
        ProfScope ps(ST_MEMSET, stream);
        LGR_CUDA_TRY(cudaMemsetAsync(geo.grad_acc, 0, sizeof(float) * ACC_STRIDE * (size_t)P, stream));
    }
    if (num_rendered > 0 && !g_det) {
        ProfScope ps(ST_BLEND_BWD, stream);
        if (g_blend_mode == 0) {
            LGR_CUDA_TRY(cudaFuncSetAttribute(blend_backward_ring_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)blend_back_smem_bytes()));
            // the host only knows the reference's num_rendered here; the number of LISTED instances (which fixes where the records
            // start inside the binning blob) sits in the geometry header on the device
            blend_backward_ring_kernel<false><<<gx * gy, BL_THREADS, blend_back_smem_bytes(), stream>>>(img.ranges, binning_blob, geo.num_rendered, W, H, gx,
                                                                                                   v->background, img.final_T, img.n_contrib,
                                                                                                   dL_dout_color, geo.grad_acc, KbackZeroArgs{});
        } else
            blend_backward_kernel<<<gx * gy, 256, 0, stream>>>(img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity, geo.rgb,
                                                                v->background, img.final_T, img.n_contrib, dL_dout_color, geo.grad_acc);
        LGR_LAUNCH_CHECK("blend_backward_kernel", debug, stream);
    }
    PreBackArgs a;
    a.P = P; a.D = v->sh_degree; a.M = M; a.W = W; a.H = H;
    a.fy = H / (2.0f * v->tan_fovy);
    a.fx = W / (2.0f * v->tan_fovx);
    a.tanx = v->tan_fovx; a.tany = v->tan_fovy; a.mod = v->scale_modifier;
    a.means3D = means3D; a.scales = scales; a.rotations = rotations; a.shs = shs;
    a.cov3D = cov3D_precomp ? cov3D_precomp : geo.cov3D;
    a.view = v->viewmatrix; a.proj = v->projmatrix; a.campos = v->campos;
    a.radii = radii; a.clamped = geo.clamped; a.acc = geo.grad_acc; a.conic_opacity = geo.conic_opacity;
    a.dL_dmeans2D = dL_dmeans2D; a.dL_dcolors = dL_dcolors; a.dL_dopacity = dL_dopacity; a.dL_dmeans3D = dL_dmeans3D;
    a.dL_dcov3D = dL_dcov3D; a.dL_dsh = dL_dsh; a.dL_dscales = dL_dscales; a.dL_drot = dL_drotations;
    {
        ProfScope ps(ST_PREPROCESS_BWD, stream);
        preprocess_backward_kernel<<<(P + 255) / 256, 256, 0, stream>>>(a);
    }
    LGR_LAUNCH_CHECK("preprocess_backward_kernel", debug, stream);
    return LGR_OK;
}

static int forward_raw_impl(const lgr_view* view, int P, int M, const lgr_raw_params* params, lgr_alloc_fn geometry_alloc,
                            void* geometry_user, lgr_alloc_fn binning_alloc, void* binning_user, lgr_alloc_fn image_alloc, void* image_user,
                            float* out_color, int32_t* gaussians_count, float* important_score, int64_t* blend_weight, int32_t* radii,
                            int32_t* num_rendered, void* cuda_stream)
{
    if (!params || M < 1) {
        g_last_error = "lgr_forward_raw: params missing or M < 1";
        return LGR_ERR_INVALID_ARG;
    }
    const bool count_mode = gaussians_count != nullptr;
    return forward_impl(view, P, M, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, geometry_alloc, geometry_user,
                        binning_alloc, binning_user, image_alloc, image_user, out_color, gaussians_count, important_score, radii,
                        num_rendered, cuda_stream, count_mode, params, nullptr, blend_weight);
}

int lgr_forward_raw(const lgr_view* view, int P, int M, const lgr_raw_params* params, lgr_alloc_fn geometry_alloc, void* geometry_user,
                    lgr_alloc_fn binning_alloc, void* binning_user, lgr_alloc_fn image_alloc, void* image_user, float* out_color,
                    int32_t* gaussians_count, float* important_score, int32_t* radii, int32_t* num_rendered, void* cuda_stream)
{
    return forward_raw_impl(view, P, M, params, geometry_alloc, geometry_user, binning_alloc, binning_user, image_alloc, image_user, out_color,
                            gaussians_count, important_score, nullptr, radii, num_rendered, cuda_stream);
}

int lgr_forward_raw_weight(const lgr_view* view, int P, int M, const lgr_raw_params* params, lgr_alloc_fn geometry_alloc, void* geometry_user,
                           lgr_alloc_fn binning_alloc, void* binning_user, lgr_alloc_fn image_alloc, void* image_user, float* out_color,
                           int32_t* gaussians_count, float* important_score, int64_t* blend_weight, int32_t* radii, int32_t* num_rendered,
                           void* cuda_stream)
{
    if (!weight_present("lgr_forward_raw_weight", P, blend_weight)) return LGR_ERR_INVALID_ARG;
    return forward_raw_impl(view, P, M, params, geometry_alloc, geometry_user, binning_alloc, binning_user, image_alloc, image_user, out_color,
                            gaussians_count, important_score, blend_weight, radii, num_rendered, cuda_stream);
}

static int forward_vq_impl(const lgr_view* view, int P, const lgr_vq_resident_params* params, lgr_alloc_fn geometry_alloc, void* geometry_user,
                           lgr_alloc_fn binning_alloc, void* binning_user, lgr_alloc_fn image_alloc, void* image_user, float* out_color,
                           int32_t* gaussians_count, float* important_score, int64_t* blend_weight, int32_t* radii, int32_t* num_rendered,
                           void* cuda_stream)
{
    const lgr_vq_resident_params* q = params;
    if (!q || q->D < 3 || q->D % 3 != 0 || q->D > 48 || q->Dp < q->D || q->Dp % 8 != 0 || q->K < 1) {
        g_last_error = "lgr_forward_vq: params missing, or D not 3*(degree+1)^2 <= 48, or Dp not a multiple of 8 >= D, or K < 1";
        return LGR_ERR_INVALID_ARG;
    }
    const int M = q->D / 3;
    if (M != 1 && M != 4 && M != 9 && M != 16) {
        g_last_error = "lgr_forward_vq: D must be 3*(degree+1)^2";
        return LGR_ERR_INVALID_ARG;
    }
    if ((gaussians_count == nullptr) != (important_score == nullptr)) {
        g_last_error = "lgr_forward_vq: gaussians_count and important_score must both be NULL or both be set";
        return LGR_ERR_INVALID_ARG;
    }
    if (P > 0) {
        const void* dev[] = {q->xyz, q->attr, q->slot, q->codebook, q->nonvq};
        for (int k = 0; k < 5; k++) {
            if (!dev[k]) {
                if (k == 4) continue;  // no non-VQ rows (vq_ratio 1)
                g_last_error = "lgr_forward_vq: xyz, attr, slot and codebook are required";
                return LGR_ERR_INVALID_ARG;
            }
            cudaPointerAttributes at;
            if (cudaPointerGetAttributes(&at, dev[k]) != cudaSuccess || at.type != cudaMemoryTypeDevice) {
                cudaGetLastError();
                g_last_error = "lgr_forward_vq: every array must be device memory";
                return LGR_ERR_INVALID_ARG;
            }
            if ((uintptr_t)dev[k] & 15) {
                g_last_error = "lgr_forward_vq: every array must be 16-byte aligned";
                return LGR_ERR_INVALID_ARG;
            }
        }
    }
    return forward_impl(view, P, M, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, geometry_alloc, geometry_user,
                        binning_alloc, binning_user, image_alloc, image_user, out_color, gaussians_count, important_score, radii,
                        num_rendered, cuda_stream, gaussians_count != nullptr, nullptr, q, blend_weight);
}

int lgr_forward_vq(const lgr_view* view, int P, const lgr_vq_resident_params* params, lgr_alloc_fn geometry_alloc, void* geometry_user,
                   lgr_alloc_fn binning_alloc, void* binning_user, lgr_alloc_fn image_alloc, void* image_user, float* out_color,
                   int32_t* gaussians_count, float* important_score, int32_t* radii, int32_t* num_rendered, void* cuda_stream)
{
    return forward_vq_impl(view, P, params, geometry_alloc, geometry_user, binning_alloc, binning_user, image_alloc, image_user, out_color,
                           gaussians_count, important_score, nullptr, radii, num_rendered, cuda_stream);
}

int lgr_forward_vq_weight(const lgr_view* view, int P, const lgr_vq_resident_params* params, lgr_alloc_fn geometry_alloc, void* geometry_user,
                          lgr_alloc_fn binning_alloc, void* binning_user, lgr_alloc_fn image_alloc, void* image_user, float* out_color,
                          int32_t* gaussians_count, float* important_score, int64_t* blend_weight, int32_t* radii, int32_t* num_rendered,
                          void* cuda_stream)
{
    if (!weight_present("lgr_forward_vq_weight", P, blend_weight)) return LGR_ERR_INVALID_ARG;
    return forward_vq_impl(view, P, params, geometry_alloc, geometry_user, binning_alloc, binning_user, image_alloc, image_user, out_color,
                           gaussians_count, important_score, blend_weight, radii, num_rendered, cuda_stream);
}

// lgr_backward_raw (one call for both stages, dense outputs) asks stage 1 to clear the gradient rows from inside the blend backward
thread_local KbackZeroArgs t_zero_req = {};
thread_local bool t_rows_zeroed = false;

// stage 1 of the raw backward: clear the accumulators, blend backward, optionally extract this view's dL/dRGB.  db: the depth variant
// of the blend backward (lgr_backward_raw_depth; the caller refused deterministic mode and blend mode 1)
// absgrad: the absgrad variant of the blend backward (lgr_backward_raw_absgrad; the caller refused deterministic mode and blend mode 1)
// adds the statistic into absgrad[P,2], which this function clears
static int backward_raw_begin_impl(const lgr_view* v, int P, int num_rendered, const int32_t* radii, char* geometry_blob, char* binning_blob,
                                   char* image_blob, const float* dL_dout_color, float* d_rgb, void* cuda_stream, const BlendDepthBack* db,
                                   float* absgrad = nullptr)
{
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    if (P == 0) return LGR_OK;
    if (!v || P < 0 || !radii || !geometry_blob || !binning_blob || !image_blob || !dL_dout_color) {
        g_last_error = "lgr_backward_raw_begin: missing required argument";
        return LGR_ERR_INVALID_ARG;
    }
    if (g_det && !det_supported("lgr_backward_raw")) { t_zero_req.P = 0; return LGR_ERR_INVALID_ARG; }
    const bool debug = v->debug != 0;
    const int W = v->image_width, H = v->image_height;
    const int gx = (W + LGR_TILE - 1) / LGR_TILE, gy = (H + LGR_TILE - 1) / LGR_TILE;
    GeometryState geo = carve_geometry(geometry_blob, (size_t)P, g_det != 0);
    ImageState img = carve_image(image_blob, W, H, false);
    BinningState bin = carve_binning(binning_blob, (size_t)(num_rendered > 0 ? num_rendered : 0), W, H, false);
    if (g_det) {
        const KbackZeroArgs zr = t_zero_req;
        t_zero_req.P = 0;
        const int st = blend_backward_det(geo, img, binning_blob, P, W, H, v->background, dL_dout_color, zr, debug, stream);
        if (st != LGR_OK) return st;
        t_rows_zeroed = zr.P > 0;
    } else {
        ProfScope ps(ST_MEMSET, stream);
        LGR_CUDA_TRY(cudaMemsetAsync(geo.grad_acc, 0, sizeof(float) * ACC_STRIDE * (size_t)P, stream));
        if (absgrad) LGR_CUDA_TRY(cudaMemsetAsync(absgrad, 0, sizeof(float) * 2 * (size_t)P, stream));
    }
    if (num_rendered > 0 && !g_det) {
        ProfScope ps(ST_BLEND_BWD, stream);
        if (g_blend_mode == 0) {
            LGR_CUDA_TRY(cudaFuncSetAttribute(blend_backward_ring_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)blend_back_smem_bytes()));
            // the host only knows the reference's num_rendered here; the number of LISTED instances (which fixes where the records
            // start inside the binning blob) sits in the geometry header on the device
            const KbackZeroArgs zr = t_zero_req;
            t_zero_req.P = 0;
            const size_t bsmem = blend_back_smem_bytes(zr.P > 0);
            if (absgrad) {
                LGR_CUDA_TRY(cudaFuncSetAttribute(blend_backward_absgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  (int)blend_back_smem_bytes(true, false, true)));
                blend_backward_absgrad_kernel<<<gx * gy, BL_THREADS, blend_back_smem_bytes(zr.P > 0, false, true), stream>>>(
                    img.ranges, binning_blob, geo.num_rendered, W, H, gx, v->background, img.final_T, img.n_contrib, dL_dout_color,
                    geo.grad_acc, zr, absgrad, P);
            } else if (db) {
                LGR_CUDA_TRY(cudaFuncSetAttribute(blend_backward_ring_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  (int)blend_back_smem_bytes(true)));
                blend_backward_ring_kernel<false, true><<<gx * gy, BL_THREADS, bsmem, stream>>>(img.ranges, binning_blob, geo.num_rendered, W, H, gx,
                                                                                             v->background, img.final_T, img.n_contrib,
                                                                                             dL_dout_color, geo.grad_acc, zr, *db);
            } else {
                LGR_CUDA_TRY(cudaFuncSetAttribute(blend_backward_ring_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)blend_back_smem_bytes(true)));
                blend_backward_ring_kernel<false><<<gx * gy, BL_THREADS, bsmem, stream>>>(img.ranges, binning_blob, geo.num_rendered, W, H, gx,
                                                                                     v->background, img.final_T, img.n_contrib,
                                                                                     dL_dout_color, geo.grad_acc, zr);
            }
            t_rows_zeroed = zr.P > 0;
        } else
            blend_backward_kernel<<<gx * gy, 256, 0, stream>>>(img.ranges, bin.point_list, W, H, gx, geo.means2D, geo.conic_opacity, geo.rgb,
                                                                v->background, img.final_T, img.n_contrib, dL_dout_color, geo.grad_acc);
        LGR_LAUNCH_CHECK("blend_backward_kernel", debug, stream);
    }
    if (d_rgb) {
        extract_drgb_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, radii, geo.clamped, geo.grad_acc, d_rgb);
        LGR_LAUNCH_CHECK("extract_drgb_kernel", debug, stream);
    }
    return LGR_OK;
}

int lgr_backward_raw_begin(const lgr_view* v, int P, int num_rendered, const int32_t* radii, char* geometry_blob, char* binning_blob,
                           char* image_blob, const float* dL_dout_color, float* d_rgb, void* cuda_stream)
{
    return backward_raw_begin_impl(v, P, num_rendered, radii, geometry_blob, binning_blob, image_blob, dL_dout_color, d_rgb, cuda_stream, nullptr);
}

// stage 2: the per-Gaussian backward (K7+K8 with the activation chain rules) from the accumulators left by stage 1
int lgr_backward_raw_end(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                         const lgr_raw_grads* grads, float* dL_dmeans2D, void* cuda_stream)
{
    return lgr_backward_raw_end_range(v, P, M, params, radii, geometry_blob, grads, dL_dmeans2D, 0, P, cuda_stream);
}

// camera gradients of one backward (lgr_backward_raw_camera): K7+K8 writes one 27-float row per block into `rows` ([27][nrows]) and
// records how many it wrote; a call that launches no K7+K8 leaves nrows at 0
struct CamGrad {
    float* rows;
    int nrows;
};

// the same for Gaussians [first, first+count) only; first must be a multiple of 256.  Lets the caller start exchanging the gradients
// of one range while the next range is still being computed.  rd: the depth variant of K7+K8 (lgr_backward_raw_depth, whole view).
// cg: the camera variant of K7+K8 (lgr_backward_raw_camera, whole view); in deterministic mode it takes the dense kernel, whose block
// rows follow the Gaussian index order
static int backward_raw_end_impl(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                                 const lgr_raw_grads* grads, float* dL_dmeans2D, int first, int count, void* cuda_stream, const RawDepth* rd,
                                 CamGrad* cg = nullptr)
{
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    if (P == 0 || count == 0) return LGR_OK;
    if (first < 0 || count < 0 || (first & 255) || first + (long long)count > P) {
        g_last_error = "lgr_backward_raw_end_range: the range must start at a multiple of 256 and lie inside [0, P)";
        return LGR_ERR_INVALID_ARG;
    }
    const bool compact = grads && grads->features_rest == nullptr;
    if (!v || P < 0 || M < 1 || !params || !grads || !radii || !geometry_blob || !dL_dmeans2D || !grads->xyz ||
        (!compact && (!grads->features_dc || (M > 1 && !grads->features_rest))) || !grads->scaling || !grads->rotation || !grads->opacity) {
        g_last_error = "lgr_backward_raw: missing required argument";
        return LGR_ERR_INVALID_ARG;
    }
    if (((uintptr_t)params->rotation & 15) || ((uintptr_t)grads->rotation & 15) || ((uintptr_t)params->features_rest & 15) ||
        ((uintptr_t)params->features_dc & 15) || ((uintptr_t)grads->features_rest & 15) || ((uintptr_t)grads->features_dc & 15)) {
        g_last_error = "lgr_backward_raw: rotation / features tensors and their gradients must be 16-byte aligned";
        return LGR_ERR_INVALID_ARG;
    }
    const bool debug = v->debug != 0;
    const int W = v->image_width, H = v->image_height;
    GeometryState geo = carve_geometry(geometry_blob, (size_t)P, false);
    RawBackArgs a;
    a.P = P; a.D = v->sh_degree; a.M = M; a.W = W; a.H = H;
    a.fy = H / (2.0f * v->tan_fovy);
    a.fx = W / (2.0f * v->tan_fovx);
    a.tanx = v->tan_fovx; a.tany = v->tan_fovy; a.mod = v->scale_modifier;
    a.xyz = params->xyz; a.dc = params->features_dc; a.rest = params->features_rest; a.scaling = params->scaling;
    a.rotation = params->rotation; a.cov3D = geo.cov3D; a.conic_opacity = geo.conic_opacity;
    a.view = v->viewmatrix; a.proj = v->projmatrix; a.campos = v->campos;
    a.radii = radii; a.clamped = geo.clamped; a.acc = geo.grad_acc;
    a.d_xyz = grads->xyz; a.d_dc = grads->features_dc; a.d_rest = grads->features_rest; a.d_scaling = grads->scaling;
    a.d_rotation = grads->rotation; a.d_opacity = grads->opacity; a.dL_dmeans2D = dL_dmeans2D;
    a.d_rgb = grads->rgb;
    if (!raw_rest_stride_ok(params, M)) {
        g_last_error = "lgr_backward_raw: features_rest_row_stride must be 0 (dense) or in [(M-1)*3, 256]";
        return LGR_ERR_INVALID_ARG;
    }
    a.rest_stride = raw_rest_stride(params, M);
    a.block0 = first / 256;
    a.P = first + count;                       // the kernel's bound check: blocks of this launch never run past the range
    if (compact) { a.d_rest = nullptr; a.d_dc = nullptr; }
    const bool rows_zeroed = t_rows_zeroed;
    t_rows_zeroed = false;
    if (!compact && first == 0 && count == P && g_kback_mode != 1 && !(cg && g_det)) {
        // whole view, dense outputs: zero-fill (unless the blend backward already did it) + flag, then K7+K8 on the compacted list of
        // Gaussians with a non-zero gradient (lgr_sparse.cuh).  The id list reuses sorted_ids (dead after the forward's binning), the
        // count a header word.
        ProfScope ps(ST_PREPROCESS_BWD, stream);
        int* counter = geo.num_rendered + HDR_LIVE;
        LGR_CUDA_TRY(cudaMemsetAsync(counter, 0, sizeof(int), stream));
        KbackZeroArgs z;
        z.P = P; z.nrest = (M - 1) * 3; z.radii = radii; z.acc = geo.grad_acc; z.idx = reinterpret_cast<int*>(geo.sorted_ids); z.counter = counter;
        z.d_xyz = a.d_xyz; z.d_dc = a.d_dc; z.d_rest = a.d_rest; z.d_scaling = a.d_scaling; z.d_rotation = a.d_rotation; z.d_opacity = a.d_opacity;
        z.dL_dmeans2D = dL_dmeans2D;
        if (M == 1) z.d_rest = a.d_dc;   // no rest coefficients: nrest = 0, pointer unused
        if (rd && rows_zeroed) kback_zero_flag_depth_kernel<false><<<(P + 255) / 256, 256, 0, stream>>>(z);
        else if (rd) kback_zero_flag_depth_kernel<true><<<(P + 255) / 256, 256, 0, stream>>>(z);
        else if (rows_zeroed) kback_zero_flag_kernel<false><<<(P + 255) / 256, 256, 0, stream>>>(z);
        else kback_zero_flag_kernel<true><<<(P + 255) / 256, 256, 0, stream>>>(z);
        LGR_LAUNCH_CHECK("kback_zero_flag_kernel", debug, stream);
        a.P = P;
        const int blocks = std::min((P + KC_THREADS - 1) / KC_THREADS, LGR_SMS * 8);
        if (cg) {
            cg->nrows = blocks;
            if (rd)
                preprocess_backward_compact_depth_cam_kernel<<<blocks, KC_THREADS, 0, stream>>>(a, reinterpret_cast<const int*>(geo.sorted_ids), counter,
                                                                                                *rd, cg->rows);
            else
                preprocess_backward_compact_cam_kernel<<<blocks, KC_THREADS, 0, stream>>>(a, reinterpret_cast<const int*>(geo.sorted_ids), counter,
                                                                                          cg->rows);
        } else if (rd)
            preprocess_backward_compact_depth_kernel<<<blocks, KC_THREADS, 0, stream>>>(a, reinterpret_cast<const int*>(geo.sorted_ids), counter, *rd);
        else
            preprocess_backward_compact_kernel<<<blocks, KC_THREADS, 0, stream>>>(a, reinterpret_cast<const int*>(geo.sorted_ids), counter);
        LGR_LAUNCH_CHECK("preprocess_backward_compact_kernel", debug, stream);
        return LGR_OK;
    }
    const size_t smem = raw_smem_bytes(M);
    if (cg) {
        const int blocks = (count + 255) / 256;
        cg->nrows = blocks;
        ProfScope ps(ST_PREPROCESS_BWD, stream);
        if (rd) {
            LGR_CUDA_TRY(cudaFuncSetAttribute(preprocess_backward_raw_depth_cam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            preprocess_backward_raw_depth_cam_kernel<<<blocks, 256, smem, stream>>>(a, *rd, cg->rows);
        } else {
            LGR_CUDA_TRY(cudaFuncSetAttribute(preprocess_backward_raw_cam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            preprocess_backward_raw_cam_kernel<<<blocks, 256, smem, stream>>>(a, cg->rows);
        }
    } else if (rd) {
        LGR_CUDA_TRY(cudaFuncSetAttribute(preprocess_backward_raw_depth_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ProfScope ps(ST_PREPROCESS_BWD, stream);
        preprocess_backward_raw_depth_kernel<<<(count + 255) / 256, 256, smem, stream>>>(a, *rd);
    } else {
        LGR_CUDA_TRY(cudaFuncSetAttribute(preprocess_backward_raw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ProfScope ps(ST_PREPROCESS_BWD, stream);
        preprocess_backward_raw_kernel<<<(count + 255) / 256, 256, smem, stream>>>(a);
    }
    LGR_LAUNCH_CHECK("preprocess_backward_raw_kernel", debug, stream);
    return LGR_OK;
}

int lgr_backward_raw_end_range(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                               const lgr_raw_grads* grads, float* dL_dmeans2D, int first, int count, void* cuda_stream)
{
    return backward_raw_end_impl(v, P, M, params, radii, geometry_blob, grads, dL_dmeans2D, first, count, cuda_stream, nullptr);
}

static int backward_raw_impl(const lgr_view* v, int P, int M, int num_rendered, const lgr_raw_params* params, const int32_t* radii,
                             char* geometry_blob, char* binning_blob, char* image_blob, const float* dL_dout_color, const lgr_raw_grads* grads,
                             float* dL_dmeans2D, void* cuda_stream, const BlendDepthBack* db, const RawDepth* rd, float* absgrad = nullptr,
                             CamGrad* cg = nullptr)
{
    t_zero_req.P = 0;
    t_rows_zeroed = false;
    if (g_kback_mode == 0 && g_blend_mode == 0 && P > 0 && M >= 1 && grads && grads->features_rest != nullptr && grads->features_dc && grads->xyz &&
        grads->scaling && grads->rotation && grads->opacity && dL_dmeans2D &&
        !(((uintptr_t)grads->xyz | (uintptr_t)grads->features_dc | (uintptr_t)grads->features_rest | (uintptr_t)grads->scaling |
           (uintptr_t)grads->rotation | (uintptr_t)grads->opacity | (uintptr_t)dL_dmeans2D) & 15)) {
        // dense outputs: the blend backward's producer thread clears the rows (runs of 4 Gaussians are 16-byte multiples in every tensor)
        KbackZeroArgs& z = t_zero_req;
        z.P = P; z.nrest = (M - 1) * 3; z.radii = nullptr; z.acc = nullptr; z.idx = nullptr; z.counter = nullptr;
        z.d_xyz = grads->xyz; z.d_dc = grads->features_dc; z.d_rest = grads->features_rest; z.d_scaling = grads->scaling;
        z.d_rotation = grads->rotation; z.d_opacity = grads->opacity; z.dL_dmeans2D = dL_dmeans2D;
    }
    const int st = backward_raw_begin_impl(v, P, num_rendered, radii, geometry_blob, binning_blob, image_blob, dL_dout_color, nullptr, cuda_stream, db,
                                           absgrad);
    t_zero_req.P = 0;
    if (st != LGR_OK) { t_rows_zeroed = false; return st; }
    return backward_raw_end_impl(v, P, M, params, radii, geometry_blob, grads, dL_dmeans2D, 0, P, cuda_stream, rd, cg);
}

int lgr_backward_raw(const lgr_view* v, int P, int M, int num_rendered, const lgr_raw_params* params, const int32_t* radii,
                     char* geometry_blob, char* binning_blob, char* image_blob, const float* dL_dout_color, const lgr_raw_grads* grads,
                     float* dL_dmeans2D, void* cuda_stream)
{
    return backward_raw_impl(v, P, M, num_rendered, params, radii, geometry_blob, binning_blob, image_blob, dL_dout_color, grads, dL_dmeans2D,
                             cuda_stream, nullptr, nullptr);
}

// ---- depth and alpha planes (DESIGN section 7) ----
static bool depth_request_ok(const char* what, int depth_mode, bool depth_plane)
{
    if (depth_mode < 0 || depth_mode > 2) {
        g_last_error = std::string(what) + ": depth_mode must be 0 (none), 1 (z) or 2 (inverse)";
        return false;
    }
    if (depth_plane && depth_mode == 0) {
        g_last_error = std::string(what) + ": a depth plane needs depth_mode 1 (z) or 2 (inverse)";
        return false;
    }
    if (g_det) {
        g_last_error = std::string(what) + ": deterministic mode has no depth or alpha output";
        return false;
    }
    if (g_blend_mode != 0) {
        g_last_error = std::string(what) + ": depth and alpha need the ring blend kernels; lgr_set_blend_mode(1) has no depth output";
        return false;
    }
    return true;
}

int lgr_forward_raw_depth(const lgr_view* view, int P, int M, const lgr_raw_params* params, lgr_alloc_fn geometry_alloc, void* geometry_user,
                          lgr_alloc_fn binning_alloc, void* binning_user, lgr_alloc_fn image_alloc, void* image_user, float* out_color,
                          int32_t* gaussians_count, float* important_score, int depth_mode, float* out_depth, float* out_alpha,
                          int32_t* radii, int32_t* num_rendered, void* cuda_stream)
{
    if (!out_depth && !out_alpha)
        return lgr_forward_raw(view, P, M, params, geometry_alloc, geometry_user, binning_alloc, binning_user, image_alloc, image_user,
                               out_color, gaussians_count, important_score, radii, num_rendered, cuda_stream);
    if (!depth_request_ok("lgr_forward_raw_depth", depth_mode, out_depth != nullptr)) return LGR_ERR_INVALID_ARG;
    if (!params || M < 1) {
        g_last_error = "lgr_forward_raw_depth: params missing or M < 1";
        return LGR_ERR_INVALID_ARG;
    }
    BlendDepth dz = {};
    dz.depth = out_depth;
    dz.alpha = out_alpha;
    dz.mode = depth_mode;
    return forward_impl(view, P, M, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, geometry_alloc, geometry_user,
                        binning_alloc, binning_user, image_alloc, image_user, out_color, gaussians_count, important_score, radii,
                        num_rendered, cuda_stream, gaussians_count != nullptr, params, nullptr, nullptr, &dz);
}

int lgr_backward_raw_depth(const lgr_view* v, int P, int M, int num_rendered, const lgr_raw_params* params, const int32_t* radii,
                           char* geometry_blob, char* binning_blob, char* image_blob, const float* dL_dout_color, int depth_mode,
                           const float* dL_ddepth, const float* dL_dalpha, const lgr_raw_grads* grads, float* dL_dmeans2D, void* cuda_stream)
{
    if (!dL_ddepth && !dL_dalpha)
        return lgr_backward_raw(v, P, M, num_rendered, params, radii, geometry_blob, binning_blob, image_blob, dL_dout_color, grads,
                                dL_dmeans2D, cuda_stream);
    if (!depth_request_ok("lgr_backward_raw_depth", depth_mode, dL_ddepth != nullptr)) return LGR_ERR_INVALID_ARG;
    if (P == 0) return LGR_OK;
    if (!geometry_blob) {
        g_last_error = "lgr_backward_raw_depth: missing required argument";
        return LGR_ERR_INVALID_ARG;
    }
    const BlendDepthBack db = {dL_ddepth, dL_dalpha, 1 + depth_mode, P};
    const RawDepth rd = {carve_geometry(geometry_blob, (size_t)P, false).depth, depth_mode};
    return backward_raw_impl(v, P, M, num_rendered, params, radii, geometry_blob, binning_blob, image_blob, dL_dout_color, grads, dL_dmeans2D,
                             cuda_stream, &db, &rd);
}

// ---- absolute-gradient densification statistic (DESIGN section 7) ----
int lgr_backward_raw_absgrad(const lgr_view* v, int P, int M, int num_rendered, const lgr_raw_params* params, const int32_t* radii,
                             char* geometry_blob, char* binning_blob, char* image_blob, const float* dL_dout_color, const lgr_raw_grads* grads,
                             float* dL_dmeans2D, float* dL_dmeans2D_abs, void* cuda_stream)
{
    if (g_det) {
        g_last_error = "lgr_backward_raw_absgrad: deterministic mode has no absgrad output (it needs fixed-order sums)";
        return LGR_ERR_INVALID_ARG;
    }
    if (g_blend_mode != 0) {
        g_last_error = "lgr_backward_raw_absgrad: absgrad needs the ring blend kernels; lgr_set_blend_mode(1) has no absgrad output";
        return LGR_ERR_INVALID_ARG;
    }
    if (P == 0) return LGR_OK;
    if (P < 0 || !dL_dmeans2D_abs || ((uintptr_t)dL_dmeans2D_abs & 7)) {
        g_last_error = "lgr_backward_raw_absgrad: dL_dmeans2D_abs must be an 8-byte aligned [P,2] float32 device array";
        return LGR_ERR_INVALID_ARG;
    }
    if (num_rendered <= 0) {   // no pair: the blend backward does not run, so the statistic is cleared here
        LGR_CUDA_TRY(cudaMemsetAsync(dL_dmeans2D_abs, 0, sizeof(float) * 2 * (size_t)P, static_cast<cudaStream_t>(cuda_stream)));
    }
    return backward_raw_impl(v, P, M, num_rendered, params, radii, geometry_blob, binning_blob, image_blob, dL_dout_color, grads, dL_dmeans2D,
                             cuda_stream, nullptr, nullptr, num_rendered > 0 ? dL_dmeans2D_abs : nullptr);
}

// ---- camera gradients (DESIGN section 7) ----
// block rows of the larger of the two K7+K8 grids: the dense kernel's (one block per 256 Gaussians) and the compacted kernel's
size_t lgr_camera_grad_workspace_bytes(int P)
{
    if (P <= 0) return 256;
    const size_t rows = (size_t)std::max((P + 255) / 256, std::min((P + KC_THREADS - 1) / KC_THREADS, LGR_SMS * 8));
    return align_up(rows * CAM_TERMS * sizeof(float), 256);
}

int lgr_backward_raw_camera(const lgr_view* v, int P, int M, int num_rendered, const lgr_raw_params* params, const int32_t* radii,
                            char* geometry_blob, char* binning_blob, char* image_blob, const float* dL_dout_color, int depth_mode,
                            const float* dL_ddepth, const float* dL_dalpha, const lgr_raw_grads* grads, float* dL_dmeans2D,
                            float* dL_dviewmatrix, float* dL_dprojmatrix, float* dL_dcampos, void* workspace, size_t workspace_bytes,
                            void* cuda_stream)
{
    const bool planes = dL_ddepth || dL_dalpha;
    if (planes && !depth_request_ok("lgr_backward_raw_camera", depth_mode, dL_ddepth != nullptr)) return LGR_ERR_INVALID_ARG;
    if (P < 0 || !dL_dviewmatrix || !dL_dprojmatrix || !dL_dcampos || !workspace || workspace_bytes < lgr_camera_grad_workspace_bytes(P) ||
        ((uintptr_t)workspace & 3)) {
        g_last_error = "lgr_backward_raw_camera: the three camera outputs and a 4-byte aligned workspace of lgr_camera_grad_workspace_bytes(P) "
                       "bytes are required";
        return LGR_ERR_INVALID_ARG;
    }
    if (planes && P > 0 && !geometry_blob) {
        g_last_error = "lgr_backward_raw_camera: missing required argument";
        return LGR_ERR_INVALID_ARG;
    }
    BlendDepthBack db = {};
    RawDepth rd = {};
    if (planes && P > 0) {
        db = {dL_ddepth, dL_dalpha, 1 + depth_mode, P};
        rd = {carve_geometry(geometry_blob, (size_t)P, false).depth, depth_mode};
    }
    CamGrad cg = {static_cast<float*>(workspace), 0};
    const int st = backward_raw_impl(v, P, M, num_rendered, params, radii, geometry_blob, binning_blob, image_blob, dL_dout_color, grads,
                                     dL_dmeans2D, cuda_stream, planes ? &db : nullptr, planes ? &rd : nullptr, nullptr, &cg);
    if (st != LGR_OK) return st;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    {
        ProfScope ps(ST_CAMERA_FINISH, stream);
        camera_grad_finish_kernel<<<1, 1024, 0, stream>>>(cg.rows, cg.nrows, dL_dviewmatrix, dL_dprojmatrix, dL_dcampos);
    }
    LGR_LAUNCH_CHECK("camera_grad_finish_kernel", v && v->debug != 0, stream);
    return LGR_OK;
}

// ---- sparse view-parallel exchange (lgr_sparse.cuh) ----
size_t lgr_sparse_exchange_bytes(int P) { return P > 0 ? sparse_layout(P).total * 4 : 256; }

static size_t sparse_scan_bytes(int P)
{
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum((void*)nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (P + 31) / 32);
    return bytes;
}

size_t lgr_sparse_workspace_bytes(int P)
{
    if (P <= 0) return 256;
    return align_up((size_t)((P + 31) / 32) * 4, 256) + align_up((size_t)P * 4, 256) + align_up(sparse_scan_bytes(P), 256) + 256;
}

int lgr_backward_raw_sparse_pack(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                                 void* exchange_buffer, void* workspace, float* dL_dmeans2D, void* cuda_stream)
{
    void* only[1] = {exchange_buffer};
    return lgr_backward_raw_sparse_pack_push(v, P, M, params, radii, geometry_blob, only, 1, 0, workspace, dL_dmeans2D, cuda_stream);
}

// push mode: slot_of_this_rank[r] = this rank's slot inside the exchange buffer of rank r (peer-mapped for r != self); the packed view
// (header, bitmap, prefix, rows) lands in all of them, so that after ONE cross-GPU barrier every rank accumulates from LOCAL memory.
int lgr_backward_raw_sparse_pack_push(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                                      void* const* slot_of_this_rank, int world, int self, void* workspace, float* dL_dmeans2D,
                                      void* cuda_stream)
{
    return lgr_backward_raw_sparse_pack_push_ex(v, P, M, params, radii, geometry_blob, slot_of_this_rank, world, self, workspace, dL_dmeans2D,
                                                nullptr, cuda_stream);
}

size_t lgr_sparse_exchange_bytes_stats(int P) { return P > 0 ? sparse_layout(P).total_stats * 4 : 256; }

// stats != NULL: the slots are lgr_sparse_exchange_bytes_stats(P) bytes and also carry the densification statistics (lgr_sparse.cuh)
int lgr_backward_raw_sparse_pack_push_ex(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                                         void* const* slot_of_this_rank, int world, int self, void* workspace, float* dL_dmeans2D,
                                         const lgr_sparse_stats* stats, void* cuda_stream)
{
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    if (P == 0) return LGR_OK;
    if (!v || P < 0 || M < 1 || !params || !radii || !geometry_blob || !slot_of_this_rank || world < 1 || world > 8 || self < 0 || self >= world ||
        !workspace || !dL_dmeans2D || ((uintptr_t)workspace & 255) || ((uintptr_t)params->rotation & 15)) {
        g_last_error = "lgr_backward_raw_sparse_pack: missing argument, more than 8 ranks, or misaligned buffer (exchange buffers and workspace: 256 bytes)";
        return LGR_ERR_INVALID_ARG;
    }
    SparsePush push;
    memset(&push, 0, sizeof(push));
    push.n = world;
    for (int r = 0; r < world; r++) {
        if (!slot_of_this_rank[r] || ((uintptr_t)slot_of_this_rank[r] & 255)) {
            g_last_error = "lgr_backward_raw_sparse_pack: exchange slot missing or not 256-byte aligned";
            return LGR_ERR_INVALID_ARG;
        }
        push.dst[r] = static_cast<uint32_t*>(slot_of_this_rank[r]);
    }
    const bool debug = v->debug != 0;
    const int W = v->image_width, H = v->image_height;
    GeometryState geo = carve_geometry(geometry_blob, (size_t)P, false);
    const SparseLayout L = sparse_layout(P);
    uint32_t* xb = push.dst[self];
    const int w32 = (P + 31) / 32;
    char* ws = static_cast<char*>(workspace);
    uint32_t* popc = reinterpret_cast<uint32_t*>(ws);
    int* idx = reinterpret_cast<int*>(ws + align_up((size_t)w32 * 4, 256));
    void* cub_tmp = ws + align_up((size_t)w32 * 4, 256) + align_up((size_t)P * 4, 256);
    size_t cub_bytes = sparse_scan_bytes(P);
    RawBackArgs a;
    memset(&a, 0, sizeof(a));
    a.P = P; a.D = v->sh_degree; a.M = M; a.W = W; a.H = H;
    a.fy = H / (2.0f * v->tan_fovy);
    a.fx = W / (2.0f * v->tan_fovx);
    a.tanx = v->tan_fovx; a.tany = v->tan_fovy; a.mod = v->scale_modifier;
    a.xyz = params->xyz; a.dc = params->features_dc; a.rest = params->features_rest; a.scaling = params->scaling;
    a.rotation = params->rotation; a.cov3D = geo.cov3D; a.conic_opacity = geo.conic_opacity;
    a.view = v->viewmatrix; a.proj = v->projmatrix; a.campos = v->campos;
    a.radii = radii; a.clamped = geo.clamped; a.acc = geo.grad_acc;
    a.dL_dmeans2D = dL_dmeans2D;
    if (!raw_rest_stride_ok(params, M)) {
        g_last_error = "lgr_backward_raw_sparse_pack: features_rest_row_stride must be 0 (dense) or in [(M-1)*3, 256]";
        return LGR_ERR_INVALID_ARG;
    }
    a.rest_stride = raw_rest_stride(params, M);
    {
        ProfScope ps(ST_SPARSE_PACK, stream);
        LGR_CUDA_TRY(cudaMemsetAsync(dL_dmeans2D, 0, sizeof(float) * 3 * (size_t)P, stream));
        if (stats)
            sparse_flag_kernel<true><<<(P + 255) / 256, 256, 0, stream>>>(P, radii, geo.grad_acc, xb + L.bitmap, popc, xb + L.vis);
        else
            sparse_flag_kernel<false><<<(P + 255) / 256, 256, 0, stream>>>(P, radii, geo.grad_acc, xb + L.bitmap, popc, nullptr);
        LGR_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_tmp, cub_bytes, popc, xb + L.prefix, w32, stream));
        sparse_index_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, xb + L.bitmap, xb + L.prefix, idx, xb + L.hdr, v->campos, stats ? 1 : 0,
                                                                 stats ? stats->serial : 0u);
        if (world > 1)
            sparse_publish_kernel<<<LGR_SMS, 256, 0, stream>>>(push, self, L.rows, L.vis, stats ? L.total_stats - L.vis : 0);
        if (stats)
            preprocess_backward_sparse_kernel<true><<<(P + SPK_THREADS - 1) / SPK_THREADS, SPK_THREADS, 0, stream>>>(a, idx, xb + L.hdr, push, L.rows);
        else
            preprocess_backward_sparse_kernel<false><<<(P + SPK_THREADS - 1) / SPK_THREADS, SPK_THREADS, 0, stream>>>(a, idx, xb + L.hdr, push, L.rows);
    }
    LGR_LAUNCH_CHECK("preprocess_backward_sparse_kernel", debug, stream);
    return LGR_OK;
}

int lgr_backward_raw_sparse_accumulate(int P, int M, int sh_degree, int world, const void* const* peer_buffers, const float* xyz,
                                       const lgr_raw_grads* grads, void* cuda_stream)
{
    if (P == 0) return LGR_OK;
    if (P < 0 || M < 2 || M > 16 || sh_degree < 0 || sh_degree > 3 || (sh_degree + 1) * (sh_degree + 1) > M || world < 1 || world > 8 ||
        !peer_buffers || !xyz || !grads || !grads->xyz || !grads->features_dc || !grads->features_rest || !grads->scaling || !grads->rotation ||
        !grads->opacity || ((uintptr_t)grads->rotation & 15) || ((uintptr_t)grads->features_rest & 15) || ((uintptr_t)grads->features_dc & 15)) {
        g_last_error = "lgr_backward_raw_sparse_accumulate: bad argument (1..8 ranks, SH degree <= 3, 2 <= M <= 16, 16-byte aligned gradient rows)";
        return LGR_ERR_INVALID_ARG;
    }
    SparseAccArgs a;
    memset(&a, 0, sizeof(a));
    a.P = P; a.D = sh_degree; a.M = M; a.world = world;
    for (int r = 0; r < world; r++) {
        if (!peer_buffers[r] || ((uintptr_t)peer_buffers[r] & 255)) {
            g_last_error = "lgr_backward_raw_sparse_accumulate: peer buffer missing or not 256-byte aligned";
            return LGR_ERR_INVALID_ARG;
        }
        a.peer[r] = static_cast<const uint32_t*>(peer_buffers[r]);
    }
    a.xyz = xyz;
    a.d_xyz = grads->xyz; a.d_dc = grads->features_dc; a.d_rest = grads->features_rest; a.d_scaling = grads->scaling;
    a.d_rotation = grads->rotation; a.d_opacity = grads->opacity;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const size_t smem = raw_smem_bytes(M);
    LGR_CUDA_TRY(cudaFuncSetAttribute(sparse_accumulate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    {
        ProfScope ps(ST_SPARSE_ACC, stream);
        sparse_accumulate_kernel<<<(P + 255) / 256, 256, smem, stream>>>(a);
    }
    LGR_LAUNCH_CHECK("sparse_accumulate_kernel", false, stream);
    return LGR_OK;
}

int lgr_densify_stats_exchanged(int P, int world, int self, const void* const* peer_buffers, uint32_t serial, const float* grad,
                                int grad_row_stride, const uint8_t* update_filter, float* accum, float* denom, uint32_t* error_word,
                                void* cuda_stream)
{
    if (P < 0 || world < 1 || world > 8 || self < 0 || self >= world || grad_row_stride < 2 || !peer_buffers ||
        (P && (!grad || !update_filter || !accum || !denom || !error_word))) {
        g_last_error = "lgr_densify_stats_exchanged: bad argument (1..8 ranks, 0 <= self < world, grad_row_stride >= 2, all pointers set)";
        return LGR_ERR_INVALID_ARG;
    }
    if (P == 0) return LGR_OK;
    DensifyExchArgs a;
    memset(&a, 0, sizeof(a));
    a.P = P; a.world = world; a.self = self; a.serial = serial;
    for (int r = 0; r < world; r++) {
        if (!peer_buffers[r] || ((uintptr_t)peer_buffers[r] & 255)) {
            g_last_error = "lgr_densify_stats_exchanged: peer buffer missing or not 256-byte aligned";
            return LGR_ERR_INVALID_ARG;
        }
        a.slot[r] = static_cast<const uint32_t*>(peer_buffers[r]);
    }
    a.grad = grad; a.grad_stride = grad_row_stride; a.filter = update_filter; a.accum = accum; a.denom = denom; a.err = error_word;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    densify_stats_exchanged_kernel<<<(P + 255) / 256, 256, 0, stream>>>(a);
    LGR_LAUNCH_CHECK("densify_stats_exchanged_kernel", false, stream);
    return LGR_OK;
}

int lgr_peer_allreduce(float* const* peer_buffers, int rank, int world, size_t n_floats, void* cuda_stream)
{
    if (world < 1 || world > 8 || rank < 0 || rank >= world || !peer_buffers || (n_floats & 3)) {
        g_last_error = "lgr_peer_allreduce: need 1..8 ranks and a float count that is a multiple of 4";
        return LGR_ERR_INVALID_ARG;
    }
    if (world == 1 || n_floats == 0) return LGR_OK;
    PeerPtrs pp;
    for (int r = 0; r < 8; r++) pp.p[r] = r < world ? peer_buffers[r] : nullptr;
    for (int r = 0; r < world; r++)
        if (!pp.p[r] || ((uintptr_t)pp.p[r] & 15)) {
            g_last_error = "lgr_peer_allreduce: peer buffer missing or not 16-byte aligned";
            return LGR_ERR_INVALID_ARG;
        }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    {
        ProfScope ps(ST_PEER_ALLREDUCE, stream);
        peer_allreduce_kernel<<<LGR_SMS * 2, 512, 0, stream>>>(pp, rank, world, n_floats / 4);
    }
    LGR_LAUNCH_CHECK("peer_allreduce_kernel", false, stream);
    return LGR_OK;
}

int lgr_multimem_allreduce(float* multicast_ptr, int rank, int world, size_t n_floats, void* cuda_stream)
{
    if (world < 1 || rank < 0 || rank >= world || !multicast_ptr || (n_floats & 3) || ((uintptr_t)multicast_ptr & 15)) {
        g_last_error = "lgr_multimem_allreduce: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    if (world == 1 || n_floats == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    {
        ProfScope ps(ST_PEER_ALLREDUCE, stream);
        multimem_allreduce_kernel<<<LGR_SMS * 2, 512, 0, stream>>>(multicast_ptr, rank, world, n_floats / 4);
    }
    LGR_LAUNCH_CHECK("multimem_allreduce_kernel", false, stream);
    return LGR_OK;
}

int lgr_sh_grad_from_views(int P, int M, int sh_degree, int n_views, const float* xyz, const float* campos, const float* d_rgb,
                           float* d_features_dc, float* d_features_rest, void* cuda_stream)
{
    if (P == 0 || n_views == 0) return LGR_OK;
    if (P < 0 || M < 2 || M > 16 || sh_degree < 0 || sh_degree > 3 || (sh_degree + 1) * (sh_degree + 1) > M || !xyz || !campos || !d_rgb ||
        !d_features_dc || !d_features_rest || ((uintptr_t)d_features_rest & 15) || ((uintptr_t)d_features_dc & 15)) {
        g_last_error = "lgr_sh_grad_from_views: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    ShGradArgs a{P, sh_degree, M, n_views, xyz, campos, d_rgb, d_features_dc, d_features_rest};
    const size_t smem = raw_smem_bytes(M);
    LGR_CUDA_TRY(cudaFuncSetAttribute(sh_grad_from_views_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    {
        ProfScope ps(ST_SH_GRAD, stream);
        sh_grad_from_views_kernel<<<(P + 255) / 256, 256, smem, stream>>>(a);
    }
    LGR_LAUNCH_CHECK("sh_grad_from_views_kernel", false, stream);
    return LGR_OK;
}

// ---- fused image loss (row N2): utils/loss_utils.py l1_loss + ssim and their backward ----
static LossWindow make_loss_window()
{
    // gaussian(11, 1.5) of utils/loss_utils.py:26-33: float32 taps, normalised by their float32 sum
    LossWindow w;
    float sum = 0.f;
    for (int k = 0; k < 11; k++) {
        w.g[k] = (float)exp(-(double)((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5));
        sum += w.g[k];
    }
    for (int k = 0; k < 11; k++) w.g[k] = w.g[k] / sum;
    return w;
}

size_t lgr_image_loss_workspace_bytes(int C, int H, int W)
{
    const size_t blocks = (size_t)((W + LT - 1) / LT) * ((H + LT - 1) / LT) * (size_t)(C > 0 ? C : 0);
    return blocks * sizeof(float2) + 256;
}

int lgr_image_loss_forward(const float* img, const float* target, int C, int H, int W, float* out2, float* dmaps, void* workspace,
                           void* cuda_stream)
{
    if (!img || !target || !out2 || !workspace || C <= 0 || H <= 0 || W <= 0 || ((uintptr_t)workspace & 7)) {
        g_last_error = "lgr_image_loss_forward: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, C);
    const int nblocks = (int)(grid.x * grid.y * grid.z);
    {
        ProfScope ps(ST_LOSS_FWD, stream);
        image_loss_forward_kernel<<<grid, 256, 0, stream>>>(img, target, C, H, W, make_loss_window(), dmaps, (float2*)workspace);
        image_loss_finish_kernel<<<1, 256, 0, stream>>>((const float2*)workspace, nblocks, 1.0 / ((double)C * H * W), out2);
    }
    LGR_LAUNCH_CHECK("image_loss_forward_kernel", false, stream);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return LGR_OK;
}

int lgr_image_l1_forward(const float* img, const float* target, int C, int H, int W, float* out2, void* workspace, void* cuda_stream)
{
    if (!img || !target || !out2 || !workspace || C <= 0 || H <= 0 || W <= 0 || ((uintptr_t)workspace & 7) || (((uintptr_t)img | (uintptr_t)target) & 15)) {
        g_last_error = "lgr_image_l1_forward: bad argument (images must be 16-byte aligned)";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const long long n = (long long)C * H * W;
    // never more blocks than the workspace of lgr_image_loss_workspace_bytes(C,H,W) holds partials for
    const long long cap = (long long)((W + LT - 1) / LT) * ((H + LT - 1) / LT) * C;
    const int blocks = (int)std::max(1LL, std::min({cap, (n / 4 + 255) / 256, (long long)LGR_SMS * 8}));
    {
        ProfScope ps(ST_LOSS_FWD, stream);
        image_l1_forward_kernel<<<blocks, 256, 0, stream>>>(img, target, n, (float2*)workspace);
        image_loss_finish_kernel<<<1, 256, 0, stream>>>((const float2*)workspace, blocks, 1.0 / (double)n, out2);
    }
    LGR_LAUNCH_CHECK("image_l1_forward_kernel", false, stream);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return LGR_OK;
}

int lgr_image_loss_backward(const float* img, const float* target, const float* dmaps, int C, int H, int W, float g_l1, float g_ssim,
                            const float* grad_scale, float* d_img, void* cuda_stream)
{
    if (!img || !target || !d_img || C <= 0 || H <= 0 || W <= 0 || (g_ssim != 0.f && !dmaps)) {
        g_last_error = "lgr_image_loss_backward: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, C);
    {
        ProfScope ps(ST_LOSS_BWD, stream);
        image_loss_backward_kernel<<<grid, 256, 0, stream>>>(img, target, dmaps, C, H, W, make_loss_window(), g_l1, g_ssim, grad_scale,
                                                              (float)(1.0 / ((double)C * H * W)), d_img);
    }
    LGR_LAUNCH_CHECK("image_loss_backward_kernel", false, stream);
    return LGR_OK;
}

// ---- optimizer (row N3) ----
// the per-tensor host scalars of one AdamW step: torch/optim/adam.py _multi_tensor_adam forms them from python floats (double), then
// casts them to the kernels' opmath type (float)
static void adamw_scalars(double lr, double step, double beta1, double beta2, double weight_decay, float* decay, float* neg_step, float* bc2_sqrt)
{
    const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
    *decay = (float)(1.0 - lr * weight_decay);
    *neg_step = (float)((lr / bc1) * -1.0);
    *bc2_sqrt = (float)pow(bc2, 0.5);
}

int lgr_adamw_step(int n_tensors, const lgr_adamw_tensor* tensors, double beta1, double beta2, double eps, double weight_decay,
                   void* cuda_stream)
{
    if (n_tensors < 0 || n_tensors > OPT_MAX_TENSORS || (n_tensors && !tensors)) {
        g_last_error = "lgr_adamw_step: between 0 and 8 tensors per call";
        return LGR_ERR_INVALID_ARG;
    }
    AdamTable t;
    memset(&t, 0, sizeof(t));
    int k = 0;
    long long chunks = 0;
    for (int i = 0; i < n_tensors; i++) {
        const lgr_adamw_tensor& a = tensors[i];
        if (a.numel == 0) continue;
        if (a.numel < 0 || !a.param || !a.grad || !a.exp_avg || !a.exp_avg_sq || a.step < 1.0) {
            g_last_error = "lgr_adamw_step: tensor with a missing pointer, negative size or step < 1";
            return LGR_ERR_INVALID_ARG;
        }
        t.p[k] = a.param; t.g[k] = a.grad; t.m[k] = a.exp_avg; t.v[k] = a.exp_avg_sq;
        t.n[k] = a.numel;
        if (a.row_elems < 0 || a.row_elems > 0x7fffffffLL || (a.row_elems > 0 && (a.param_row_stride < a.row_elems || a.param_row_stride > 0x7fffffffLL ||
                                                                                 a.numel % a.row_elems != 0))) {
            g_last_error = "lgr_adamw_step: row-strided parameter needs row_elems dividing numel and param_row_stride >= row_elems";
            return LGR_ERR_INVALID_ARG;
        }
        t.row_elems[k] = (a.row_elems > 0 && a.param_row_stride != a.row_elems) ? (int)a.row_elems : 0;
        t.row_stride[k] = (int)a.param_row_stride;
        adamw_scalars(a.lr, a.step, beta1, beta2, weight_decay, &t.decay[k], &t.neg_step[k], &t.bc2_sqrt[k]);
        t.chunk_start[k] = (int)chunks;
        chunks += (a.numel + OPT_CHUNK - 1) / OPT_CHUNK;
        k++;
    }
    if (chunks > 0x7fffffffLL) {
        g_last_error = "lgr_adamw_step: too many elements for one launch";
        return LGR_ERR_INVALID_ARG;
    }
    for (int i = k; i <= OPT_MAX_TENSORS; i++) t.chunk_start[i] = (int)chunks;
    t.count = k;
    t.w1 = (float)(1.0 - beta1); t.beta2 = (float)beta2; t.w2 = (float)(1.0 - beta2); t.eps = (float)eps;
    if (chunks == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    {
        ProfScope ps(ST_ADAMW, stream);
        adamw_multi_kernel<<<(unsigned)chunks, 256, 0, stream>>>(t);
    }
    LGR_LAUNCH_CHECK("adamw_multi_kernel", false, stream);
    return LGR_OK;
}

// the [rows, width] view (row stride rs, column stride cs) reaches no element twice: rows lie side by side (cs*width <= rs) or
// columns do (rs*rows <= cs)
static bool row_view_ok(long long rows, long long width, long long rs, long long cs)
{
    if (rs < 0 || cs < 0 || rs > (1LL << 40) || cs > (1LL << 40)) return false;
    if (rows > 1 && width > 1) return (cs >= 1 && cs * width <= rs) || (rs >= 1 && rs * rows <= cs);
    if (rows > 1) return rs >= 1;
    if (width > 1) return cs >= 1;
    return true;
}

int lgr_adamw_step_selective(int n_tensors, const lgr_adamw_row_tensor* tensors, long long rows, double beta1, double beta2, double eps,
                             double weight_decay, void* cuda_stream)
{
    if (n_tensors < 0 || n_tensors > OPT_MAX_TENSORS || (n_tensors && !tensors) || rows < 0 || rows > (1LL << 37)) {
        g_last_error = "lgr_adamw_step_selective: between 0 and 8 tensors per call and 0 <= rows < 2^37";
        return LGR_ERR_INVALID_ARG;
    }
    SelAdamTable t;
    memset(&t, 0, sizeof(t));
    int k = 0, row_floats = 0;
    for (int i = 0; i < n_tensors; i++) {
        const lgr_adamw_row_tensor& a = tensors[i];
        if (a.width < 0 || a.width > SEL_MAX_ROW_FLOATS) {
            g_last_error = "lgr_adamw_step_selective: width must be between 0 and 400";
            return LGR_ERR_INVALID_ARG;
        }
        if (a.width == 0 || rows == 0) continue;
        if (!a.param || !a.grad || !a.exp_avg || !a.exp_avg_sq || a.step < 1.0) {
            g_last_error = "lgr_adamw_step_selective: tensor with a missing pointer or step < 1";
            return LGR_ERR_INVALID_ARG;
        }
        const long long rs[4] = {a.param_row_stride, a.grad_row_stride, a.exp_avg_row_stride, a.exp_avg_sq_row_stride};
        const long long cs[4] = {a.param_col_stride, a.grad_col_stride, a.exp_avg_col_stride, a.exp_avg_sq_col_stride};
        for (int j = 0; j < 4; j++) {
            if (!row_view_ok(rows, a.width, rs[j], cs[j])) {
                g_last_error = "lgr_adamw_step_selective: a [rows, width] view whose strides overlap its own elements or are negative";
                return LGR_ERR_INVALID_ARG;
            }
            t.rs[k][j] = rs[j];
            t.cs[k][j] = cs[j];
        }
        row_floats += (int)a.width;
        if (row_floats > SEL_MAX_ROW_FLOATS) {
            g_last_error = "lgr_adamw_step_selective: the widths add up to more than 400 floats per row";
            return LGR_ERR_INVALID_ARG;
        }
        t.p[k] = a.param; t.g[k] = a.grad; t.m[k] = a.exp_avg; t.v[k] = a.exp_avg_sq;
        t.width[k] = (int)a.width;
        t.smem_off[k] = (row_floats - (int)a.width) * SEL_ROWS;
        adamw_scalars(a.lr, a.step, beta1, beta2, weight_decay, &t.decay[k], &t.neg_step[k], &t.bc2_sqrt[k]);
        k++;
    }
    t.count = k;
    t.rows = rows;
    t.w1 = (float)(1.0 - beta1); t.beta2 = (float)beta2; t.w2 = (float)(1.0 - beta2); t.eps = (float)eps;
    if (k == 0) return LGR_OK;
    const size_t smem = (size_t)row_floats * SEL_ROWS * sizeof(float);
    // always: static + dynamic shared memory together may pass 48 KB even when the dynamic part alone does not
    LGR_CUDA_TRY(cudaFuncSetAttribute(adamw_selective_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(smem, (size_t)48 * 1024)));
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    {
        ProfScope ps(ST_ADAMW_SELECTIVE, stream);
        adamw_selective_kernel<<<(unsigned)((rows + SEL_ROWS - 1) / SEL_ROWS), SEL_THREADS, smem, stream>>>(t);
    }
    LGR_LAUNCH_CHECK("adamw_selective_kernel", false, stream);
    return LGR_OK;
}

static size_t compact_cub_bytes(int P)
{
    size_t bytes = 0;
    cub::DeviceSelect::Flagged((void*)nullptr, bytes, thrust::counting_iterator<int>(0), (const uint8_t*)nullptr, (int*)nullptr, (int*)nullptr, P);
    return bytes;
}

size_t lgr_compact_workspace_bytes(int P) { return P > 0 ? align_up(compact_cub_bytes(P), 256) + 256 : 256; }

int lgr_compact_plan(int P, const uint8_t* keep, int32_t* src_row, void* workspace, size_t workspace_bytes, int32_t* rows_out_host,
                     void* cuda_stream)
{
    if (!rows_out_host || P < 0) {
        g_last_error = "lgr_compact_plan: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    *rows_out_host = 0;
    if (P == 0) return LGR_OK;
    if (!keep || !src_row || !workspace || workspace_bytes < lgr_compact_workspace_bytes(P) || ((uintptr_t)workspace & 255)) {
        g_last_error = "lgr_compact_plan: missing pointer or workspace smaller than lgr_compact_workspace_bytes(P) / not 256-byte aligned";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    int* d_count = reinterpret_cast<int*>(workspace);
    size_t cub_bytes = workspace_bytes - 256;
    {
        ProfScope ps(ST_COMPACT, stream);
        LGR_CUDA_TRY(cub::DeviceSelect::Flagged(static_cast<char*>(workspace) + 256, cub_bytes, thrust::counting_iterator<int>(0), keep, src_row,
                                                d_count, P, stream));
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    LGR_CUDA_TRY(cudaMemcpyAsync(rows_out_host, d_count, sizeof(int), cudaMemcpyDeviceToHost, stream));
    LGR_CUDA_TRY(cudaStreamSynchronize(stream));
    return LGR_OK;
}

int lgr_compact_rows(int rows_out, const int32_t* src_row, int n_tensors, const lgr_compact_tensor* tensors, void* cuda_stream)
{
    if (rows_out < 0 || n_tensors < 0 || n_tensors > CMP_MAX_TENSORS || (n_tensors && !tensors) || (rows_out && !src_row)) {
        g_last_error = "lgr_compact_rows: bad argument (at most 24 tensors per call)";
        return LGR_ERR_INVALID_ARG;
    }
    if (rows_out == 0 || n_tensors == 0) return LGR_OK;
    CompactTable t;
    memset(&t, 0, sizeof(t));
    long long chunks = 0;
    int k = 0;
    for (int i = 0; i < n_tensors; i++) {
        if (tensors[i].row_words == 0) continue;
        if (tensors[i].row_words < 0 || !tensors[i].src || !tensors[i].dst) {
            g_last_error = "lgr_compact_rows: tensor with a missing pointer or negative row width";
            return LGR_ERR_INVALID_ARG;
        }
        t.src[k] = static_cast<const float*>(tensors[i].src);
        t.dst[k] = static_cast<float*>(tensors[i].dst);
        t.width[k] = tensors[i].row_words;
        t.chunk_start[k] = (int)chunks;
        chunks += ((long long)rows_out * tensors[i].row_words + CMP_CHUNK - 1) / CMP_CHUNK;
        k++;
    }
    if (chunks > 0x7fffffffLL) {
        g_last_error = "lgr_compact_rows: too many elements for one launch";
        return LGR_ERR_INVALID_ARG;
    }
    for (int i = k; i <= CMP_MAX_TENSORS; i++) t.chunk_start[i] = (int)chunks;
    t.count = k;
    t.rows_out = rows_out;
    if (chunks == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    {
        ProfScope ps(ST_COMPACT, stream);
        compact_gather_kernel<<<(unsigned)chunks, 256, 0, stream>>>(t, src_row);
    }
    LGR_LAUNCH_CHECK("compact_gather_kernel", false, stream);
    return LGR_OK;
}

// ---- VecTree vector quantisation (row N4) ----
// workspace: best[n] (64-bit score | code) followed by the deterministic mode's sort buffers (codes and sample rows, in and out) and the
// radix sort's temporary storage; the size does not depend on the mode, so a workspace stays valid when the mode changes
struct VqDetLayout { size_t codes_in, codes_out, rows_in, rows_out, temp, temp_bytes, total; };
VqDetLayout vq_det_layout(int64_t n)
{
    VqDetLayout L;
    const size_t m = (size_t)(n > 0 ? n : 0);
    L.codes_in = align_up(m * sizeof(unsigned long long), 256);
    L.codes_out = L.codes_in + align_up(m * 4, 256);
    L.rows_in = L.codes_out + align_up(m * 4, 256);
    L.rows_out = L.rows_in + align_up(m * 4, 256);
    L.temp = L.rows_out + align_up(m * 4, 256);
    L.temp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, L.temp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)(m ? m : 1), 0, 32);
    L.total = L.temp + align_up(L.temp_bytes, 256) + 256;
    return L;
}
size_t lgr_vq_workspace_bytes(int64_t n) { return vq_det_layout(n).total; }

int lgr_vq_assign(int n, int d, int K, const float* x, const float* embed, const float* weight, const float* weight_sum, int32_t* idx,
                  float* cluster_batch, float* embed_sum, void* workspace, void* cuda_stream)
{
    if (n < 0 || d <= 0 || d > 64 || K <= 0 || (n && (!x || !workspace)) || !embed || (weight && !weight_sum) || ((uintptr_t)workspace & 7)) {
        g_last_error = "lgr_vq_assign: bad argument (1 <= d <= 64, K >= 1, workspace of lgr_vq_workspace_bytes(n) bytes)";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    if (cluster_batch) LGR_CUDA_TRY(cudaMemsetAsync(cluster_batch, 0, sizeof(float) * K, stream));
    if (embed_sum) LGR_CUDA_TRY(cudaMemsetAsync(embed_sum, 0, sizeof(float) * (size_t)K * d, stream));
    if (n == 0) return LGR_OK;
    unsigned long long* best = static_cast<unsigned long long*>(workspace);
    if (g_vq_mode == 0 && d <= VT_DP && (long long)n * K >= (1ll << 20)) {
        // coarse pass on the tensor cores (wgmma, lgr_vq_tc.cuh) + exact FP32 rescore of the undecided rows
        const int n_pad = (n + VT_M - 1) / VT_M * VT_M, K_pad = (K + VT_N - 1) / VT_N * VT_N;
        const size_t oA = 0, oB = oA + vt_align((size_t)(n_pad / VT_M) * VT_A_BYTES), oN = oB + vt_align((size_t)(K_pad / VT_N) * VT_B_BYTES),
                     oX = oN + vt_align((size_t)K_pad * 4), oC = oX + vt_align((size_t)n_pad * 4), oL = oC + 1024, total = oL + vt_align((size_t)n * 4);
        int dev = 0;
        LGR_CUDA_TRY(cudaGetDevice(&dev));
        static VtScratch scratch[16];
        static std::mutex scratch_mutex;
        char* sp = nullptr;
        {
            std::lock_guard<std::mutex> l(scratch_mutex);
            VtScratch& sc = scratch[dev & 15];
            if (sc.bytes < total) {   // grow-only; cudaMalloc synchronises, but only when a larger problem shows up
                if (sc.p) LGR_CUDA_TRY(cudaFree(sc.p));
                sc.p = nullptr; sc.bytes = 0;
                LGR_CUDA_TRY(cudaMalloc(&sc.p, total + total / 4));
                sc.bytes = total + total / 4;
            }
            sp = static_cast<char*>(sc.p);
        }
        unsigned char* tA = reinterpret_cast<unsigned char*>(sp + oA);
        unsigned char* tB = reinterpret_cast<unsigned char*>(sp + oB);
        float* norms = reinterpret_cast<float*>(sp + oN);
        float* xnorm = reinterpret_cast<float*>(sp + oX);
        unsigned* emax = reinterpret_cast<unsigned*>(sp + oC);
        int* n_und = reinterpret_cast<int*>(sp + oC + 4);
        int* und = reinterpret_cast<int*>(sp + oL);
        {
            ProfScope ps(ST_VQ_ASSIGN, stream);
            LGR_CUDA_TRY(cudaMemsetAsync(sp + oC, 0, 8, stream));
            vt_prep_x_kernel<<<(n_pad + 255) / 256, 256, 0, stream>>>(n, n_pad, d, x, tA, xnorm);
            vt_prep_e_kernel<<<(K_pad + 255) / 256, 256, 0, stream>>>(K, K_pad, d, embed, tB, norms, emax);
            LGR_CUDA_TRY(cudaFuncSetAttribute(vt_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(VtSmem)));
            vt_assign_kernel<<<n_pad / VT_M, VT_THREADS, sizeof(VtSmem), stream>>>(n, K_pad, tA, tB, norms, xnorm, emax, best, und, n_und);
            constexpr int RXR = 4;
            const int row_tiles = (n + RXR * VQ_THREADS - 1) / (RXR * VQ_THREADS);
            const int code_tiles = (K + VQ_TC - 1) / VQ_TC;
            int splits = std::max(1, std::min(code_tiles, 64));
            const int codes_per_split = (code_tiles + splits - 1) / splits * VQ_TC;
            splits = (K + codes_per_split - 1) / codes_per_split;
            vq_assign_rows_kernel<VT_DP, RXR><<<dim3(row_tiles, splits), VQ_THREADS, 0, stream>>>(und, n_und, d, K, x, embed, codes_per_split, best);
            g_launches.fetch_add(3, std::memory_order_relaxed);
        }
        LGR_LAUNCH_CHECK("vt_assign_kernel", false, stream);
    } else {
        ProfScope ps(ST_VQ_ASSIGN, stream);
        vq_init_best_kernel<<<(n + 255) / 256, 256, 0, stream>>>(n, best);
        if (d <= 8) vq_launch_assign<8>(n, d, K, x, embed, best, stream);
        else if (d <= 16) vq_launch_assign<16>(n, d, K, x, embed, best, stream);
        else if (d <= 28) vq_launch_assign<28>(n, d, K, x, embed, best, stream);
        else if (d <= 32) vq_launch_assign<32>(n, d, K, x, embed, best, stream);
        else if (d <= 48) vq_launch_assign<48>(n, d, K, x, embed, best, stream);
        else vq_launch_assign<64>(n, d, K, x, embed, best, stream);
        LGR_LAUNCH_CHECK("vq_assign_kernel", false, stream);
    }
    if (g_det) {
        // deterministic mode: stable sort of (code, sample) pairs on log2(K) bits, then per-code sums in ascending sample order
        const VqDetLayout L = vq_det_layout(n);
        char* ws = static_cast<char*>(workspace);
        uint32_t* codes_in = reinterpret_cast<uint32_t*>(ws + L.codes_in);
        uint32_t* codes_out = reinterpret_cast<uint32_t*>(ws + L.codes_out);
        uint32_t* rows_in = reinterpret_cast<uint32_t*>(ws + L.rows_in);
        uint32_t* rows_out = reinterpret_cast<uint32_t*>(ws + L.rows_out);
        int bits = 1;
        while ((1ll << bits) < (long long)K) bits++;
        ProfScope ps(ST_VQ_ASSIGN, stream);
        vq_det_keys_kernel<<<(n + 255) / 256, 256, 0, stream>>>(n, best, idx, codes_in, rows_in);
        LGR_LAUNCH_CHECK("vq_det_keys_kernel", false, stream);
        if (cluster_batch || embed_sum) {
            size_t tmp = L.temp_bytes;
            LGR_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.temp, tmp, codes_in, codes_out, rows_in, rows_out, n, 0, bits, stream));
            vq_det_segsum_kernel<<<(unsigned)K, VQ_SEG_WARPS * 32, 0, stream>>>(n, d, K, codes_out, rows_out, x, weight, (float)n, weight_sum,
                                                                                         cluster_batch, embed_sum);
            LGR_LAUNCH_CHECK("vq_det_segsum_kernel", false, stream);
        }
        return LGR_OK;
    }
    const long long total = (long long)n * (d + 1);
    vq_accumulate_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(n, d, best, x, weight, (float)n, weight_sum, idx, cluster_batch,
                                                                                 embed_sum);
    LGR_LAUNCH_CHECK("vq_accumulate_kernel", false, stream);
    return LGR_OK;
}

int lgr_vq_ema_update(int K, int d, double decay, double eps, float* cluster_size, float* embed, const float* cluster_batch,
                      const float* embed_sum, float* scratch, void* cuda_stream)
{
    if (K <= 0 || d <= 0 || !cluster_size || !embed || !cluster_batch || !embed_sum || !scratch) {
        g_last_error = "lgr_vq_ema_update: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    {
        ProfScope ps(ST_VQ_UPDATE, stream);
        vq_ema_cluster_kernel<<<1, 1024, 0, stream>>>(K, (float)decay, (float)(1.0 - decay), cluster_size, cluster_batch, scratch);
        vq_ema_embed_kernel<<<(K * d + 255) / 256, 256, 0, stream>>>(K, d, (float)decay, (float)(1.0 - decay), (float)eps, (float)((double)K * eps),
                                                                      cluster_size, scratch, embed_sum, embed);
    }
    LGR_LAUNCH_CHECK("vq_ema_embed_kernel", false, stream);
    return LGR_OK;
}

int lgr_vq_gather(int n, int d, const int32_t* idx, const float* embed, float* out, void* cuda_stream)
{
    if (n < 0 || d <= 0 || (n && (!idx || !embed || !out))) {
        g_last_error = "lgr_vq_gather: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    if (n == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const long long total = (long long)n * d;
    vq_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(n, d, idx, embed, out);
    LGR_LAUNCH_CHECK("vq_gather_kernel", false, stream);
    return LGR_OK;
}

int lgr_vq_pack_indices(int64_t n, int bits, const int32_t* idx, uint8_t* out, void* cuda_stream)
{
    if (n < 0 || bits < 1 || bits > 31 || (n && (!idx || !out))) {
        g_last_error = "lgr_vq_pack_indices: bad argument (1 <= bits <= 31)";
        return LGR_ERR_INVALID_ARG;
    }
    if (n == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    const long long n_bytes = ((long long)n * bits + 7) / 8;
    vq_pack_kernel<<<(unsigned)((n_bytes + 255) / 256), 256, 0, stream>>>(n, bits, idx, out, n_bytes);
    LGR_LAUNCH_CHECK("vq_pack_kernel", false, stream);
    return LGR_OK;
}

int lgr_vq_unpack_indices(int64_t n, int bits, const uint8_t* in, int32_t* idx, void* cuda_stream)
{
    if (n < 0 || bits < 1 || bits > 31 || (n && (!idx || !in))) {
        g_last_error = "lgr_vq_unpack_indices: bad argument (1 <= bits <= 31)";
        return LGR_ERR_INVALID_ARG;
    }
    if (n == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    vq_unpack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(n, bits, in, idx);
    LGR_LAUNCH_CHECK("vq_unpack_kernel", false, stream);
    return LGR_OK;
}

int lgr_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present, void* cuda_stream)
{
    (void)projmatrix;
    if (P == 0) return LGR_OK;
    if (P < 0 || !means3D || !viewmatrix || !present) {
        g_last_error = "lgr_mark_visible: missing required argument";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, present);
    LGR_LAUNCH_CHECK("mark_visible_kernel", false, stream);
    return LGR_OK;
}

size_t lgr_knn_workspace_bytes(int P) { return knn_layout(P).total; }

int lgr_knn_mean_dist3(int P, const float* points, float* out, void* workspace, size_t workspace_bytes, void* cuda_stream)
{
    if (P < 0) {
        g_last_error = "lgr_knn_mean_dist3: P < 0";
        return LGR_ERR_INVALID_ARG;
    }
    if (P == 0) return LGR_OK;
    const KnnLayout L = knn_layout(P);
    if (!points || !out || !workspace || workspace_bytes < L.total || ((uintptr_t)workspace & 255) || ((uintptr_t)points & 3)) {
        g_last_error = "lgr_knn_mean_dist3: missing pointer, or workspace smaller than lgr_knn_workspace_bytes(P) / not 256-byte aligned";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    char* ws = static_cast<char*>(workspace);
    unsigned* bbox = reinterpret_cast<unsigned*>(ws + L.bbox);
    uint32_t* codes = reinterpret_cast<uint32_t*>(ws + L.codes);
    uint32_t* codes_sorted = reinterpret_cast<uint32_t*>(ws + L.codes_sorted);
    uint32_t* ids = reinterpret_cast<uint32_t*>(ws + L.ids);
    uint32_t* ids_sorted = reinterpret_cast<uint32_t*>(ws + L.ids_sorted);
    float4* sorted = reinterpret_cast<float4*>(ws + L.sorted);
    float4* leafbox = reinterpret_cast<float4*>(ws + L.leafbox);
    float4* nodebox = reinterpret_cast<float4*>(ws + L.nodebox);
    const int nleaf = (P + KNN_LEAF - 1) / KNN_LEAF, nnode = (nleaf + KNN_NODE - 1) / KNN_NODE;

    LGR_CUDA_TRY(cudaMemsetAsync(bbox, 0xff, 3 * sizeof(unsigned), stream));
    LGR_CUDA_TRY(cudaMemsetAsync(bbox + 3, 0, 3 * sizeof(unsigned), stream));
    knn_bbox_kernel<<<std::min((P + 255) / 256, 4 * LGR_SMS), 256, 0, stream>>>(P, points, bbox);
    LGR_LAUNCH_CHECK("knn_bbox_kernel", false, stream);
    knn_morton_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, points, bbox, codes, ids);
    LGR_LAUNCH_CHECK("knn_morton_kernel", false, stream);
    size_t cub_bytes = L.cub_bytes;
    LGR_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, codes, codes_sorted, ids, ids_sorted, P, 0, 30, stream));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    knn_leaf_kernel<<<(nleaf + 7) / 8, 256, 0, stream>>>(P, nleaf, points, ids_sorted, sorted, leafbox);
    LGR_LAUNCH_CHECK("knn_leaf_kernel", false, stream);
    knn_node_kernel<<<(nnode + 7) / 8, 256, 0, stream>>>(nleaf, nnode, leafbox, nodebox);
    LGR_LAUNCH_CHECK("knn_node_kernel", false, stream);
    constexpr int warps = KNN_SEARCH_THREADS / 32;
    knn_search_kernel<<<(nleaf + warps - 1) / warps, KNN_SEARCH_THREADS, 0, stream>>>(P, nleaf, nnode, sorted, leafbox, nodebox, out);
    LGR_LAUNCH_CHECK("knn_search_kernel", false, stream);
    return LGR_OK;
}

}  // extern "C"

// ---- densification (csrc/lgr_densify.cuh) ----
namespace {
struct DensifyLayout {
    size_t cls, scan, counts, cub, cub_bytes, total;
};
DensifyLayout densify_layout(int P)
{
    DensifyLayout L{};
    const int n = P > 0 ? P : 1;
    L.cls = 0;
    L.scan = align_up((size_t)n, 256);
    L.counts = align_up(L.scan + sizeof(int4) * (size_t)n, 256);
    L.cub = L.counts + 256;
    cub::DeviceScan::InclusiveScan((void*)nullptr, L.cub_bytes, thrust::make_transform_iterator((const uint8_t*)nullptr, DenClassCounts()),
                                   (int4*)nullptr, DenInt4Sum(), n);
    L.total = align_up(L.cub + L.cub_bytes, 256);
    return L;
}
}  // namespace

extern "C" {

int lgr_densify_stats(int P, const float* grad, int grad_row_stride, const uint8_t* update_filter, float* accum, float* denom,
                      void* cuda_stream)
{
    if (P < 0 || grad_row_stride < 2 || (P && (!grad || !update_filter || !accum || !denom))) {
        g_last_error = "lgr_densify_stats: bad argument (P >= 0, grad_row_stride >= 2, all pointers set)";
        return LGR_ERR_INVALID_ARG;
    }
    if (P == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    densify_stats_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, grad, grad_row_stride, update_filter, accum, denom);
    LGR_LAUNCH_CHECK("densify_stats_kernel", false, stream);
    return LGR_OK;
}

int lgr_densify_stats_encode(int P, const float* grad, int grad_row_stride, const uint8_t* update_filter, float* out, void* cuda_stream)
{
    if (P < 0 || grad_row_stride < 2 || (P && (!grad || !update_filter || !out))) {
        g_last_error = "lgr_densify_stats_encode: bad argument (P >= 0, grad_row_stride >= 2, all pointers set)";
        return LGR_ERR_INVALID_ARG;
    }
    if (P == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    densify_stats_encode_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, grad, grad_row_stride, update_filter, out);
    LGR_LAUNCH_CHECK("densify_stats_encode_kernel", false, stream);
    return LGR_OK;
}

int lgr_densify_stats_add_views(int P, int world, const float* views, float* accum, float* denom, void* cuda_stream)
{
    if (P < 0 || world < 1 || (P && (!views || !accum || !denom))) {
        g_last_error = "lgr_densify_stats_add_views: bad argument (P >= 0, world >= 1, all pointers set)";
        return LGR_ERR_INVALID_ARG;
    }
    if (P == 0) return LGR_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    densify_stats_views_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, world, views, accum, denom);
    LGR_LAUNCH_CHECK("densify_stats_views_kernel", false, stream);
    return LGR_OK;
}

size_t lgr_densify_workspace_bytes(int P) { return densify_layout(P).total; }

int lgr_densify_plan(int P, const float* accum, const float* denom, const float* scaling, const float* opacity, float max_grad,
                     float dense_scale, float min_opacity, float big_scale, int prune_all, int prune_big, void* workspace,
                     size_t workspace_bytes, int32_t* counts_host, void* cuda_stream)
{
    if (P < 0 || !counts_host) {
        g_last_error = "lgr_densify_plan: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    for (int k = 0; k < 4; k++) counts_host[k] = 0;
    if (P == 0) return LGR_OK;
    const DensifyLayout L = densify_layout(P);
    if (!accum || !denom || !scaling || !opacity || !workspace || workspace_bytes < L.total || ((uintptr_t)workspace & 255)) {
        g_last_error = "lgr_densify_plan: missing pointer, or workspace smaller than lgr_densify_workspace_bytes(P) / not 256-byte aligned";
        return LGR_ERR_INVALID_ARG;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    char* ws = static_cast<char*>(workspace);
    uint8_t* cls = reinterpret_cast<uint8_t*>(ws + L.cls);
    int4* scan = reinterpret_cast<int4*>(ws + L.scan);
    const DensifyPlanArgs a{accum, denom, scaling, opacity, max_grad, dense_scale, min_opacity, big_scale, prune_all ? 1 : 0, prune_big ? 1 : 0};
    densify_plan_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, a, cls);
    LGR_LAUNCH_CHECK("densify_plan_kernel", false, stream);
    size_t cub_bytes = L.cub_bytes;
    LGR_CUDA_TRY(cub::DeviceScan::InclusiveScan(ws + L.cub, cub_bytes, thrust::make_transform_iterator((const uint8_t*)cls, DenClassCounts()),
                                                scan, DenInt4Sum(), P, stream));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    LGR_CUDA_TRY(cudaMemcpyAsync(counts_host, scan + (P - 1), sizeof(int4), cudaMemcpyDeviceToHost, stream));
    LGR_CUDA_TRY(cudaStreamSynchronize(stream));
    return LGR_OK;
}

int lgr_densify_split_inputs(int P, const void* workspace, const int32_t* counts, const float* scaling, const float* rotation,
                             const float* normals, float* rotations_out, float* samples_out, void* cuda_stream)
{
    if (P < 0 || !counts) {
        g_last_error = "lgr_densify_split_inputs: bad argument";
        return LGR_ERR_INVALID_ARG;
    }
    if (P == 0 || counts[3] == 0) return LGR_OK;
    if (!workspace || ((uintptr_t)workspace & 255) || !scaling || !rotation || ((uintptr_t)rotation & 15) || !normals || !rotations_out ||
        !samples_out) {
        g_last_error = "lgr_densify_split_inputs: missing pointer, or a workspace / rotation pointer that is not aligned";
        return LGR_ERR_INVALID_ARG;
    }
    const char* ws = static_cast<const char*>(workspace);
    const DensifyLayout L = densify_layout(P);
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    densify_split_inputs_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, reinterpret_cast<const uint8_t*>(ws + L.cls),
                                                                     reinterpret_cast<const int4*>(ws + L.scan), scaling, rotation, normals,
                                                                     counts[3], rotations_out, samples_out);
    LGR_LAUNCH_CHECK("densify_split_inputs_kernel", false, stream);
    return LGR_OK;
}

int lgr_densify_rows(int P, const void* workspace, const int32_t* counts, const float* xyz, const float* child_offsets, int n_tensors,
                     const lgr_densify_tensor* tensors, void* cuda_stream)
{
    if (P < 0 || !counts || n_tensors < 0 || n_tensors > DEN_MAX_TENSORS || (n_tensors && !tensors)) {
        g_last_error = "lgr_densify_rows: bad argument (at most 24 tensors per call)";
        return LGR_ERR_INVALID_ARG;
    }
    const long long rows_out = (long long)counts[0] + counts[1] + 2LL * counts[2];
    if (P == 0 || rows_out == 0 || n_tensors == 0) return LGR_OK;
    if (!workspace || ((uintptr_t)workspace & 255) || !xyz || (counts[2] && !child_offsets)) {
        g_last_error = "lgr_densify_rows: missing pointer, or a workspace that is not 256-byte aligned";
        return LGR_ERR_INVALID_ARG;
    }
    DensifyTable t;
    memset(&t, 0, sizeof(t));
    for (int i = 0; i < n_tensors; i++) {
        const lgr_densify_tensor& d = tensors[i];
        const bool geometric = d.role == LGR_DENSIFY_XYZ || d.role == LGR_DENSIFY_SCALING;
        if (d.role < LGR_DENSIFY_COPY || d.role > LGR_DENSIFY_ZERO || d.row_words < 0 || (geometric && d.row_words != 3)) {
            g_last_error = "lgr_densify_rows: tensor with a bad role or a bad row width";
            return LGR_ERR_INVALID_ARG;
        }
        if (d.row_words == 0) continue;   // an empty row, such as _features_rest [P,0,3] at SH degree 0: nothing to write
        if (!d.dst || (!d.src && d.role != LGR_DENSIFY_ZERO)) {
            g_last_error = "lgr_densify_rows: tensor with a missing pointer";
            return LGR_ERR_INVALID_ARG;
        }
        t.src[t.count] = static_cast<const float*>(d.src);
        t.dst[t.count] = static_cast<float*>(d.dst);
        t.width[t.count] = d.row_words;
        t.role[t.count] = d.role;
        t.count++;
    }
    const char* ws = static_cast<const char*>(workspace);
    const DensifyLayout L = densify_layout(P);
    const DensifyRowsArgs a{reinterpret_cast<const uint8_t*>(ws + L.cls), reinterpret_cast<const int4*>(ws + L.scan), xyz, child_offsets,
                            counts[0], counts[1], counts[2], counts[3]};
    cudaStream_t stream = static_cast<cudaStream_t>(cuda_stream);
    densify_rows_kernel<<<(unsigned)((P + 7) / 8), 256, 0, stream>>>(P, t, a);
    LGR_LAUNCH_CHECK("densify_rows_kernel", false, stream);
    return LGR_OK;
}

}  // extern "C"
