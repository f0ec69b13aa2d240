// lgr_knn.cuh -- distCUDA2 of submodules/simple-knn (spatial.cu:15-26, simple_knn.cu:147-221): for every point the mean of the
// squared distances to its three nearest other points, the initial Gaussian scales of GaussianModel.create_from_pcd
// (scene/gaussian_model.py:152-156).
//
// Result, bit for bit the reference's:
//   * the pair value is d = candidate - query per axis and dy*dy, then + dx*dx, then + dz*dz with two fused multiply-adds.  That is
//     what ptxas makes of `d.x*d.x + d.y*d.y + d.z*d.z` in updateKBest (simple_knn.cu:134-135): the SASS of boxMeanDist built for
//     sm_90a by nvcc 12.9 has, per pair, FADD dy / FADD dx / FMUL dy*dy / FADD dz / FFMA dx,dx,+ / FFMA dz,dz,+ (its box distance,
//     distBoxPoint at :119-129, is contracted in the same order).  knn_pair pins that order with _rn intrinsics.
//   * b0 <= b1 <= b2 are the three smallest pair values over all j != i, excluded by index (a duplicate point counts, at 0).  A slot
//     that no neighbour fills keeps the reference's FLT_MAX (:154), and a pair value is inserted only when strictly smaller (:138),
//     so an overflowing pair (+inf) never enters.  out = ((b0 + b1) + b2) / 3.0f with IEEE division (:182).
//   * Why any exact search returns the reference's bits: its box-pruned search is exact in its own arithmetic (a box's per-axis gap
//     never exceeds that of a point inside it, rounding is monotone, the skip test is a strict `>`), so the three smallest pair values
//     are one well-defined multiset.  This search prunes with the same argument and the same pinned arithmetic.
//
// Algorithm (all on one stream, no host synchronisation, every buffer in the caller's workspace):
//   knn_bbox_kernel     bounding box by atomicMin / atomicMax on order-preserving integer encodings of the coordinates
//   knn_morton_kernel   30-bit Morton codes in that box (they only order the points: the quantisation affects speed, never the result)
//   cub radix sort      (code, id) pairs
//   knn_leaf_kernel     points gathered into sorted order as float4 (w = id), AABB of every leaf of 32 consecutive sorted points
//   knn_node_kernel     AABB of every node of 32 leaves
//   knn_search_kernel   one warp per leaf, lane = query.  Seed each lane's three best from its own leaf, then sweep the nodes starting at
//                       its own.  Nodes and then their leaves are tested lane-parallel (lane j tests box j) with the box-to-box gap between
//                       the box and the warp's own leaf box against the largest third-best in the warp; a surviving leaf is tested once more
//                       per lane with its point-to-box gap against that lane's own third-best, and is scanned when any lane needs it:
//                       its 32 points loaded coalesced and broadcast by shuffle.  Both gaps are lower bounds of every pair value inside
//                       the box in the pinned arithmetic, and a box is skipped only when they are strictly larger, so no candidate that
//                       could enter a top three is skipped.  Every leaf is scanned at most once per warp; visit order does not matter.
namespace {

constexpr int KNN_LEAF = 32;           // points per leaf (one per lane)
constexpr int KNN_NODE = 32;           // leaves per node
constexpr int KNN_SEARCH_THREADS = 128;

// The pair value of updateKBest as compiled for sm_90a: FMUL dy*dy, FFMA dx*dx + that, FFMA dz*dz + that.
__device__ __forceinline__ float knn_pair(float dx, float dy, float dz)
{
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}

// Per-axis gap from q to [lo, hi]: 0 inside, else the rounded distance to the nearer face.  For any c in [lo, hi], |fl(c - q)| >= gap.
__device__ __forceinline__ float knn_gap(float q, float lo, float hi)
{
    return fmaxf(fmaxf(__fsub_rn(lo, q), __fsub_rn(q, hi)), 0.0f);
}

__device__ __forceinline__ float knn_point_box(const float4& q, const float4& lo, const float4& hi)
{
    return knn_pair(knn_gap(q.x, lo.x, hi.x), knn_gap(q.y, lo.y, hi.y), knn_gap(q.z, lo.z, hi.z));
}

// Per-axis gap between two boxes; for any q in [qlo, qhi] and c in [lo, hi], |fl(c - q)| >= gap.
__device__ __forceinline__ float knn_gap2(float lo, float hi, float qlo, float qhi)
{
    return fmaxf(fmaxf(__fsub_rn(lo, qhi), __fsub_rn(qlo, hi)), 0.0f);
}

__device__ __forceinline__ float knn_box_box(const float4& lo, const float4& hi, const float4& qlo, const float4& qhi)
{
    return knn_pair(knn_gap2(lo.x, hi.x, qlo.x, qhi.x), knn_gap2(lo.y, hi.y, qlo.y, qhi.y), knn_gap2(lo.z, hi.z, qlo.z, qhi.z));
}

// order-preserving map of a float to an unsigned integer (for atomicMin / atomicMax)
__device__ __forceinline__ unsigned knn_float_key(float f)
{
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float knn_key_float(unsigned u)
{
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// bbox[0..2] = keys of the minimum, bbox[3..5] = keys of the maximum; the caller presets them to 0xffffffff and 0
__global__ void knn_bbox_kernel(int P, const float* __restrict__ pts, unsigned* __restrict__ bbox)
{
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        for (int a = 0; a < 3; a++) {
            const float v = pts[3 * i + a];
            lo[a] = fminf(lo[a], v);
            hi[a] = fmaxf(hi[a], v);
        }
    }
    for (int a = 0; a < 3; a++) {
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(FULL, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(FULL, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0 && lo[0] <= hi[0]) {
        for (int a = 0; a < 3; a++) {
            atomicMin(bbox + a, knn_float_key(lo[a]));
            atomicMax(bbox + 3 + a, knn_float_key(hi[a]));
        }
    }
}

__device__ __forceinline__ uint32_t knn_spread10(uint32_t x)
{
    x = (x | (x << 16)) & 0x030000FFu;
    x = (x | (x << 8)) & 0x0300F00Fu;
    x = (x | (x << 4)) & 0x030C30C3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}

__global__ void knn_morton_kernel(int P, const float* __restrict__ pts, const unsigned* __restrict__ bbox, uint32_t* __restrict__ codes,
                                  uint32_t* __restrict__ ids)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    uint32_t code = 0;
    for (int a = 0; a < 3; a++) {
        const float lo = knn_key_float(bbox[a]), ext = knn_key_float(bbox[3 + a]) - lo;
        const float s = ext > 0.0f ? 1023.0f / ext : 0.0f;
        const float v = fminf(fmaxf((pts[3 * i + a] - lo) * s, 0.0f), 1023.0f);   // NaN -> 0
        code |= knn_spread10((uint32_t)v) << a;
    }
    codes[i] = code;
    ids[i] = (uint32_t)i;
}

// one warp per leaf: gather the leaf's points in sorted order (w = original index) and reduce its AABB
__global__ void knn_leaf_kernel(int P, int nleaf, const float* __restrict__ pts, const uint32_t* __restrict__ ids_sorted,
                                float4* __restrict__ sorted, float4* __restrict__ leafbox)
{
    const int leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (leaf >= nleaf) return;
    const int i = leaf * KNN_LEAF + lane;
    float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.0f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.0f);
    if (i < P) {
        const uint32_t id = ids_sorted[i];
        const float4 p = make_float4(pts[3 * id], pts[3 * id + 1], pts[3 * id + 2], __uint_as_float(id));
        sorted[i] = p;
        lo = make_float4(p.x, p.y, p.z, 0.0f);
        hi = lo;
    }
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(FULL, lo.x, o)); hi.x = fmaxf(hi.x, __shfl_xor_sync(FULL, hi.x, o));
        lo.y = fminf(lo.y, __shfl_xor_sync(FULL, lo.y, o)); hi.y = fmaxf(hi.y, __shfl_xor_sync(FULL, hi.y, o));
        lo.z = fminf(lo.z, __shfl_xor_sync(FULL, lo.z, o)); hi.z = fmaxf(hi.z, __shfl_xor_sync(FULL, hi.z, o));
    }
    if (lane == 0) {
        leafbox[2 * leaf] = lo;
        leafbox[2 * leaf + 1] = hi;
    }
}

// one warp per node: AABB of its (up to) 32 leaves
__global__ void knn_node_kernel(int nleaf, int nnode, const float4* __restrict__ leafbox, float4* __restrict__ nodebox)
{
    const int node = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (node >= nnode) return;
    const int leaf = node * KNN_NODE + lane;
    float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.0f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.0f);
    if (leaf < nleaf) {
        lo = leafbox[2 * leaf];
        hi = leafbox[2 * leaf + 1];
    }
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(FULL, lo.x, o)); hi.x = fmaxf(hi.x, __shfl_xor_sync(FULL, hi.x, o));
        lo.y = fminf(lo.y, __shfl_xor_sync(FULL, lo.y, o)); hi.y = fmaxf(hi.y, __shfl_xor_sync(FULL, hi.y, o));
        lo.z = fminf(lo.z, __shfl_xor_sync(FULL, lo.z, o)); hi.z = fmaxf(hi.z, __shfl_xor_sync(FULL, hi.z, o));
    }
    if (lane == 0) {
        nodebox[2 * node] = lo;
        nodebox[2 * node + 1] = hi;
    }
}

__device__ __forceinline__ float knn_warp_max(float v)
{
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, o));
    return v;
}

// every lane's query against the (up to) 32 points of leaf L, broadcast by shuffle; self excluded by original index
__device__ __forceinline__ void knn_scan_leaf(int P, const float4* __restrict__ sorted, int L, int lane, const float4& q, int qid,
                                              float& b0, float& b1, float& b2)
{
    const int base = L * KNN_LEAF, cnt = min(KNN_LEAF, P - base);
    const float4 c = lane < cnt ? sorted[base + lane] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    for (int k = 0; k < cnt; k++) {
        const float cx = __shfl_sync(FULL, c.x, k), cy = __shfl_sync(FULL, c.y, k), cz = __shfl_sync(FULL, c.z, k);
        const int cid = __float_as_int(__shfl_sync(FULL, c.w, k));
        const float d = knn_pair(__fsub_rn(cx, q.x), __fsub_rn(cy, q.y), __fsub_rn(cz, q.z));
        if (cid != qid && d < b2) {   // updateKBest<3> (simple_knn.cu:136-144): strict, so equal values leave the multiset unchanged
            if (d < b1) {
                b2 = b1;
                if (d < b0) { b1 = b0; b0 = d; } else { b1 = d; }
            } else {
                b2 = d;
            }
        }
    }
}

__global__ void __launch_bounds__(KNN_SEARCH_THREADS) knn_search_kernel(int P, int nleaf, int nnode, const float4* __restrict__ sorted,
                                                                       const float4* __restrict__ leafbox, const float4* __restrict__ nodebox,
                                                                       float* __restrict__ out)
{
    const int leaf = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (leaf >= nleaf) return;   // warp-uniform
    const int i = leaf * KNN_LEAF + lane;
    const bool valid = i < P;
    const float4 q = valid ? sorted[i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    const int qid = valid ? __float_as_int(q.w) : -1;
    float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;   // simple_knn.cu:154
    knn_scan_leaf(P, sorted, leaf, lane, q, qid, b0, b1, b2);

    const float4 qlo = leafbox[2 * leaf], qhi = leafbox[2 * leaf + 1];
    const int own_node = leaf / KNN_NODE;
    for (int c = 0; c < nnode; c += 32) {
        int n = own_node + c + lane;
        if (n >= nnode) n -= nnode;
        const float bound = knn_warp_max(valid ? b2 : -INFINITY);
        const bool visit = c + lane < nnode && !(knn_box_box(nodebox[2 * n], nodebox[2 * n + 1], qlo, qhi) > bound);
        for (unsigned nm = __ballot_sync(FULL, visit); nm; nm &= nm - 1) {
            const int node = __shfl_sync(FULL, n, __ffs(nm) - 1);
            const float bound2 = knn_warp_max(valid ? b2 : -INFINITY);
            const int L = node * KNN_NODE + lane;
            const bool lv = L < nleaf && L != leaf && !(knn_box_box(leafbox[2 * L], leafbox[2 * L + 1], qlo, qhi) > bound2);
            for (unsigned lm = __ballot_sync(FULL, lv); lm; lm &= lm - 1) {
                const int Lk = node * KNN_NODE + __ffs(lm) - 1;
                const bool need = valid && !(knn_point_box(q, leafbox[2 * Lk], leafbox[2 * Lk + 1]) > b2);
                if (__any_sync(FULL, need)) knn_scan_leaf(P, sorted, Lk, lane, q, qid, b0, b1, b2);
            }
        }
    }
    if (valid) out[qid] = __fdiv_rn(__fadd_rn(__fadd_rn(b0, b1), b2), 3.0f);   // simple_knn.cu:182
}

// workspace layout of lgr_knn_mean_dist3 (every part 256-byte aligned)
struct KnnLayout {
    size_t bbox, codes, codes_sorted, ids, ids_sorted, sorted, leafbox, nodebox, cub, cub_bytes, total;
};

inline KnnLayout knn_layout(int P)
{
    KnnLayout L{};
    const size_t n = (size_t)(P > 0 ? P : 0);
    const size_t nleaf = (n + KNN_LEAF - 1) / KNN_LEAF, nnode = (nleaf + KNN_NODE - 1) / KNN_NODE;
    size_t o = 0;
    auto take = [&o](size_t bytes) { const size_t at = o; o = align_up(o + bytes, 256); return at; };
    L.bbox = take(6 * sizeof(unsigned));
    L.codes = take(n * sizeof(uint32_t));
    L.codes_sorted = take(n * sizeof(uint32_t));
    L.ids = take(n * sizeof(uint32_t));
    L.ids_sorted = take(n * sizeof(uint32_t));
    L.sorted = take(n * sizeof(float4));
    L.leafbox = take(2 * nleaf * sizeof(float4));
    L.nodebox = take(2 * nnode * sizeof(float4));
    L.cub_bytes = 0;
    if (P > 0)
        cub::DeviceRadixSort::SortPairs(nullptr, L.cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, P, 0, 30);
    L.cub = take(L.cub_bytes);
    L.total = o;
    return L;
}

}  // namespace
