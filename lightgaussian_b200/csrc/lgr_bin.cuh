// lgr_bin.cuh -- hand-written binning (round 2): the per-tile, depth-ordered instance lists without any library sort / scan,
// without the unsorted key / id arrays and without a host synchronisation in the middle.
//
// What must come out (RAST/cuda_rasterizer/rasterizer_impl.cu:70-138, 278-319): for every 16x16 tile the Gaussians that overlap
// it, ordered by (depth bits, Gaussian id) -- the order of the reference's stable 64-bit sort on (tile << 32 | depth).
//
//   1. depth order of the P Gaussians: LSD radix sort of the 32-bit depth keys in THREE passes of 11 / 11 / 10 bits (the library
//      sort took four 8-bit passes), ids implicit in the first pass, keys dropped in the last.
//   2. tile bucketing: ONE stable counting-sort pass over the (up to 32 768) tile indices.  Instances are never materialised
//      unsorted: a count kernel and a scatter kernel both regenerate them from the 16-byte per-Gaussian bin record
//      (tile rectangle + exact 64-bit keep mask, written by the preprocess kernel) walking the Gaussians in depth order.
//
// Every pass is the same three-kernel pattern on a count matrix M[BIN_V blocks][bins]:
//      count    block b histograms ITS contiguous chunk of the input in shared memory -> row b of M
//      scan     M[b][bin] <- sum over b' < b (exclusive, per bin); the last block to finish turns the bin totals into bin bases
//               (and, for the tile pass, writes the per-tile ranges, the instance total and the capacity-overflow flag)
//      scatter  block b re-reads its chunk IN ORDER; destination = base[bin] + M[b][bin] + (rank among the block's earlier items
//               of that bin).  Items are ranked 32 at a time: lanes holding the same bin are found with one ballot per key bit
//               (warp_match: cost = number of bits, where __match_any_sync costs one round per DISTINCT value -- measured 10x
//               slower on these mostly-distinct keys), the lowest lane of each group bumps a shared-memory counter, the others
//               add their position in the group.  Depth sort (2048 bins): every warp owns a contiguous eighth of the chunk and
//               a private row of counters, no warp waits for another.  Tile pass (8160 bins, one 32-bit cursor per tile): the
//               cursor updates of a block must follow the depth order; one ranking warp owns the cursors and consumes rows that
//               seven producer warps prepare ahead of it through a ring of shared-memory slots (full / empty mbarriers).
//
// The instance count R is needed on the host only to size the binning blob.  The blob is sized from a running estimate BEFORE the
// count is known; the kernels bound every store by that capacity and raise a flag when it is too small, the host looks at the
// count (a 16-byte copy that arrives while the blend kernel is already running) and repeats the scatter and the blend in the
// rare case of an overflow.  The GPU never idles on the host.
#pragma once

namespace {

constexpr int BIN_V = 528;            // blocks of every count / scatter kernel = rows of the count matrix (132 SMs x 4)
constexpr int DS_BITS = 11;
constexpr int DS_BINS = 1 << DS_BITS;
constexpr uint32_t BIN_NONE = 0xffffffffu;
constexpr int TB_THREADS = 192;       // tile scatter block: 5 producer warps + 1 ranking warp
constexpr int TC_THREADS = 256;       // tile count block: 8 warps
constexpr int TB_BUF = 256;           // instances of one 32-Gaussian row that fit a ring slot of the tile scatter
constexpr int SCAN_THREADS = 512;     // scan block: 16 warps share the rows of a 32-bin strip
constexpr int SCAN_ROWS = 40;         // rows per scan warp held in registers: BIN_V <= 16 * 40
constexpr int BIN_MAX_TILES = 32768;  // shared-memory cursor per tile (4 B) + staging: above this the library path is used

static_assert(BIN_V <= (SCAN_THREADS / 32) * SCAN_ROWS, "scan kernel: too many matrix rows");

__host__ __device__ inline int bin_pad(int bins) { return (bins + 255) / 256 * 256; }
inline int bin_per_block(int P) { return ((P + BIN_V - 1) / BIN_V + 255) / 256 * 256; }

// header words at the start of the geometry blob
// HDR_DET: 1 when the forward ran in deterministic mode (its records carry the permutation the deterministic backward needs)
// HDR_DEPTH: 1 + depth mode when the forward ran the depth/alpha blend (record word 11 holds z or 1/z), 0 otherwise; every forward
// clears words 0-15 before its blend
enum { HDR_LISTED = 0, HDR_RENDERED = 1, HDR_CAPACITY = 2, HDR_OVERFLOW = 3, HDR_DONE = 8, HDR_LIVE = 9, HDR_DET = 10, HDR_DEPTH = 11 };

// lanes with the same key (and valid) get the same mask of lanes; invalid lanes get 0.  One ballot per key bit.
template <int BITS>
__device__ __forceinline__ unsigned warp_match(uint32_t key, bool valid)
{
    unsigned m = __ballot_sync(FULL, valid);
#pragma unroll
    for (int b = 0; b < BITS; b++) {
        const bool bit = (key >> b) & 1u;
        const unsigned bal = __ballot_sync(FULL, bit);
        m &= bit ? bal : ~bal;
    }
    return valid ? m : 0u;
}

// shared-memory mbarriers (the tile scatter's turn hand-off): a waiting warp is suspended by the hardware instead of polling
__device__ __forceinline__ uint32_t bin_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bin_mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bin_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void bin_mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bin_smem_u32(bar)) : "memory");
}
// SLEEP_NS > 0: back off between polls.  Measured (profiles/r02e): a warp polling a barrier -- try_wait returns within tens of
// nanoseconds whatever suspend-time hint it is given -- takes issue slots and shared-memory bandwidth from the warps that work; with
// seven waiting warps per block the one working warp ran 5-10x slower.  So only the warp on the serial path polls hot.
template <int SLEEP_NS>
__device__ __forceinline__ void bin_mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok = 0;
    for (uint32_t spin = 0; !ok; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(bin_smem_u32(bar)), "r"(parity)
                     : "memory");
        if (!ok) {
            if (SLEEP_NS > 0) __nanosleep(SLEEP_NS);
            if (spin > (1u << 24)) {   // a protocol bug becomes an error, not a hung GPU
                printf("lgrast: tile scatter ring barrier timed out (block %d warp %d)\n", (int)blockIdx.x, (int)(threadIdx.x >> 5));
                __trap();
            }
        }
    }
}

// the same with a run-time number of key bits (tile indices: ceil(log2(tiles)) bits)
__device__ __forceinline__ unsigned warp_match_bits(uint32_t key, bool valid, int bits)
{
    unsigned m = __ballot_sync(FULL, valid);
    for (int b = 0; b < bits; b++) {
        const bool bit = (key >> b) & 1u;
        const unsigned bal = __ballot_sync(FULL, bit);
        m &= bit ? bal : ~bal;
    }
    return valid ? m : 0u;
}

// ------------------------------------------------------------------------------------------------
// depth sort: one LSD pass = count -> scan -> scatter
// ------------------------------------------------------------------------------------------------
template <int SHIFT, bool FIRST>
__global__ void __launch_bounds__(256) dsort_count_kernel(const uint32_t* __restrict__ keys, int P, int per_block, uint32_t* __restrict__ M,
                                                          int* __restrict__ header)
{
    __shared__ uint32_t hist[DS_BINS];
    for (int i = threadIdx.x; i < DS_BINS; i += 256) hist[i] = 0;
    if (FIRST && blockIdx.x == 0 && threadIdx.x < 16) header[threadIdx.x] = 0;
    __syncthreads();
    const int lo = blockIdx.x * per_block, hi = min(P, lo + per_block);   // lo is a multiple of 256: 16-byte aligned key quads
    for (int k = lo + 4 * (int)threadIdx.x; k < hi; k += 4 * 256) {
        const uint4 q = *reinterpret_cast<const uint4*>(keys + k);   // may read past hi, still inside the blob; masked below
        atomicAdd(&hist[(q.x >> SHIFT) & (DS_BINS - 1)], 1u);
        if (k + 1 < hi) atomicAdd(&hist[(q.y >> SHIFT) & (DS_BINS - 1)], 1u);
        if (k + 2 < hi) atomicAdd(&hist[(q.z >> SHIFT) & (DS_BINS - 1)], 1u);
        if (k + 3 < hi) atomicAdd(&hist[(q.w >> SHIFT) & (DS_BINS - 1)], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < DS_BINS; i += 256) M[(size_t)blockIdx.x * DS_BINS + i] = hist[i];
}

struct BinScanArgs {
    uint32_t* M;          // [V][bins_pad] counts in, exclusive prefixes over the blocks out
    int V, bins, bins_pad;
    uint32_t* bin_total;  // [bins_pad] scratch
    uint32_t* bin_base;   // [bins_pad] out: exclusive scan of the bin totals
    int* header;          // geometry header (done counter; tile pass: totals and flags)
    uint2* ranges;        // tile pass: [bins] per-tile [start, end)
    uint32_t capacity;    // tile pass: instances the binning blob can hold
};

template <bool TILES>
__global__ void __launch_bounds__(SCAN_THREADS) bin_scan_kernel(BinScanArgs a)
{
    constexpr int NW = SCAN_THREADS / 32;
    __shared__ uint32_t part[NW][32];
    __shared__ uint32_t wsum[NW];
    __shared__ bool last;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bin = blockIdx.x * 32 + lane;   // gridDim.x = bins_pad / 32
    const int rows_per = (a.V + NW - 1) / NW;  // <= SCAN_ROWS
    const int r0 = warp * rows_per, r1 = min(a.V, r0 + rows_per);
    uint32_t* col = a.M + bin;
    const size_t stride = (size_t)a.bins_pad;
    // the warp's rows of this 32-bin strip: every load in flight at once, the prefix runs over registers
    uint32_t v[SCAN_ROWS];
#pragma unroll
    for (int u = 0; u < SCAN_ROWS; u++) v[u] = (r0 + u < r1) ? col[(size_t)(r0 + u) * stride] : 0u;
    uint32_t s = 0;
#pragma unroll
    for (int u = 0; u < SCAN_ROWS; u++) s += v[u];
    part[warp][lane] = s;
    __syncthreads();
    uint32_t run = 0, total = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) {
        const uint32_t c = part[w][lane];
        if (w < warp) run += c;
        total += c;
    }
#pragma unroll
    for (int u = 0; u < SCAN_ROWS; u++) {
        if (r0 + u < r1) col[(size_t)(r0 + u) * stride] = run;
        run += v[u];
    }
    if (warp == 0) a.bin_total[bin] = total;

    // the last block to arrive scans the bin totals: every warp takes a contiguous segment, lanes read it 32 bins at a time (all the
    // segment's loads in flight before the carry chain starts), a warp scan per 32 bins, then the warp offsets
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(reinterpret_cast<unsigned*>(a.header + HDR_DONE), 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    constexpr int TB = 16;                                  // 32-bin groups fetched at once
    const int seg = a.bins_pad / NW;                          // bins per warp (bins_pad is a multiple of 256 = 16 warps x 16)
    const int nit = (seg + 31) / 32;
    const int sbase = warp * seg;
    uint32_t mine = 0;
    for (int it0 = 0; it0 < nit; it0 += TB) {
        uint32_t c[TB];
#pragma unroll
        for (int u = 0; u < TB; u++) {
            const int o = (it0 + u) * 32 + lane;
            c[u] = (it0 + u < nit && o < seg) ? __ldcg(a.bin_total + sbase + o) : 0u;
        }
#pragma unroll
        for (int u = 0; u < TB; u++) mine += c[u];
    }
    mine = __reduce_add_sync(FULL, mine);
    if (lane == 0) wsum[warp] = mine;
    __syncthreads();
    uint32_t carry = 0, grand = 0;
#pragma unroll
    for (int w = 0; w < NW; w++) {
        const uint32_t t = wsum[w];
        if (w < warp) carry += t;
        grand += t;
    }
    for (int it0 = 0; it0 < nit; it0 += TB) {
        uint32_t c[TB];
#pragma unroll
        for (int u = 0; u < TB; u++) {
            const int o = (it0 + u) * 32 + lane;
            c[u] = (it0 + u < nit && o < seg) ? __ldcg(a.bin_total + sbase + o) : 0u;
        }
#pragma unroll
        for (int u = 0; u < TB; u++) {
            uint32_t incl = c[u];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(FULL, incl, d);
                if (lane >= d) incl += t;
            }
            const int o = (it0 + u) * 32 + lane;
            if (it0 + u < nit && o < seg) {
                const uint32_t bs = carry + incl - c[u];
                a.bin_base[sbase + o] = bs;
                if (TILES && sbase + o < a.bins) a.ranges[sbase + o] = c[u] ? make_uint2(bs, bs + c[u]) : make_uint2(0u, 0u);   // empty tiles: (0,0), the reference's memset
            }
            carry += __shfl_sync(FULL, incl, 31);
        }
    }
    if (threadIdx.x == 0) {
        if (TILES) {
            a.header[HDR_LISTED] = (int)grand;
            a.header[HDR_CAPACITY] = (int)a.capacity;
            a.header[HDR_OVERFLOW] = grand > a.capacity ? 1 : 0;
        }
        a.header[HDR_DONE] = 0;   // ready for the next pass
    }
}

// Scatter of one depth-sort pass.  The block's chunk is cut into 4 contiguous sub-chunks, one per warp, so that "input order" inside the
// block is (warp, position in the warp's sub-chunk) and no warp ever waits for another: pass A counts every warp's digits into ITS row of
// a shared 4 x 2048 table (shared-memory atomics, no ordering needed), a prefix over the 4 rows turns the counts into each warp's first
// slot per digit, pass B walks the sub-chunk again and hands out the slots in order (warp_match + one read-modify-write per group).
// Keys are fetched four steps ahead (and come from L1 in pass B).
constexpr int DS_AHEAD = 4;
constexpr int DS_THREADS = 128;

template <int SHIFT, bool FIRST, bool LAST>
__global__ void __launch_bounds__(DS_THREADS) dsort_scatter_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ ids_in,
                                                                   uint32_t* __restrict__ keys_out, uint32_t* __restrict__ ids_out,
                                                                   const uint32_t* __restrict__ E, const uint32_t* __restrict__ bin_base, int P,
                                                                   int per_block)
{
    constexpr int BITS = (32 - SHIFT) < DS_BITS ? (32 - SHIFT) : DS_BITS;
    constexpr int NW = DS_THREADS / 32;
    __shared__ uint32_t wcnt[NW][DS_BINS];
    __shared__ uint32_t base[DS_BINS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < NW * DS_BINS; i += DS_THREADS) (&wcnt[0][0])[i] = 0u;
    for (int i = threadIdx.x; i < DS_BINS; i += DS_THREADS) base[i] = bin_base[i] + E[(size_t)blockIdx.x * DS_BINS + i];
    __syncthreads();
    const int lo = blockIdx.x * per_block, hi = min(P, lo + per_block);
    const int per_warp = per_block / NW;   // per_block is a multiple of 256
    const int wlo = lo + warp * per_warp, whi = min(hi, wlo + per_warp);
    uint32_t* mine = wcnt[warp];
    for (int k0 = wlo; k0 < whi; k0 += 32 * DS_AHEAD) {
        uint32_t key[DS_AHEAD];
#pragma unroll
        for (int j = 0; j < DS_AHEAD; j++) {
            const int k = k0 + 32 * j + lane;
            key[j] = k < whi ? keys_in[k] : 0u;
        }
#pragma unroll
        for (int j = 0; j < DS_AHEAD; j++)
            if (k0 + 32 * j + lane < whi) atomicAdd(&mine[(key[j] >> SHIFT) & (DS_BINS - 1)], 1u);
    }
    __syncthreads();
    for (int d = threadIdx.x; d < DS_BINS; d += DS_THREADS) {
        uint32_t run = base[d];
#pragma unroll
        for (int w = 0; w < NW; w++) {
            const uint32_t c = wcnt[w][d];
            wcnt[w][d] = run;
            run += c;
        }
    }
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
    for (int k0 = wlo; k0 < whi; k0 += 32 * DS_AHEAD) {
        uint32_t key[DS_AHEAD], id[DS_AHEAD];
#pragma unroll
        for (int j = 0; j < DS_AHEAD; j++) {
            const int k = k0 + 32 * j + lane;
            const bool valid = k < whi;
            key[j] = valid ? keys_in[k] : 0u;
            id[j] = FIRST ? (uint32_t)k : (valid ? ids_in[k] : 0u);
        }
#pragma unroll
        for (int j = 0; j < DS_AHEAD; j++) {
            const bool valid = k0 + 32 * j + lane < whi;
            const uint32_t d = (key[j] >> SHIFT) & (DS_BINS - 1);
            const unsigned m = warp_match<BITS>(d, valid);
            const int leader = __ffs(m) - 1;
            uint32_t old = 0;
            if (valid && lane == leader) {
                old = mine[d];
                mine[d] = old + (uint32_t)__popc(m);
            }
            __syncwarp();
            old = __shfl_sync(FULL, old, leader & 31);
            if (valid) {
                const uint32_t pos = old + (uint32_t)__popc(m & lt);
                if (!LAST) keys_out[pos] = key[j];
                ids_out[pos] = id[j];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// tile bucketing
// ------------------------------------------------------------------------------------------------
// bin record of a Gaussian (written by the preprocess kernels):  x = x0 | y0 << 16   y = w | h << 16   (z, w) = 64-bit keep mask.
// Tile b (row-major inside the w x h rectangle) is listed iff bit b is set; rectangles above 64 tiles are listed whole (mask all ones).
// Culled Gaussians have w = h = 0.
__device__ __forceinline__ uint4 make_bin_rec(int x0, int y0, int w, int h, unsigned long long mask)
{
    return make_uint4((uint32_t)x0 | ((uint32_t)y0 << 16), (uint32_t)w | ((uint32_t)h << 16), (uint32_t)mask, (uint32_t)(mask >> 32));
}

struct BinRowRaw {   // one lane's Gaussian of a 32-Gaussian row, as loaded
    uint32_t id;
    uint4 rec;
};

struct BinRow {   // ... and decoded
    uint32_t id, cnt, off, total, area;
    int x0, y0, w;
    unsigned long long mask;
};

__device__ __forceinline__ BinRowRaw bin_row_fetch(const uint32_t* __restrict__ sorted_ids, const uint4* __restrict__ bin_rec, int k, int kend)
{
    BinRowRaw r;
    r.id = 0;
    r.rec = make_uint4(0u, 0u, 0u, 0u);
    if (k < kend) {
        r.id = sorted_ids[k];
        r.rec = __ldg(bin_rec + r.id);
    }
    return r;
}

__device__ __forceinline__ void bin_row_decode(const BinRowRaw& in, int lane, BinRow& r)
{
    r.id = in.id; r.cnt = 0; r.x0 = 0; r.y0 = 0; r.w = 1; r.mask = ~0ull;
    const uint4 q = in.rec;
    const int w = (int)(q.y & 0xffffu), h = (int)(q.y >> 16);
    r.area = (uint32_t)(w * h);
    if (r.area) {
        r.x0 = (int)(q.x & 0xffffu); r.y0 = (int)(q.x >> 16); r.w = w;
        r.mask = (unsigned long long)q.z | ((unsigned long long)q.w << 32);
        r.cnt = r.area > 64u ? r.area : (uint32_t)__popcll(r.mask);
    }
    uint32_t incl = r.cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += t;
    }
    r.off = incl - r.cnt;
    r.total = __shfl_sync(FULL, incl, 31);
}

// instance j (row-local, j < r.total for valid lanes) -> tile index, owner id and owner lane; BIN_NONE for lanes past the end
__device__ __forceinline__ uint32_t bin_row_instance(const BinRow& r, uint32_t j, int gx, uint32_t& owner_id, int& owner_lane)
{
    int lo = 0, hi = 31;   // largest lane m with off[m] <= j
#pragma unroll
    for (int it = 0; it < 5; it++) {
        const int mid = (lo + hi + 1) >> 1;
        const uint32_t v = __shfl_sync(FULL, r.off, mid);
        if (v <= j) lo = mid;
        else hi = mid - 1;
    }
    const uint32_t o_off = __shfl_sync(FULL, r.off, lo);
    owner_id = __shfl_sync(FULL, r.id, lo);
    owner_lane = lo;
    const int o_x0 = __shfl_sync(FULL, r.x0, lo), o_y0 = __shfl_sync(FULL, r.y0, lo), o_w = __shfl_sync(FULL, r.w, lo);
    const unsigned long long o_mask = __shfl_sync(FULL, r.mask, lo);
    if (j >= r.total) return BIN_NONE;
    int local = (int)(j - o_off);
    if (o_mask != ~0ull) {   // local-th kept tile of the rectangle
        const uint32_t mlo = (uint32_t)o_mask;
        const int clo = __popc(mlo);
        local = local < clo ? (int)__fns(mlo, 0, local + 1) : 32 + (int)__fns((uint32_t)(o_mask >> 32), 0, local - clo + 1);
    }
    const int ry = (int)__fdividef((float)local + 0.5f, (float)o_w);   // exact: |error| << 0.5 / w for rectangles of a few thousand tiles
    const int rx = local - ry * o_w;
    return (uint32_t)((o_y0 + ry) * gx + (o_x0 + rx));
}

// the lane's OWN Gaussian (rectangle of at most 64 tiles): its kept tiles in row-major order -> f(tile, j), j = 0 .. cnt-1.
// For rows of small splats (the common case: 3-4 kept tiles per Gaussian) this per-lane walk costs a third of the instructions of the
// warp-cooperative expansion (owner search + seven shuffles per instance), which remains the path for rows with larger rectangles.
template <class F>
__device__ __forceinline__ void bin_lane_tiles(const BinRow& r, int gx, F f)
{
    unsigned long long m = r.cnt ? r.mask : 0ull;
    const float fw = (float)r.w;
    uint32_t j = 0;
    while (m) {
        const int b = __ffsll((long long)m) - 1;
        m &= m - 1;
        const int ry = (int)__fdividef((float)b + 0.5f, fw), rx = b - ry * r.w;
        f((uint32_t)((r.y0 + ry) * gx + (r.x0 + rx)), j++);
    }
}

__global__ void __launch_bounds__(TC_THREADS) tile_count_kernel(const uint32_t* __restrict__ sorted_ids, const uint4* __restrict__ bin_rec, int P,
                                                                int per_block, int gx, int tiles_pad, uint32_t* __restrict__ M, int* __restrict__ header)
{
    extern __shared__ uint32_t tb_smem[];
    uint32_t* hist = tb_smem;
    for (int i = threadIdx.x; i < tiles_pad; i += TC_THREADS) hist[i] = 0;
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int lo = blockIdx.x * per_block, hi = min(P, lo + per_block);
    constexpr int STEP = (TC_THREADS / 32) * 32;
    uint32_t area = 0;
    int row = lo + warp * 32;
    BinRowRaw next = bin_row_fetch(sorted_ids, bin_rec, row + lane, hi);
    for (; row < hi; row += STEP) {
        const BinRowRaw cur = next;
        next = bin_row_fetch(sorted_ids, bin_rec, row + STEP + lane, hi);   // the next row's loads fly while this one is expanded
        BinRow r;
        bin_row_decode(cur, lane, r);
        area += r.area;
        if (__all_sync(FULL, r.area <= 64u)) {
            bin_lane_tiles(r, gx, [&](uint32_t tile, uint32_t) { atomicAdd(&hist[tile], 1u); });
        } else {
            for (uint32_t base = 0; base < r.total; base += 32) {
                uint32_t owner;
                int olane;
                const uint32_t tile = bin_row_instance(r, base + lane, gx, owner, olane);
                if (tile != BIN_NONE) atomicAdd(&hist[tile], 1u);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < tiles_pad; i += TC_THREADS) M[(size_t)blockIdx.x * tiles_pad + i] = hist[i];
    // the reference's num_rendered = sum of the rectangle areas (rasterizer_impl.cu:278-283)
    area = __reduce_add_sync(FULL, area);
    if (lane == 0 && area) atomicAdd(reinterpret_cast<unsigned*>(header + HDR_RENDERED), area);
}

// ---- tile scatter: producer warps, one ranking warp, a ring of row slots between them ----
constexpr int TS_SLOTS = 8;                 // rows in flight between producers and the ranker
constexpr int TS_SLOT = TB_BUF;             // instances a slot holds (one 32-Gaussian row; larger rows travel raw)
constexpr int TS_PRODUCERS = TB_THREADS / 32 - 1;
constexpr uint32_t TS_RAW = 0xffffffffu;

struct TileSlot {
    uint32_t mask[TS_SLOT];   // group mask of the instance inside its 32-instance step   (raw rows: the 32 bin records, 4 words each)
    uint32_t id[TS_SLOT];     // Gaussian id                                              (raw rows: the 32 ids)
    uint16_t tile[TS_SLOT];
};

inline size_t tile_scatter_smem(int tiles_pad) { return sizeof(uint32_t) * (size_t)tiles_pad + sizeof(TileSlot) * TS_SLOTS; }

__global__ void __launch_bounds__(TB_THREADS) tile_scatter_kernel(const uint32_t* __restrict__ sorted_ids, const uint4* __restrict__ bin_rec, int P,
                                                                  int per_block, int gx, int tiles_pad, const uint32_t* __restrict__ E,
                                                                  const uint32_t* __restrict__ bin_base, const int* __restrict__ header,
                                                                  uint32_t* __restrict__ point_list)
{
    // The cursor of a tile must be advanced in depth order, i.e. row after row of the block's chunk.  ONE warp (the ranker) owns the
    // cursors and walks the rows in order; the other seven warps prepare rows ahead of it: load (the next row's loads already in flight),
    // expand the row into its instances in row order, group every 32-instance step by tile (warp_match), and publish {tile, group mask,
    // Gaussian id} per instance in a ring slot (full / empty mbarriers, as in the blend kernels).  Per step the ranker does three shared
    // loads, one cursor read-modify-write by the lowest lane of each group, one shuffle and the store -- nothing else sits on the serial
    // path, and nobody but the ranker ever waits on the critical hand-off.  (Earlier versions passed a ticket between eight equal warps:
    // the seven waiting warps' polling -- shared-memory spin, __nanosleep or mbarrier.try_wait alike -- slowed the one working warp 5-10x.)
    extern __shared__ uint32_t tb_smem[];
    uint32_t* cursor = tb_smem;                                              // [tiles_pad]
    TileSlot* slots = reinterpret_cast<TileSlot*>(tb_smem + tiles_pad);      // [TS_SLOTS]
    __shared__ __align__(8) uint64_t full[TS_SLOTS];
    __shared__ __align__(8) uint64_t empty[TS_SLOTS];
    __shared__ uint32_t slot_n[TS_SLOTS];
    for (int i = threadIdx.x; i < tiles_pad; i += TB_THREADS) cursor[i] = bin_base[i] + E[(size_t)blockIdx.x * tiles_pad + i];
    if (threadIdx.x == 0) {
        for (int k = 0; k < TS_SLOTS; k++) {
            bin_mbar_init(&full[k], 1);
            bin_mbar_init(&empty[k], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t capacity = (uint32_t)header[HDR_CAPACITY];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int lo = blockIdx.x * per_block, hi = min(P, lo + per_block);
    const int nrows = (hi - lo + 31) / 32;
    const unsigned lt = (1u << lane) - 1u;
    int tbits = 1;
    while ((1 << tbits) < tiles_pad) tbits++;

    if (warp < TS_PRODUCERS) {
        BinRowRaw next = bin_row_fetch(sorted_ids, bin_rec, lo + warp * 32 + lane, hi);
        for (int t = warp; t < nrows; t += TS_PRODUCERS) {
            const BinRowRaw cur = next;
            next = bin_row_fetch(sorted_ids, bin_rec, lo + (t + TS_PRODUCERS) * 32 + lane, hi);
            BinRow r;
            bin_row_decode(cur, lane, r);
            const int k = t % TS_SLOTS;
            const uint32_t ph = (uint32_t)(t / TS_SLOTS) & 1u;
            bin_mbar_wait<2000>(&empty[k], ph ^ 1u);   // passes at once the first time round; producers can afford to doze
            TileSlot& sl = slots[k];
            if (r.total <= (uint32_t)TS_SLOT) {
                if (__all_sync(FULL, r.area <= 64u)) {
                    bin_lane_tiles(r, gx, [&](uint32_t tile, uint32_t j) {
                        sl.tile[r.off + j] = (uint16_t)tile;
                        sl.id[r.off + j] = r.id;
                    });
                } else {
                    for (uint32_t base = 0; base < r.total; base += 32) {
                        uint32_t owner;
                        int olane;
                        const uint32_t tile = bin_row_instance(r, base + lane, gx, owner, olane);
                        if (tile != BIN_NONE) {
                            sl.tile[base + lane] = (uint16_t)tile;
                            sl.id[base + lane] = owner;
                        }
                    }
                }
                __syncwarp();
                for (uint32_t base = 0; base < r.total; base += 32) {
                    const bool valid = base + lane < r.total;
                    const uint32_t tile = valid ? (uint32_t)sl.tile[base + lane] : 0u;
                    const unsigned m = warp_match_bits(tile, valid, tbits);
                    if (valid) sl.mask[base + lane] = m;
                }
                if (lane == 0) slot_n[k] = r.total;
            } else {   // a row of screen-filling splats: hand the row itself to the ranker
                sl.id[lane] = cur.id;
                sl.mask[4 * lane + 0] = cur.rec.x; sl.mask[4 * lane + 1] = cur.rec.y; sl.mask[4 * lane + 2] = cur.rec.z; sl.mask[4 * lane + 3] = cur.rec.w;
                if (lane == 0) slot_n[k] = TS_RAW;
            }
            __syncwarp();
            if (lane == 0) bin_mbar_arrive(&full[k]);   // release: the slot's contents are visible to the ranker
        }
        return;
    }

    // ---- the ranker ----
    for (int t = 0; t < nrows; t++) {
        const int k = t % TS_SLOTS;
        const uint32_t ph = (uint32_t)(t / TS_SLOTS) & 1u;
        bin_mbar_wait<0>(&full[k], ph);
        const TileSlot& sl = slots[k];
        const uint32_t n = slot_n[k];
        if (n != TS_RAW) {
            for (uint32_t base = 0; base < n; base += 32) {
                const bool valid = base + lane < n;
                uint32_t tile = 0, id = 0;
                unsigned m = 0;
                if (valid) {
                    tile = sl.tile[base + lane];
                    m = sl.mask[base + lane];
                    id = sl.id[base + lane];
                }
                const int leader = __ffs(m) - 1;
                uint32_t old = 0;
                if (valid && lane == leader) {
                    old = cursor[tile];
                    cursor[tile] = old + (uint32_t)__popc(m);
                }
                __syncwarp();
                const uint32_t pos = __shfl_sync(FULL, old, leader & 31) + (uint32_t)__popc(m & lt);
                if (valid && pos < capacity) point_list[pos] = id;
            }
        } else {
            BinRowRaw raw;
            raw.id = sl.id[lane];
            raw.rec = make_uint4(sl.mask[4 * lane + 0], sl.mask[4 * lane + 1], sl.mask[4 * lane + 2], sl.mask[4 * lane + 3]);
            BinRow r;
            bin_row_decode(raw, lane, r);
            for (uint32_t base = 0; base < r.total; base += 32) {
                uint32_t owner;
                int olane;
                const uint32_t tile = bin_row_instance(r, base + lane, gx, owner, olane);
                const bool valid = tile != BIN_NONE;
                const unsigned m = warp_match_bits(tile, valid, tbits);
                const int leader = __ffs(m) - 1;
                uint32_t old = 0;
                if (valid && lane == leader) {
                    old = cursor[tile];
                    cursor[tile] = old + (uint32_t)__popc(m);
                }
                __syncwarp();
                const uint32_t pos = __shfl_sync(FULL, old, leader & 31) + (uint32_t)__popc(m & lt);
                if (valid && pos < capacity) point_list[pos] = owner;
            }
        }
        __syncwarp();
        if (lane == 0) bin_mbar_arrive(&empty[k]);
    }
}

}  // namespace
