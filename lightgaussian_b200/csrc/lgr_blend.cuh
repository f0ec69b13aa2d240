// lgr_blend.cuh -- round-2 blend kernels (K4/K5 forward, K6 backward): shared per-tile staging ring + instruction diet.
//
// Block = one 16x16 tile: 8 consumer warps (warp w owns the 8x4 pixel sub-tile (w&1, w>>1), exactly as before) + 1 producer warp.
// The tile's depth-sorted instance list is streamed through a 4-stage shared-memory ring of 32-record chunks; a record is 48 bytes
//     q0 = (mean2D.x, mean2D.y, conic.x, conic.y)   q1 = (conic.z, opacity, r, g)   q2 = (b, Gaussian id, -, -)
// full[s] / empty[s] mbarriers hand the stages back and forth, so the 8 warps no longer gather every list entry 8 times over.
//
//   forward : the producer warp gathers (point_list -> means2D / conic_opacity / rgb) ONCE per tile into the stage, and writes the
//             stage out to the per-instance record array of the binning blob with one TMA bulk store (cp.async.bulk S2G) -- only the
//             chunks the tile actually visits before its pixels saturate (~25 % of the lists) ever exist.
//   backward: no gather at all -- one elected producer thread streams those records back with TMA bulk loads (cp.async.bulk G2S,
//             mbarrier complete_tx), back to front; the consumers read records from the stage only.
//
// Instruction diet of the inner (warp, Gaussian) loop (the kernels are issue-bound, profiles/r01c_ncu_full_summary.txt):
//   * "done" is the sign of T: a finished pixel keeps T = -|T|, T*(1-alpha) < 1e-4 then holds forever and the reference's own
//     termination branch freezes it -- no flag register, no skip branch, no predicate juggling; final_T = |T|.
//   * one address computation per record (three LDS at immediate offsets), uniform loop control.
//   * backward: the nine per-lane partial sums of a pair are LINEAR in two scalars, w = alpha*T and wg = G*dL/dalpha, with per-lane
//     coefficients that do not change during the whole kernel (the pixel's dL/dpix and its integer offset inside the sub-tile):
//         dL/dcolor[c] = sum_l w[l] * dpix_c[l]          S_k = sum_l wg[l] * {1, x_l, y_l, x_l^2, x_l y_l, y_l^2}
//     so a pair parks TWO floats per lane (was nine), and every 16 pairs the warp contracts the 16x32 tables against the coefficient
//     table in shared memory -- lane p owns pair p, half-warps split the 32 source lanes, immediates for the offsets -- converts the
//     moments from sub-tile-origin to Gaussian-centred form and adds the nine sums to the record with two 16-byte vector reductions
//     and one scalar reduction (three L2 atomic operations per pair, not nine).  ~14 instructions per pair instead of ~45.
//   * backward: exp through ex2.approx on log2(e)*power (1e-3 contract), non-contributing lanes are folded in as alpha = 0
//     (neutral for T, the colour recurrence and every sum), so the pair body is branch-free.
#pragma once

namespace {

constexpr int BL_CH = 32;            // records per chunk
constexpr int BL_STAGES = 4;
constexpr int BL_REC = 12;           // floats per record
constexpr int BL_THREADS = 288;      // 8 consumer warps + 1 producer warp
constexpr uint32_t BL_END = 0xffffffffu;
constexpr int BL_FLUSH = 16;         // pairs buffered between backward flushes
constexpr int BL_ROW = 33;           // floats per buffered pair row (32 lanes + 1 pad: conflict-free transposed reads)

__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// unbounded-looking wait with a trap: a protocol bug becomes an error, not a hung GPU
__device__ __forceinline__ void mbar_wait_ring(uint64_t* bar, uint32_t parity)
{
    for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
        if (spin > (1u << 26)) {
            printf("lgrast: blend ring barrier timed out (block %d warp %d)\n", (int)blockIdx.x, (int)(threadIdx.x >> 5));
            __trap();
        }
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// two float atomic adds to consecutive words as one vector reduction (SASS REDG.E.ADD.F32x2); `addr` must be 8-byte aligned
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b)
{
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}
// four float atomic adds to consecutive words as ONE vector reduction (sm_90, SASS REDG.E.ADD.F32x4): one L2 operation instead of four.
// `addr` must be 16-byte aligned.  Like atomicAdd on f32, it flushes subnormals to zero.
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// sub-tile cull with a magnitude-aware margin: the 1 % alpha margin covers the rounding of q only while its terms stay below ~1e4;
// an elongated splat far from the rectangle can cancel terms of 1e6-1e7 down to a small q, so the rounding bound of the evaluated
// terms is added to the threshold (never culls a pair the reference would blend).
__device__ __forceinline__ bool subtile_cull2(float gxp, float gyp, float A, float B, float Cc, float o, float rx0, float rx1, float ry0, float ry1)
{
    const float t = 257.55f * o;  // 255 * 1.01 * opacity
    if (t <= 1.0f) return true;
    const float dx_lo = gxp - rx1, dx_hi = gxp - rx0, dy_lo = gyp - ry1, dy_hi = gyp - ry0;
    const float cx = fminf(fmaxf(0.f, dx_lo), dx_hi), cy = fminf(fmaxf(0.f, dy_lo), dy_hi);
    if (cx == 0.f && cy == 0.f) return false;
    if (!(A > 0.f && Cc > 0.f && A * Cc - B * B > 0.f)) return false;
    const float thr = __logf(t);
    float qmin = 3.0e38f, mag = 0.f;
    if (cx != 0.f) {
        const float dy = fminf(fmaxf(__fdividef(-B * cx, Cc), dy_lo), dy_hi);
        const float t0 = A * cx * cx, t1 = Cc * dy * dy, t2 = B * cx * dy;
        qmin = 0.5f * (t0 + t1) + t2;
        mag = t0 + t1 + fabsf(t2);
    }
    if (cy != 0.f) {
        const float dx = fminf(fmaxf(__fdividef(-B * cy, A), dx_lo), dx_hi);
        const float t0 = A * dx * dx, t1 = Cc * cy * cy, t2 = B * dx * cy;
        const float q = 0.5f * (t0 + t1) + t2;
        if (q < qmin) { qmin = q; mag = t0 + t1 + fabsf(t2); }
    }
    return qmin > thr + 2.0e-6f * mag;
}

// ---- zero-fill of the dense per-Gaussian gradient rows (see lgr_sparse.cuh, "Single-GPU K7+K8 on the compacted list") ----
constexpr int KB_ZERO_BYTES = 5760;   // 32 rows x 45 floats: the dense dL/dfeatures_rest run of one warp at degree 3

struct KbackZeroArgs {
    int P, nrest;
    const int* radii;
    const float* acc;
    int* idx;        // [P] out: ids with a non-zero gradient (unordered)
    int* counter;    // out: how many
    float* d_xyz; float* d_dc; float* d_rest; float* d_scaling; float* d_rotation; float* d_opacity; float* dL_dmeans2D;
};

__device__ __forceinline__ void bulk_zero(float* dst, size_t floats, const void* zero_page)
{
    size_t bytes = floats * 4;
    char* p = reinterpret_cast<char*>(dst);
    while (bytes) {
        const uint32_t n = (uint32_t)(bytes < (size_t)KB_ZERO_BYTES ? bytes : (size_t)KB_ZERO_BYTES);
        bulk_s2g(p, zero_page, n);
        p += n;
        bytes -= n;
    }
}


// the tile's share of the rows: tiles split [0, P) into runs of G Gaussians, G a multiple of 4 so that every run of every tensor starts
// 16-byte aligned and is a multiple of 16 bytes (cp.async.bulk's granularity); the tail that is not is cleared with plain stores
__device__ __forceinline__ void tile_zero_rows(const KbackZeroArgs& z, int tile, int tiles, const void* zero_page)
{
    const int G = ((z.P + tiles - 1) / tiles + 3) & ~3;
    const long long first = (long long)tile * G;
    if (first >= z.P) return;
    const int n = (int)min((long long)G, z.P - first), nb = n & ~3;
    if (nb) {
        bulk_zero(z.d_rest + (size_t)first * z.nrest, (size_t)nb * z.nrest, zero_page);
        bulk_zero(z.d_dc + (size_t)first * 3, (size_t)nb * 3, zero_page);
        bulk_zero(z.d_xyz + (size_t)first * 3, (size_t)nb * 3, zero_page);
        bulk_zero(z.d_scaling + (size_t)first * 3, (size_t)nb * 3, zero_page);
        bulk_zero(z.d_rotation + (size_t)first * 4, (size_t)nb * 4, zero_page);
        bulk_zero(z.d_opacity + (size_t)first, (size_t)nb, zero_page);
        bulk_zero(z.dL_dmeans2D + (size_t)first * 3, (size_t)nb * 3, zero_page);
        bulk_commit();
    }
    for (long long i = first + nb; i < first + n; i++) {   // at most 3 Gaussians, last run only
        for (int k = 0; k < z.nrest; k++) z.d_rest[(size_t)i * z.nrest + k] = 0.f;
        for (int k = 0; k < 3; k++) {
            z.d_dc[(size_t)i * 3 + k] = 0.f; z.d_xyz[(size_t)i * 3 + k] = 0.f; z.d_scaling[(size_t)i * 3 + k] = 0.f; z.dL_dmeans2D[(size_t)i * 3 + k] = 0.f;
        }
        for (int k = 0; k < 4; k++) z.d_rotation[(size_t)i * 4 + k] = 0.f;
        z.d_opacity[(size_t)i] = 0.f;
    }
}

struct BlendRing {
    float rec[BL_STAGES][BL_CH * BL_REC];
    uint64_t full[BL_STAGES];
    uint64_t empty[BL_STAGES];
    uint32_t count[BL_STAGES];
    int live;
    unsigned tile_max;
};

__device__ __forceinline__ void ring_init(BlendRing& r, int consumers)
{
    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < BL_STAGES; s++) {
            mbar_init(&r.full[s], 1);
            mbar_init(&r.empty[s], consumers);
        }
        r.live = consumers;
        r.tile_max = 0;
        fence_mbar_init();
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// K4/K5 forward
// ------------------------------------------------------------------------------------------------
// PERM (deterministic mode): word 10 of each stored record is the instance's unsorted index perm[pos], which the deterministic
// backward uses to address its per-instance partial rows.
// WEIGHT (count mode only): also weight[i] += sum over the pixels that blend Gaussian i of q = rint(fl(alpha*T) * 2^32), alpha*T
// being the share of the pixel's colour the Gaussian supplies (DESIGN section 3, "Blending-weight significance").  q < 0.99*2^32
// fits 32 bits; the warp sums each 16-bit half with REDUX (< 2^21, exact) and lane 0 adds them with one 64-bit integer atomic, so the
// per-view sums are exact and independent of every ordering.
// DEPTH (lgr_forward_raw_depth, DESIGN section 7): the producer also stores each Gaussian's depth value (z, 1/z, or 0 when only alpha
// is wanted) in record word 11, each lane blends it with the pixel's colour weights in the colour's operation order, and the epilogue
// writes the depth plane sum_i alpha_i*T_i*value_i and the alpha plane fl(1 - final_T); the mode goes to header word HDR_DEPTH.
struct BlendDepth {
    const float* z;   // [P] view-space depth of the geometry blob
    float* depth;     // [H,W] out, or NULL
    float* alpha;     // [H,W] out, or NULL
    int* header;      // the geometry header (HDR_DEPTH := 1 + mode)
    int mode;         // 0 = alpha only (value 0), 1 = z, 2 = 1/z (correctly rounded)
};

template <bool COUNT, bool STORE, bool PERM = false, bool WEIGHT = false, bool DEPTH = false>
__global__ void __launch_bounds__(BL_THREADS)
blend_forward_ring_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H, int tiles_x,
                          const float2* __restrict__ means2D, const float4* __restrict__ conic_opacity, const float4* __restrict__ rgb,
                          const float* __restrict__ bg, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                          float* __restrict__ out_color, int* __restrict__ count, float* __restrict__ rec_out, const int* __restrict__ header,
                          const uint32_t* __restrict__ perm = nullptr, unsigned long long* __restrict__ weight = nullptr,
                          BlendDepth dz = BlendDepth{})
{
    static_assert(!WEIGHT || COUNT, "the blending weight is a count-mode output");
    static_assert(!DEPTH || (!COUNT && STORE && !PERM && !WEIGHT), "depth and alpha are outputs of the default training forward only");
    if (header[HDR_OVERFLOW]) return;   // the binning blob was too small for this view: the host repeats scatter + blend (lgr_bin.cuh)
    if (DEPTH && blockIdx.x == 0 && threadIdx.x == 0) dz.header[HDR_DEPTH] = 1 + dz.mode;
    __shared__ __align__(128) BlendRing ring;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    const uint2 range = ranges[tile];
    ring_init(ring, 8);

    if (warp == 8) {
        // ===== producer warp: gather the tile's list once, 32 instances per stage =====
        for (uint32_t c = 0;; c++) {
            const int s = c % BL_STAGES;
            const uint32_t ph = (c / BL_STAGES) & 1u;
            mbar_wait_ring(&ring.empty[s], ph ^ 1u);
            if (STORE) {  // the bulk store issued from this stage BL_STAGES chunks ago must have read it out
                if (lane == 0) bulk_wait_read<BL_STAGES - 1>();
                __syncwarp();
            }
            const uint32_t pos0 = range.x + c * BL_CH;
            const int live = *reinterpret_cast<volatile int*>(&ring.live);
            if (pos0 >= range.y || live <= 0) {
                if (lane == 0) {
                    ring.count[s] = BL_END;
                    mbar_arrive(&ring.full[s]);
                }
                break;
            }
            const uint32_t n = min((uint32_t)BL_CH, range.y - pos0);
            if ((uint32_t)lane < n) {
                const uint32_t id = point_list[pos0 + lane];
                const float2 xy = means2D[id];
                const float4 co = conic_opacity[id];
                const float4 col = rgb[id];
                float4* r4 = reinterpret_cast<float4*>(&ring.rec[s][lane * BL_REC]);
                r4[0] = make_float4(xy.x, xy.y, co.x, co.y);
                r4[1] = make_float4(co.z, co.w, col.x, col.y);
                float zv = 0.f;
                if (DEPTH && dz.mode != 0) zv = dz.mode == 2 ? __frcp_rn(dz.z[id]) : dz.z[id];
                r4[2] = make_float4(col.z, __uint_as_float(id), PERM ? __uint_as_float(perm[pos0 + lane]) : 0.f, zv);
            }
            if (lane == 0) ring.count[s] = n;
            if (STORE) fence_async_smem();
            __syncwarp();
            if (lane == 0) {
                if (STORE) {
                    bulk_s2g(rec_out + (size_t)pos0 * BL_REC, &ring.rec[s][0], n * (uint32_t)(BL_REC * 4));
                    bulk_commit();
                }
                mbar_arrive(&ring.full[s]);
            }
        }
        if (STORE && lane == 0) bulk_wait_all();
        return;
    }

    // ===== consumer warps =====
    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int sx0 = tx * LGR_TILE + (warp & 1) * 8, sy0 = ty * LGR_TILE + (warp >> 1) * 4;
    const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
    const bool inside = px < W && py < H;
    float pxf = (float)px, pyf = (float)py;
    const float rx0 = (float)sx0, rx1 = (float)min(sx0 + 7, W - 1), ry0 = (float)sy0, ry1 = (float)min(sy0 + 3, H - 1);

    float T = inside ? 1.0f : -1.0f;  // sign = "done"
    float C0 = 0.f, C1 = 0.f, C2 = 0.f;
    float Cz = 0.f;   // DEPTH: the depth value's blend
    uint32_t last = 0;
    bool warp_done = __all_sync(FULL, T < 0.f);
    if (warp_done && lane == 0) atomicSub(&ring.live, 1);

    for (uint32_t c = 0;; c++) {
        const int s = c % BL_STAGES;
        const uint32_t ph = (c / BL_STAGES) & 1u;
        mbar_wait_ring(&ring.full[s], ph);
        const uint32_t n = ring.count[s];
        if (n == BL_END) break;
        if (!warp_done) {
            const float* stage = &ring.rec[s][0];
            bool keep = false;
            if ((uint32_t)lane < n) {
                const float4 q0 = *reinterpret_cast<const float4*>(stage + lane * BL_REC);
                const float4 q1 = *reinterpret_cast<const float4*>(stage + lane * BL_REC + 4);   // 128-bit: conflict-free at the 48-byte stride
                keep = !subtile_cull2(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, rx0, rx1, ry0, ry1);
            }
            unsigned mask = __ballot_sync(FULL, keep);
            const uint32_t pos_base = c * BL_CH + 1u;
            while (mask) {
                const int j = __ffs(mask) - 1;
                mask &= mask - 1;
                const float* r = stage + j * BL_REC;
                const float4 q0 = *reinterpret_cast<const float4*>(r);
                const float4 q1 = *reinterpret_cast<const float4*>(r + 4);
                const float dx = LGR_SUB(q0.x, pxf), dy = LGR_SUB(q0.y, pyf);
                const float power = lgr::pair_power(dx, dy, q0.z, q0.w, q1.x);
                bool contrib = false;
                uint32_t q = 0;   // WEIGHT: this lane's fixed-point alpha*T (0 when it does not blend the Gaussian)
                if (!(power > 0.0f)) {
                    const float alpha = fminf(0.99f, LGR_MUL(q1.y, expf(power)));
                    if (!(alpha < 1.0f / 255.0f)) {
                        const float test_T = LGR_MUL(T, LGR_SUB(1.0f, alpha));
                        if (test_T < 0.0001f) {
                            T = -fabsf(T);  // done (and stays done: T < 0 keeps test_T below the threshold)
                        } else {
                            const float b = r[8];
                            C0 = LGR_FMA(T, LGR_MUL(alpha, q1.z), C0);
                            C1 = LGR_FMA(T, LGR_MUL(alpha, q1.w), C1);
                            C2 = LGR_FMA(T, LGR_MUL(alpha, b), C2);
                            if (DEPTH) Cz = LGR_FMA(T, LGR_MUL(alpha, r[11]), Cz);
                            if (WEIGHT) q = __float2uint_rn(__fmul_rn(__fmul_rn(alpha, T), 4294967296.0f));   // 2^32: exact scaling
                            T = test_T;
                            last = pos_base + (uint32_t)j;
                            contrib = true;
                        }
                    }
                }
                if (COUNT) {
                    const unsigned cm = __ballot_sync(FULL, contrib);
                    if (cm != 0 && lane == 0) atomicAdd(&count[__float_as_uint(r[9])], __popc(cm));
                    if (WEIGHT && cm != 0) {
                        const unsigned lo = __reduce_add_sync(FULL, q & 0xffffu), hi = __reduce_add_sync(FULL, q >> 16);
                        if (lane == 0) atomicAdd(&weight[__float_as_uint(r[9])], ((unsigned long long)hi << 16) + lo);
                    }
                }
                if (__all_sync(FULL, T < 0.f)) break;
            }
            warp_done = __all_sync(FULL, T < 0.f);
            if (warp_done && lane == 0) atomicSub(&ring.live, 1);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&ring.empty[s]);
    }
    if (inside) {
        const size_t pix = (size_t)py * W + px;
        const size_t plane = (size_t)H * W;
        const float Tf = fabsf(T);
        final_T[pix] = Tf;
        n_contrib[pix] = last;
        out_color[pix] = LGR_FMA(bg[0], Tf, C0);
        out_color[plane + pix] = LGR_FMA(bg[1], Tf, C1);
        out_color[2 * plane + pix] = LGR_FMA(bg[2], Tf, C2);
        if (DEPTH) {
            if (dz.depth) dz.depth[pix] = Cz;
            if (dz.alpha) dz.alpha[pix] = __fsub_rn(1.0f, Tf);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// K6 backward
// ------------------------------------------------------------------------------------------------
struct BlendBackWarp {
    float w[BL_FLUSH][BL_ROW];     // alpha*T per (buffered pair, lane)
    float g[BL_FLUSH][BL_ROW];     // G*dL/dalpha
    float mid[BL_FLUSH], mgx[BL_FLUSH], mgy[BL_FLUSH];   // per buffered pair: Gaussian id (bits), mean2D.x, mean2D.y
    float4 d[32];                  // the lanes' dL/dpix (r, g, b) and, DEPTH, dL/ddepth
};

// The absgrad backward's per-warp buffer (blend_backward_absgrad_kernel): the pair's conic and opacity next to its mean, so the flush
// can form each source lane's |dL/dmean2D| term from the parked g and the lane's pixel offset.  256 bytes more per warp.
struct BlendBackWarpAbs : BlendBackWarp {
    float4 mco[BL_FLUSH];          // per buffered pair: (conic A, conic B, conic C, opacity)
};

// Where the absgrad backward adds its sums: out[2*id + {0,1}] += (o*0.5W*sum_p |g*(A*dx + B*dy)|, o*0.5H*sum_p |g*(B*dx + C*dy)|).
struct BlendAbsOut {
    float* out;    // [P,2]
    float sx, sy;  // 0.5*W, 0.5*H: the reference's ddelx_dx, ddely_dy
};

// Deterministic mode: instead of float atomics, each consumer warp parks its 9 sums of every record it blended in this block of
// shared memory (per stage, warp and record), and the producer warp adds the 8 warps' sums in warp order once the stage is released.
struct BlendDetStage {
    float c[BL_STAGES][8][BL_CH * DET_ROW];
    uint32_t mask[BL_STAGES][8];   // bit j: the warp wrote record j of the stage's chunk (a culled record counts as zero)
};

// Where the deterministic regions of a library-path binning blob start (carve_binning with det = true).  Computed from the
// capacity the blob was sized for, which the backward reads from the geometry header on the device.
__host__ __device__ __forceinline__ size_t det_partial_offset(size_t Rn)
{
    return (Rn * 4 + 255) / 256 * 256 + (Rn * 48 + 255) / 256 * 256;
}
__host__ __device__ __forceinline__ size_t det_reached_offset(size_t Rn)
{
    return det_partial_offset(Rn) + (Rn * DET_ROW * 4 + 255) / 256 * 256;
}
__host__ __device__ __forceinline__ size_t det_ids_offset(size_t Rn)   // ids_unsorted, behind the bitmap
{
    return det_reached_offset(Rn) + ((Rn + 31) / 32 * 4 + 255) / 256 * 256;
}

// contract the buffered pairs of one warp and add them to the accumulator records (see the header comment).  DET: `acc` is the
// warp's slice of BlendDetStage::c for the current stage and bw.mid holds the record's slot in the chunk; plain stores, no atomics.
// DEPTH: a tenth sum, sum_l w[l] * dL/ddepth[l] = dL/d(depth value), goes to word 9 together with word 8 (one 8-byte reduction).
// ABS (blend_backward_absgrad_kernel): also the two absolute sums of the pair's per-pixel dL/dmean2D terms over the 16 source lanes of
// each half, from the parked g and each lane's offset d = mean2D - pixel; the lanes that add words 0-3 add them to abs.out with one
// 8-byte reduction.  `mco` is the warp's BlendBackWarpAbs::mco.
template <bool DET = false, bool DEPTH = false, bool ABS = false>
__device__ __forceinline__ void back_flush(const BlendBackWarp& bw, int nbuf, int lane, float ox, float oy, float* __restrict__ acc,
                                           const float4* mco = nullptr, BlendAbsOut abs = BlendAbsOut{})
{
    __syncwarp();
    const int p = lane & 15, h = lane >> 4;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, s0 = 0.f, mx = 0.f, my = 0.f, mxx = 0.f, mxy = 0.f, myy = 0.f;
    float cz = 0.f;
    const float* wr = &bw.w[p][16 * h];
    const float* gr = &bw.g[p][16 * h];
    const float4* dr = &bw.d[16 * h];
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const float w = wr[i], g = gr[i];
        const float4 d = dr[i];
        const float xl = (float)(i & 7), yl = (float)(i >> 3);  // offset of source lane 16h+i inside its half of the sub-tile
        c0 = fmaf(w, d.x, c0);
        c1 = fmaf(w, d.y, c1);
        c2 = fmaf(w, d.z, c2);
        if (DEPTH) cz = fmaf(w, d.w, cz);
        s0 += g;
        mx = fmaf(g, xl, mx);
        my = fmaf(g, yl, my);
        mxx = fmaf(g, xl * xl, mxx);
        mxy = fmaf(g, xl * yl, mxy);
        myy = fmaf(g, yl * yl, myy);
    }
    // moments about the half's origin (ox, oy + 2h)  ->  moments of d = mean2D - pixel
    const float X = bw.mgx[p] - ox, Y = bw.mgy[p] - (oy + 2.0f * (float)h);
    float s1x = fmaf(X, s0, -mx), s1y = fmaf(Y, s0, -my);
    float s2xx = fmaf(X, fmaf(X, s0, -2.0f * mx), mxx);
    float s2xy = fmaf(X, fmaf(Y, s0, -my), fmaf(-Y, mx, mxy));
    float s2yy = fmaf(Y, fmaf(Y, s0, -2.0f * my), myy);
    c0 += __shfl_xor_sync(FULL, c0, 16);
    c1 += __shfl_xor_sync(FULL, c1, 16);
    c2 += __shfl_xor_sync(FULL, c2, 16);
    s0 += __shfl_xor_sync(FULL, s0, 16);
    s1x += __shfl_xor_sync(FULL, s1x, 16);
    s1y += __shfl_xor_sync(FULL, s1y, 16);
    s2xx += __shfl_xor_sync(FULL, s2xx, 16);
    s2xy += __shfl_xor_sync(FULL, s2xy, 16);
    s2yy += __shfl_xor_sync(FULL, s2yy, 16);
    if (DEPTH) cz += __shfl_xor_sync(FULL, cz, 16);
    if (DET && p < nbuf) {
        float* row = acc + __float_as_uint(bw.mid[p]) * DET_ROW;
        if (h == 0) {
            row[0] = c0; row[1] = c1; row[2] = c2; row[3] = s0; row[4] = s1x;
        } else {
            row[5] = s1y; row[6] = s2xx; row[7] = s2xy; row[8] = s2yy;
        }
    } else if (p < nbuf) {
        // both halves hold all nine sums: lane p adds words 0-3 of the record, lane p + 16 words 4-7 and word 8.  Records are 48 bytes
        // and grad_acc is 256-byte aligned (a 256-byte offset in carve_geometry of a blob lgr_alloc_fn returns 256-byte aligned), so rec
        // and rec + 4 are 16-byte aligned.
        float* rec = acc + (size_t)__float_as_uint(bw.mid[p]) * ACC_STRIDE;
        if (h == 0) {
            red_add_v4(rec, c0, c1, c2, s0);
        } else if (DEPTH) {
            red_add_v4(rec + 4, s1x, s1y, s2xx, s2xy);
            red_add_v2(rec + 8, s2yy, cz);
        } else {
            red_add_v4(rec + 4, s1x, s1y, s2xx, s2xy);
            atomicAdd(rec + 8, s2yy);
        }
    }
    if (ABS) {
        // a second pass over the parked g once the nine sums are issued, so that the two absolute sums never share registers with them.
        // Source lane 16h + 8r + c sits at d = (X - c, Y - r): A*dx + B*dy = u0 - A*c and B*dx + C*dy = v0 - B*c, (u0, v0) at c = 0.
        // One row of 8 lanes per iteration keeps c an immediate without holding all 16 parked g in registers.
        const float4 co = mco[p];
        float ax = 0.f, ay = 0.f;
#pragma unroll 1
        for (int r = 0; r < 2; r++) {
            const float ey = Y - (float)r;
            const float u0 = fmaf(co.x, X, co.y * ey), v0 = fmaf(co.y, X, co.z * ey);
#pragma unroll
            for (int c = 0; c < 8; c++) {
                const float g = gr[8 * r + c];
                ax += fabsf(g * fmaf(-co.x, (float)c, u0));
                ay += fabsf(g * fmaf(-co.y, (float)c, v0));
            }
        }
        ax += __shfl_xor_sync(FULL, ax, 16);
        ay += __shfl_xor_sync(FULL, ay, 16);
        if (p < nbuf && h == 0)
            red_add_v2(abs.out + 2 * (size_t)__float_as_uint(bw.mid[p]), co.w * abs.sx * ax, co.w * abs.sy * ay);
    }
    __syncwarp();
}

// back_flush for either warp buffer: only the absgrad kernel's has the conic / opacity rows
template <bool DET, bool DEPTH, bool ABS, class Warp>
__device__ __forceinline__ void back_flush_any(const Warp& bw, int nbuf, int lane, float ox, float oy, float* __restrict__ acc, BlendAbsOut abs)
{
    if constexpr (ABS) back_flush<false, false, true>(bw, nbuf, lane, ox, oy, acc, bw.mco, abs);
    else back_flush<DET, DEPTH>(bw, nbuf, lane, ox, oy, acc);
}

constexpr size_t BL_DET_BYTES = (sizeof(BlendDetStage) + 127) / 128 * 128;

constexpr size_t blend_back_smem_bytes(bool zero_rows = false, bool det = false, bool abs = false)
{
    return (sizeof(BlendRing) + 127) / 128 * 128 + (8 * (abs ? sizeof(BlendBackWarpAbs) : sizeof(BlendBackWarp)) + 127) / 128 * 128 +
           (det ? BL_DET_BYTES : 0) + (zero_rows ? (size_t)KB_ZERO_BYTES : 0);
}

// The depth variant's per-pixel inputs (lgr_backward_raw_depth).  `tag` is the HDR_DEPTH value the forward must have left: when the
// header holds another, the records' word 11 is not this mode's depth value, and the kernel writes NaN into words 0-9 of all P
// accumulator records instead of reading them, so every gradient shows the mismatch.
struct BlendDepthBack {
    const float* dL_ddepth;   // [H,W] or NULL (zero)
    const float* dL_dalpha;   // [H,W] or NULL (zero)
    int tag;
    int P;
};

// DET = false: every (warp, Gaussian) sum goes into acc[id] with float atomics (acc cleared beforehand).
// DET = true (deterministic mode): the sums of the 8 warps are added in warp order per record and written as one partial row per
// instance, at the instance's unsorted index (record word 10), into the binning blob; det_gather_kernel then adds each Gaussian's rows
// in ascending unsorted-index order.  The bitmap behind the rows marks the instances that got a row.  No float atomics.
// DEPTH: the depth and alpha terms (DESIGN section 7): per pixel d.w = dL/ddepth, and D starts at T_final * (bg.dL/dpix - dL/dalpha);
// per pair cd gains value * dL/ddepth, and the flush adds the tenth sum to record word 9.
// ABS (blend_backward_absgrad_kernel only): also the absolute-gradient densification statistic (back_flush, DESIGN section 7) into
// abs.out, which the caller cleared.  Like DEPTH it reads header word HDR_DEPTH: a forward that ran the depth blend (db.tag = 0 differs)
// gets NaN accumulators and NaN absgrad rows.
template <bool DET, bool DEPTH, bool ABS>
__device__ __forceinline__ void
blend_backward_ring_body(const uint2* __restrict__ ranges, const char* __restrict__ binning_blob, const int* __restrict__ header, int W, int H,
                         int tiles_x, const float* __restrict__ bg, const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
                         const float* __restrict__ dL_dpix, float* __restrict__ acc, const KbackZeroArgs& zero, const BlendDepthBack& db,
                         BlendAbsOut abs)
{
    static_assert(!(DET && DEPTH), "deterministic mode has no depth variant");
    static_assert(!ABS || (!DET && !DEPTH), "the absgrad backward extends the default kernel only");
    using Warp = typename std::conditional<ABS, BlendBackWarpAbs, BlendBackWarp>::type;
    extern __shared__ __align__(128) unsigned char blend_dyn_smem[];
    BlendRing& ring = *reinterpret_cast<BlendRing*>(blend_dyn_smem);
    Warp* warps = reinterpret_cast<Warp*>(blend_dyn_smem + ((sizeof(BlendRing) + 127) / 128) * 128);
    unsigned char* behind_warps = reinterpret_cast<unsigned char*>(warps) + (8 * sizeof(Warp) + 127) / 128 * 128;
    BlendDetStage* det = reinterpret_cast<BlendDetStage*>(behind_warps);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    const uint2 range = ranges[tile];
    // zero.P > 0: this launch also clears the dense gradient rows K7+K8 will (sparsely) write -- a page of zeros behind the per-warp
    // buffers, one thread, a handful of bulk stores per tile; the HBM writes overlap the blend, which leaves DRAM ~97 % idle
    float* zero_page = reinterpret_cast<float*>(behind_warps + (DET ? BL_DET_BYTES : 0));
    const bool zero_rows = zero.P > 0;
    if (zero_rows) {
        for (int k = threadIdx.x; k < KB_ZERO_BYTES / 4; k += BL_THREADS) zero_page[k] = 0.f;
        fence_async_smem();
    }
    ring_init(ring, 8);
    if (zero_rows && threadIdx.x == 8 * 32) tile_zero_rows(zero, tile, gridDim.x, zero_page);

    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int sx0 = tx * LGR_TILE + (warp & 1) * 8, sy0 = ty * LGR_TILE + (warp >> 1) * 4;
    const int px = sx0 + (lane & 7), py = sy0 + (lane >> 3);
    const bool inside = warp < 8 && px < W && py < H;
    const size_t pix = (size_t)py * W + px;
    const size_t plane = (size_t)H * W;
    const uint32_t last = inside ? n_contrib[pix] : 0u;
    const uint32_t warp_max = __reduce_max_sync(FULL, last);
    if (lane == 0 && warp_max) atomicMax(&ring.tile_max, warp_max);
    __syncthreads();
    const uint32_t tile_max = ring.tile_max;
    // DEPTH: a forward that ran without depth or in another mode left no (or another) value in record word 11: the records are not read,
    // and NaN accumulators make the misuse show in every gradient (see BlendDepthBack)
    if ((DEPTH || ABS) && header[HDR_DEPTH] != db.tag) {
        const float nan = __int_as_float(0x7fc00000);
        for (int i = blockIdx.x * BL_THREADS + threadIdx.x; i < db.P; i += gridDim.x * BL_THREADS) {
            float4* rec = reinterpret_cast<float4*>(acc + (size_t)i * ACC_STRIDE);
            rec[0] = rec[1] = make_float4(nan, nan, nan, nan);
            rec[2] = make_float4(nan, nan, 0.f, 0.f);
            if (ABS) reinterpret_cast<float2*>(abs.out)[i] = make_float2(nan, nan);
        }
        if (zero_rows && threadIdx.x == 8 * 32) bulk_wait_all();   // the zero page must outlive the stores that read it
        return;
    }
    // DET: a forward that did not run in deterministic mode stored no permutation; nothing is read or written (det_gather_kernel then
    // writes NaN accumulators, so the misuse shows in every gradient instead of corrupting memory)
    if (tile_max == 0 || (DET && header[HDR_DET] != 1)) {
        if (zero_rows && threadIdx.x == 8 * 32) bulk_wait_all();   // the zero page must outlive the stores that read it
        return;
    }
    const uint32_t nchunks = (tile_max + BL_CH - 1) / BL_CH;

    if (DET && warp == 8) {
        // ===== producer, deterministic mode: lane 0 streams the records as below; before a stage is refilled (and for the last
        // BL_STAGES chunks after the loads), the whole warp adds the consumers' sums of the chunk it held, lane j for record j =====
        const size_t Rn = (size_t)max(header[HDR_CAPACITY], 1);
        const float* rec_in = reinterpret_cast<const float*>(binning_blob + (Rn * 4 + 255) / 256 * 256);
        float* partial = reinterpret_cast<float*>(const_cast<char*>(binning_blob) + det_partial_offset(Rn));
        uint32_t* reached = reinterpret_cast<uint32_t*>(const_cast<char*>(binning_blob) + det_reached_offset(Rn));
        for (uint32_t i = 0; i < nchunks + BL_STAGES; i++) {
            const int s = i % BL_STAGES;
            const uint32_t ph = (i / BL_STAGES) & 1u;
            if (i >= BL_STAGES) {
                mbar_wait_ring(&ring.empty[s], ph ^ 1u);   // all 8 warps released chunk i - BL_STAGES
                const uint32_t b = nchunks - 1 - (i - BL_STAGES);
                const uint32_t n = min((uint32_t)BL_CH, tile_max - b * BL_CH);
                if ((uint32_t)lane < n) {
                    const uint32_t u = __float_as_uint(ring.rec[s][lane * BL_REC + 10]);
                    float v[DET_ROW];
#pragma unroll
                    for (int k = 0; k < DET_ROW; k++) v[k] = 0.f;
#pragma unroll
                    for (int w = 0; w < 8; w++) {
                        if ((det->mask[s][w] >> lane) & 1u) {
                            const float* c = &det->c[s][w][lane * DET_ROW];
#pragma unroll
                            for (int k = 0; k < DET_ROW; k++) v[k] += c[k];
                        }
                    }
                    if (u < Rn) {
#pragma unroll
                        for (int k = 0; k < DET_ROW; k++) partial[(size_t)u * DET_ROW + k] = v[k];
                        atomicOr(&reached[u >> 5], 1u << (u & 31));
                    }
                }
                __syncwarp();
            }
            if (i >= nchunks) continue;
            if (lane == 0) {
                if (i < BL_STAGES) mbar_wait_ring(&ring.empty[s], ph ^ 1u);
                const uint32_t b = nchunks - 1 - i;
                const uint32_t n = min((uint32_t)BL_CH, tile_max - b * BL_CH);
                const uint32_t bytes = n * (uint32_t)(BL_REC * 4);
                mbar_expect_tx(&ring.full[s], bytes);
                bulk_g2s(&ring.rec[s][0], rec_in + ((size_t)range.x + (size_t)b * BL_CH) * BL_REC, bytes, &ring.full[s]);
            }
            __syncwarp();
        }
        if (zero_rows && lane == 0) bulk_wait_all();
        return;
    }
    if (warp == 8) {
        // ===== producer: one thread streams the records back to front with TMA bulk loads =====
        if (lane == 0) {
            // records = second region of the binning blob (carve_binning): right behind the 4-byte ids of the instances the blob
            // was sized for (header word HDR_CAPACITY, written on the device by the forward)
            const size_t Rn = (size_t)max(header[HDR_CAPACITY], 1);
            const float* rec_in = reinterpret_cast<const float*>(binning_blob + (Rn * 4 + 255) / 256 * 256);
            for (uint32_t i = 0; i < nchunks; i++) {
                const uint32_t b = nchunks - 1 - i;
                const int s = i % BL_STAGES;
                const uint32_t ph = (i / BL_STAGES) & 1u;
                mbar_wait_ring(&ring.empty[s], ph ^ 1u);
                const uint32_t n = min((uint32_t)BL_CH, tile_max - b * BL_CH);
                const uint32_t bytes = n * (uint32_t)(BL_REC * 4);
                mbar_expect_tx(&ring.full[s], bytes);
                bulk_g2s(&ring.rec[s][0], rec_in + ((size_t)range.x + (size_t)b * BL_CH) * BL_REC, bytes, &ring.full[s]);
            }
            if (zero_rows) bulk_wait_all();   // long done by now
        }
        return;
    }

    // ===== consumers =====
    Warp& bw = warps[warp];
    float pxf = (float)px, pyf = (float)py;
    const float rx0 = (float)sx0, rx1 = (float)min(sx0 + 7, W - 1), ry0 = (float)sy0, ry1 = (float)min(sy0 + 3, H - 1);
    const float T_final = inside ? final_T[pix] : 0.f;
    float T = T_final;
    float d0 = 0.f, d1 = 0.f, d2 = 0.f;
    if (inside) {
        d0 = dL_dpix[pix];
        d1 = dL_dpix[plane + pix];
        d2 = dL_dpix[2 * plane + pix];
    }
    float dz = 0.f, da = 0.f;   // DEPTH: this pixel's dL/ddepth and dL/dalpha
    if (DEPTH && inside) {
        if (db.dL_ddepth) dz = db.dL_ddepth[pix];
        if (db.dL_dalpha) da = db.dL_dalpha[pix];
    }
    bw.d[lane] = make_float4(d0, d1, d2, dz);
    // D = sum_c dL/dpix_c * (background + everything blended BEHIND the current Gaussian), in absolute (not T-normalised) units:
    // the reference's  T*(c - accum_rec).dpix - T_final/(1-alpha)*bg.dpix  (backward.cu:505-518) equals  T*(c.dpix) - D/(1-alpha),
    // and D grows by alpha*T*(c.dpix) per blended Gaussian -- one scalar recurrence instead of three colour recurrences.
    // DEPTH: alpha = 1 - prod(1 - alpha_i) has dA/dalpha_i = T_final/(1 - alpha_i), the form of the background term: -dL/dalpha joins it
    float D = DEPTH ? T_final * ((bg[0] * d0 + bg[1] * d1 + bg[2] * d2) - da) : T_final * (bg[0] * d0 + bg[1] * d1 + bg[2] * d2);
    int nbuf = 0;
    __syncwarp();

    for (uint32_t i = 0; i < nchunks; i++) {
        const uint32_t b = nchunks - 1 - i;
        const int s = i % BL_STAGES;
        const uint32_t ph = (i / BL_STAGES) & 1u;
        mbar_wait_ring(&ring.full[s], ph);
        uint32_t wrote = 0;   // DET: records of this chunk with a parked row
        float* parked = DET ? &det->c[s][warp][0] : acc;
        if (b * BL_CH < warp_max) {
            const float* stage = &ring.rec[s][0];
            const uint32_t n = min((uint32_t)BL_CH, tile_max - b * BL_CH);
            bool keep = false;
            if ((uint32_t)lane < n && b * BL_CH + (uint32_t)lane < warp_max) {
                const float4 q0 = *reinterpret_cast<const float4*>(stage + lane * BL_REC);
                const float4 q1 = *reinterpret_cast<const float4*>(stage + lane * BL_REC + 4);
                keep = !subtile_cull2(q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, rx0, rx1, ry0, ry1);
            }
            unsigned mask = __ballot_sync(FULL, keep);
            while (mask) {
                const int j = 31 - __clz(mask);  // back to front
                mask &= ~(1u << j);
                const float* r = stage + j * BL_REC;
                const float4 q0 = *reinterpret_cast<const float4*>(r);
                const float4 q1 = *reinterpret_cast<const float4*>(r + 4);
                const float2 q2 = *reinterpret_cast<const float2*>(r + 8);
                const float dx = q0.x - pxf, dy = q0.y - pyf;
                const float power = fmaf(-0.5f, fmaf(q0.z * dx, dx, q1.x * dy * dy), -q0.w * dx * dy);
                float G;
                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(G) : "f"(power * 1.4426950408889634f));
                float alpha = fminf(0.99f, q1.y * G);
                const bool on = (b * BL_CH + (uint32_t)j < last) && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
                if (!__any_sync(FULL, on)) continue;
                // a lane that does not blend this Gaussian takes part as alpha = 0: T, D and both sums are unchanged
                G = on ? G : 0.f;
                alpha = on ? alpha : 0.f;
                const float one_m_a = 1.0f - alpha;   // in [0.01, 1]: MUFU.RCP + one Newton step is within 1 ulp
                float rcp;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rcp) : "f"(one_m_a));
                rcp = fmaf(rcp, fmaf(-one_m_a, rcp, 1.0f), rcp);
                T = T * rcp;
                float cd = fmaf(q1.z, d0, fmaf(q1.w, d1, q2.x * d2));
                if (DEPTH) cd = fmaf(r[11], dz, cd);
                const float dL_dalpha = fmaf(T, cd, -rcp * D);
                const float w = alpha * T;
                D = fmaf(w, cd, D);
                bw.w[nbuf][lane] = w;
                bw.g[nbuf][lane] = G * dL_dalpha;
                if (lane == 0) {
                    bw.mid[nbuf] = DET ? __uint_as_float((uint32_t)j) : q2.y;
                    bw.mgx[nbuf] = q0.x;
                    bw.mgy[nbuf] = q0.y;
                    if constexpr (ABS) bw.mco[nbuf] = make_float4(q0.z, q0.w, q1.x, q1.y);
                }
                if (DET) wrote |= 1u << j;
                if (++nbuf == BL_FLUSH) {
                    back_flush_any<DET, DEPTH, ABS>(bw, nbuf, lane, rx0, ry0, parked, abs);
                    nbuf = 0;
                }
            }
        }
        if (DET) {   // every row of this chunk is parked before the stage is released
            if (nbuf) back_flush<DET>(bw, nbuf, lane, rx0, ry0, parked);
            nbuf = 0;
            if (lane == 0) det->mask[s][warp] = wrote;
            __threadfence_block();
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&ring.empty[s]);
    }
    if (!DET && nbuf) back_flush_any<false, DEPTH, ABS>(bw, nbuf, lane, rx0, ry0, acc, abs);
}

template <bool DET = false, bool DEPTH = false>
__global__ void __launch_bounds__(BL_THREADS)
blend_backward_ring_kernel(const uint2* __restrict__ ranges, const char* __restrict__ binning_blob, const int* __restrict__ header, int W, int H,
                           int tiles_x, const float* __restrict__ bg, const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
                           const float* __restrict__ dL_dpix, float* __restrict__ acc, KbackZeroArgs zero, BlendDepthBack db = BlendDepthBack{})
{
    blend_backward_ring_body<DET, DEPTH, false>(ranges, binning_blob, header, W, H, tiles_x, bg, final_T, n_contrib, dL_dpix, acc, zero, db,
                                                BlendAbsOut{});
}

// The default kernel plus the absolute-gradient densification statistic (lgr_backward_raw_absgrad): absgrad[P,2] (cleared by the
// caller) gains, per (warp, Gaussian), o*(0.5W, 0.5H) times the sums over the warp's pixels of |g*(A*dx + B*dy)| and |g*(B*dx + C*dy)|.
// Four blocks per SM like the default kernel: 56 registers or fewer.
__global__ void __launch_bounds__(BL_THREADS, 4)
blend_backward_absgrad_kernel(const uint2* __restrict__ ranges, const char* __restrict__ binning_blob, const int* __restrict__ header, int W, int H,
                              int tiles_x, const float* __restrict__ bg, const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
                              const float* __restrict__ dL_dpix, float* __restrict__ acc, KbackZeroArgs zero, float* __restrict__ absgrad, int P)
{
    const BlendDepthBack db = {nullptr, nullptr, 0, P};   // tag 0: the forward must not have run the depth blend
    blend_backward_ring_body<false, false, true>(ranges, binning_blob, header, W, H, tiles_x, bg, final_T, n_contrib, dL_dpix, acc, zero, db,
                                                 BlendAbsOut{absgrad, 0.5f * (float)W, 0.5f * (float)H});
}

// ---- deterministic mode, across tiles: the Gaussian of depth rank k owns the unsorted instances [offsets[k-1], offsets[k]) (emit
// order: row-major tiles of its rectangle).  Thread t adds the partial rows of rank t's instances in ascending unsorted-index order and
// writes that Gaussian's whole accumulator record, and writes a zero record for Gaussian t if it has no instance.  Replaces the memset +
// atomics.  Reads only what the forward left (tiles_kept, offsets, the blob's ids_unsorted), not sorted_ids, which K7+K8 reuses.
__global__ void __launch_bounds__(256)
det_gather_kernel(int P, const uint32_t* __restrict__ tiles_kept, const unsigned long long* __restrict__ offsets,
                  const char* __restrict__ binning_blob, const int* __restrict__ header, float* __restrict__ acc)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P) return;
    if (header[HDR_DET] != 1) {   // the forward did not run in deterministic mode: refuse with NaN rather than read foreign data
        float4* rec = reinterpret_cast<float4*>(acc + (size_t)t * ACC_STRIDE);
        rec[0] = rec[1] = rec[2] = make_float4(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000), 0.f);
        return;
    }
    if (tiles_kept[t] == 0) {
        float4* rec = reinterpret_cast<float4*>(acc + (size_t)t * ACC_STRIDE);
        rec[0] = rec[1] = rec[2] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const uint32_t end = (uint32_t)offsets[t], begin = t ? (uint32_t)offsets[t - 1] : 0u;
    if (end == begin) return;
    const size_t Rn = (size_t)max(header[HDR_CAPACITY], 1);
    const float* partial = reinterpret_cast<const float*>(binning_blob + det_partial_offset(Rn));
    const uint32_t* reached = reinterpret_cast<const uint32_t*>(binning_blob + det_reached_offset(Rn));
    const uint32_t* ids_unsorted = reinterpret_cast<const uint32_t*>(binning_blob + det_ids_offset(Rn));
    float v[DET_ROW];
#pragma unroll
    for (int q = 0; q < DET_ROW; q++) v[q] = 0.f;
    for (uint32_t u = begin; u < end; u++) {
        if (!((reached[u >> 5] >> (u & 31)) & 1u)) continue;   // never walked by the backward: contributes exactly zero
        const float* r = partial + (size_t)u * DET_ROW;
#pragma unroll
        for (int q = 0; q < DET_ROW; q++) v[q] += r[q];
    }
    float4* rec = reinterpret_cast<float4*>(acc + (size_t)ids_unsorted[begin] * ACC_STRIDE);
    rec[0] = make_float4(v[0], v[1], v[2], v[3]);
    rec[1] = make_float4(v[4], v[5], v[6], v[7]);
    rec[2] = make_float4(v[8], 0.f, 0.f, 0.f);
}

}  // namespace
