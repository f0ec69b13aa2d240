// lgr_vq_tc.cuh -- nearest-code search of the VecTree k-means (vectree/vq.py:262-306: cdist + argmax) on the Hopper tensor cores (wgmma).
//
// score[i][c] = |e_c|^2 - 2 x_i . e_c is a GEMM with a 27-long contraction (n = 80 000 samples x K = 8192 codes).  bf16 operands alone
// would flip nearest-code decisions, and the parity contract is on the INDICES, so the kernel does a coarse pass on the tensor cores and an
// exact FP32 rescore of the rows it cannot decide:
//
//   operands   x = x_hi + x_lo, e = e_hi + e_lo (two bf16 terms each, 16 bits of mantissa); the contraction is laid out as
//              A' = [x_hi | x_hi | x_lo] (96 columns), B' = [e_hi | e_lo | e_hi], so ONE bf16 GEMM with K = 96 yields
//              x_hi.e_hi + x_hi.e_lo + x_lo.e_hi with FP32 accumulation; the dropped terms are bounded by 3 * 2^-18 |x||e|.
//   kernel     one CTA = 128 samples against all codes in tiles of 256, operands in shared memory as canonical K-major core-matrix
//              tiles (no swizzle) that a prepare kernel wrote to global memory in exactly that order, so a tile arrives with ONE
//              cp.async.bulk (producer warp 8, two stages).  Warpgroups 0 and 1 each own 64 of the samples and compute a tile as two
//              halves of 128 codes, six wgmma.m64n128k16 per half with the FP32 accumulators in registers; the epilogue of half 0 runs
//              while the tensor cores work on half 1.  Each thread holds two rows x 32 columns of a half, forms score = |e|^2 - 2 acc and
//              keeps (best, second best, argmin); the four lanes that share a row merge at the end.  Smallest index wins ties like the
//              first-index argmax.
//   decision   a row whose second-best score is within 2 * 1e-4 * |x_i| * max|e| of its best (>= 4x the error bound) is NOT decided here:
//              its slot keeps ~0 and the exact FP32 kernel (vq_assign_kernel, lgr_vq.cuh) runs on the list of such rows (a few per cent).
//              Every other row's argmin is provably the exact one.
#pragma once

namespace {

constexpr int VT_M = 128;          // samples per CTA
constexpr int VT_N = 256;          // codes per tile
constexpr int VT_DP = 32;          // padded feature dimension
constexpr int VT_K = 3 * VT_DP;    // contraction length of the split GEMM
constexpr int VT_A_BYTES = VT_M * VT_K * 2;
constexpr int VT_B_BYTES = VT_N * VT_K * 2;
constexpr int VT_HN = 128;         // codes per wgmma (half a tile)
constexpr int VT_THREADS = 288;    // warps 0-7 = two consumer warpgroups (64 samples each), warp 8 loads
constexpr float VT_MARGIN = 2.0e-4f;

__device__ __forceinline__ uint32_t vt_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// element (r, k) of a K-major operand tile with ROWS rows, canonical no-swizzle core-matrix order:
// 8 x 16-byte core matrices, 128 bytes each; matrices adjacent in M/N are 128 B apart (SBO), matrices adjacent in K are (ROWS/8)*128 B apart (LBO)
__host__ __device__ inline size_t vt_tile_offset(int rows, int r, int k) { return ((size_t)(k >> 3) * (rows >> 3) + (r >> 3)) * 128 + (r & 7) * 16 + (k & 7) * 2; }

__device__ __forceinline__ unsigned short vt_bf16_rn(float f)
{
    const unsigned u = __float_as_uint(f);
    return (unsigned short)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);   // round to nearest even (finite inputs)
}
__device__ __forceinline__ float vt_bf16_f(unsigned short h) { return __uint_as_float((unsigned)h << 16); }

// rows of x -> A' tiles [n_pad/128][128 x 96] and |x_i|
__global__ void __launch_bounds__(256) vt_prep_x_kernel(int n, int n_pad, int d, const float* __restrict__ x, unsigned char* __restrict__ A, float* __restrict__ xnorm)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    unsigned char* tile = A + (size_t)(i / VT_M) * VT_A_BYTES;
    const int r = i % VT_M;
    float s = 0.f;
    for (int k = 0; k < VT_DP; k++) {
        const float v = (i < n && k < d) ? x[(size_t)i * d + k] : 0.f;
        s = fmaf(v, v, s);
        const unsigned short hi = vt_bf16_rn(v), lo = vt_bf16_rn(v - vt_bf16_f(hi));
        *reinterpret_cast<unsigned short*>(tile + vt_tile_offset(VT_M, r, k)) = hi;
        *reinterpret_cast<unsigned short*>(tile + vt_tile_offset(VT_M, r, VT_DP + k)) = hi;
        *reinterpret_cast<unsigned short*>(tile + vt_tile_offset(VT_M, r, 2 * VT_DP + k)) = lo;
    }
    xnorm[i] = sqrtf(s);
}

// codes -> B' tiles [K_pad/256][256 x 96], |e_c|^2 (+huge for padding) and max |e_c| (bits of a non-negative float order like integers)
__global__ void __launch_bounds__(256) vt_prep_e_kernel(int K, int K_pad, int d, const float* __restrict__ e, unsigned char* __restrict__ B, float* __restrict__ norms,
                                                        unsigned* __restrict__ emax_bits)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= K_pad) return;
    unsigned char* tile = B + (size_t)(c / VT_N) * VT_B_BYTES;
    const int r = c % VT_N;
    float s = 0.f;
    for (int k = 0; k < VT_DP; k++) {
        const float v = (c < K && k < d) ? e[(size_t)c * d + k] : 0.f;
        s = fmaf(v, v, s);
        const unsigned short hi = vt_bf16_rn(v), lo = vt_bf16_rn(v - vt_bf16_f(hi));
        *reinterpret_cast<unsigned short*>(tile + vt_tile_offset(VT_N, r, k)) = hi;
        *reinterpret_cast<unsigned short*>(tile + vt_tile_offset(VT_N, r, VT_DP + k)) = lo;
        *reinterpret_cast<unsigned short*>(tile + vt_tile_offset(VT_N, r, 2 * VT_DP + k)) = hi;
    }
    norms[c] = c < K ? s : 3.0e38f;
    if (c < K) atomicMax(emax_bits, __float_as_uint(sqrtf(s)));
}

// ---- mbarrier / bulk-copy / wgmma wrappers ----
__device__ __forceinline__ void vt_mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(vt_smem(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void vt_mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(vt_smem(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void vt_mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(vt_smem(bar)) : "memory"); }
__device__ __forceinline__ void vt_mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok = 0;
    for (uint32_t spin = 0; !ok; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(vt_smem(bar)), "r"(parity)
                     : "memory");
        // a protocol bug becomes a launch error, not a hung GPU (no printf here: a call inside the consumer loop would make ptxas
        // serialise the wgmma pipeline)
        if (!ok && spin > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ void vt_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(vt_smem(dst)), "l"(src), "r"(bytes),
                 "r"(vt_smem(bar))
                 : "memory");
}
__device__ __forceinline__ uint64_t vt_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    // wgmma shared-memory matrix descriptor: start address [0,14), leading byte offset [16,30) (core matrices adjacent in K), stride byte
    // offset [32,46) (core matrices adjacent in M/N) -- all without their 4 LSBs --, base offset 0, layout type 0 = no swizzle at [62,64)
    return (uint64_t)((smem_addr >> 4) & 0x3fffu) | ((uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32);
}
__device__ __forceinline__ void vt_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void vt_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void vt_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x 128] (+)= A[64 x 16] B[128 x 16]^T, bf16 operands (both K-major) from shared memory, FP32 accumulators in registers
__device__ __forceinline__ void vt_wgmma(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, "
        "%29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, "
        "%57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
          "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
          "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate)
        : "memory");
}

// (best, second best, argmin) of the columns a thread holds for one row.  Accumulator element i of an m64nNk16 wgmma sits in row
// 16 * (warp % 4) + lane / 4 + 8 * ((i >> 1) & 1) and column 8 * (i >> 2) + 2 * (lane & 3) + (i & 1) of the warpgroup's 64 x N block.
struct VtBest {
    float best = 3.0e38f, second = 3.0e38f;
    int arg = 0;
    __device__ __forceinline__ void add(float sc, int c)   // columns arrive in increasing order: strict < keeps the smallest index
    {
        if (sc < best) { second = best; best = sc; arg = c; }
        else if (sc < second) second = sc;
    }
    __device__ __forceinline__ void merge(float ob, float os, int oa)
    {
        if (ob < best || (ob == best && oa < arg)) { second = fminf(best, os); best = ob; arg = oa; }
        else second = fminf(second, ob);
    }
};

__device__ __forceinline__ void vt_epilogue(const float (&d)[64], const float* nrm, int cbase, int lane, VtBest& r0, VtBest& r1)
{
#pragma unroll
    for (int i = 0; i < 64; i++) {
        const int c = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        const float sc = fmaf(-2.0f, d[i], nrm[c]);
        if ((i >> 1) & 1) r1.add(sc, cbase + c);
        else r0.add(sc, cbase + c);
    }
}

struct VtSmem {
    unsigned char a[VT_A_BYTES];         // 24 576 B
    unsigned char b[2][VT_B_BYTES];      // 2 x 49 152 B
    float norm[2][VT_N];
    uint64_t full_a, full_b[2], stage_free[2];
};

__global__ void __launch_bounds__(VT_THREADS, 1)
vt_assign_kernel(int n, int K_pad, const unsigned char* __restrict__ A, const unsigned char* __restrict__ B, const float* __restrict__ norms,
                 const float* __restrict__ xnorm, const unsigned* __restrict__ emax_bits, unsigned long long* __restrict__ best, int* __restrict__ undecided,
                 int* __restrict__ n_undecided)
{
    extern __shared__ __align__(1024) unsigned char vt_dyn[];
    VtSmem& sm = *reinterpret_cast<VtSmem*>(vt_dyn);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ntiles = K_pad / VT_N;

    if (threadIdx.x == 0) {
        vt_mbar_init(&sm.full_a, 1);
        for (int s = 0; s < 2; s++) {
            vt_mbar_init(&sm.full_b[s], 1);
            vt_mbar_init(&sm.stage_free[s], 8);   // lane 0 of each consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ===== loads: the CTA's sample tile once, then the code tiles through two stages =====
        if (lane == 0) {
            vt_mbar_expect_tx(&sm.full_a, VT_A_BYTES);
            vt_bulk_g2s(sm.a, A + (size_t)blockIdx.x * VT_A_BYTES, VT_A_BYTES, &sm.full_a);
            for (int t = 0; t < ntiles; t++) {
                const int s = t & 1;
                const uint32_t ph = (uint32_t)(t >> 1) & 1u;
                vt_mbar_wait(&sm.stage_free[s], ph ^ 1u);   // passes at once the first time round
                vt_mbar_expect_tx(&sm.full_b[s], VT_B_BYTES + VT_N * 4);
                vt_bulk_g2s(sm.b[s], B + (size_t)t * VT_B_BYTES, VT_B_BYTES, &sm.full_b[s]);
                vt_bulk_g2s(sm.norm[s], norms + (size_t)t * VT_N, VT_N * 4, &sm.full_b[s]);
            }
        }
        return;
    }

    // ===== consumers: warpgroup g owns samples 64 g .. 64 g + 63 of the CTA's tile =====
    const int g = warp >> 2;
    const uint32_t a_addr = vt_smem(sm.a) + (uint32_t)g * (64 / 8) * 128u;
    VtBest r0, r1;
    float acc[2][64];
    vt_mbar_wait(&sm.full_a, 0);
    for (int t = 0; t < ntiles; t++) {
        const int s = t & 1;
        const uint32_t ph = (uint32_t)(t >> 1) & 1u;
        vt_mbar_wait(&sm.full_b[s], ph);
        const uint32_t b_addr = vt_smem(sm.b[s]);
        vt_wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int k = 0; k < VT_K / 16; k++) {
                const uint64_t da = vt_desc(a_addr + (uint32_t)k * 2u * (VT_M / 8) * 128u, (VT_M / 8) * 128u, 128u);
                const uint64_t db = vt_desc(b_addr + (uint32_t)h * (VT_HN / 8) * 128u + (uint32_t)k * 2u * (VT_N / 8) * 128u, (VT_N / 8) * 128u, 128u);
                vt_wgmma(acc[h], da, db, k > 0 ? 1u : 0u);
            }
            vt_wgmma_commit();
        }
        vt_wgmma_wait<1>();   // half 0 is complete; half 1 still runs on the tensor cores
        vt_epilogue(acc[0], sm.norm[s], t * VT_N, lane, r0, r1);
        vt_wgmma_wait<0>();
        vt_epilogue(acc[1], sm.norm[s] + VT_HN, t * VT_N + VT_HN, lane, r0, r1);
        __syncwarp();
        if (lane == 0) vt_mbar_arrive(&sm.stage_free[s]);   // this warp no longer reads stage s
    }
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {   // the four lanes of a quad hold the same two rows
        r0.merge(__shfl_xor_sync(0xffffffffu, r0.best, m), __shfl_xor_sync(0xffffffffu, r0.second, m), __shfl_xor_sync(0xffffffffu, r0.arg, m));
        r1.merge(__shfl_xor_sync(0xffffffffu, r1.best, m), __shfl_xor_sync(0xffffffffu, r1.second, m), __shfl_xor_sync(0xffffffffu, r1.arg, m));
    }
    if ((lane & 3) < 2) {
        const VtBest& r = (lane & 3) ? r1 : r0;
        const int row = blockIdx.x * VT_M + 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * (lane & 3);
        if (row < n) {
            const float margin = 2.0f * VT_MARGIN * xnorm[row] * __uint_as_float(*emax_bits);
            if (r.second - r.best > margin) {
                best[row] = ((unsigned long long)vq_order_bits(r.best) << 32) | (unsigned)r.arg;
            } else {
                best[row] = ~0ull;   // undecided here: the exact FP32 kernel fills it
                undecided[atomicAdd(n_undecided, 1)] = row;
            }
        }
    }
}

// the exact FP32 kernel of lgr_vq.cuh on a LIST of rows (the ones the tensor-core pass left undecided)
template <int DP, int RX>
__global__ void __launch_bounds__(VQ_THREADS)
vq_assign_rows_kernel(const int* __restrict__ rows, const int* __restrict__ n_rows, int d, int K, const float* __restrict__ x, const float* __restrict__ embed,
                      int codes_per_split, unsigned long long* __restrict__ best)
{
    __shared__ __align__(16) float s_e[VQ_TC][DP];
    __shared__ float s_n[VQ_TC];
    const int n = *n_rows;
    if ((int)blockIdx.x * (RX * VQ_THREADS) >= n) return;
    const int slot0 = blockIdx.x * (RX * VQ_THREADS) + threadIdx.x;
    float xr[RX][DP];
    int rowid[RX];
#pragma unroll
    for (int r = 0; r < RX; r++) {
        const int slot = slot0 + r * VQ_THREADS;
        rowid[r] = slot < n ? rows[slot] : -1;
#pragma unroll
        for (int j = 0; j < DP; j++) xr[r][j] = (j < d && rowid[r] >= 0) ? -2.0f * x[(size_t)rowid[r] * d + j] : 0.f;
    }
    const int c_begin = blockIdx.y * codes_per_split, c_end = min(K, c_begin + codes_per_split);
    float bestv[RX];
    int arg[RX];
#pragma unroll
    for (int r = 0; r < RX; r++) { bestv[r] = 3.0e38f; arg[r] = c_begin; }
    for (int c0 = c_begin; c0 < c_end; c0 += VQ_TC) {
        __syncthreads();
        for (int t = threadIdx.x; t < VQ_TC * DP; t += VQ_THREADS) {
            const int c = t / DP, j = t - c * DP;
            s_e[c][j] = (j < d && c0 + c < c_end) ? embed[(size_t)(c0 + c) * d + j] : 0.f;
        }
        __syncthreads();
        if (threadIdx.x < VQ_TC) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < DP; j++) s = fmaf(s_e[threadIdx.x][j], s_e[threadIdx.x][j], s);
            s_n[threadIdx.x] = (c0 + threadIdx.x < c_end) ? s : 3.0e38f;
        }
        __syncthreads();
#pragma unroll 2
        for (int c = 0; c < VQ_TC; c++) {
            float dist[RX];
            const float nrm = s_n[c];
#pragma unroll
            for (int r = 0; r < RX; r++) dist[r] = nrm;
            const float4* e4 = reinterpret_cast<const float4*>(s_e[c]);
#pragma unroll
            for (int q = 0; q < DP / 4; q++) {
                const float4 e = e4[q];
#pragma unroll
                for (int r = 0; r < RX; r++) {
                    dist[r] = fmaf(xr[r][4 * q + 0], e.x, dist[r]);
                    dist[r] = fmaf(xr[r][4 * q + 1], e.y, dist[r]);
                    dist[r] = fmaf(xr[r][4 * q + 2], e.z, dist[r]);
                    dist[r] = fmaf(xr[r][4 * q + 3], e.w, dist[r]);
                }
            }
#pragma unroll
            for (int r = 0; r < RX; r++)
                if (dist[r] < bestv[r]) { bestv[r] = dist[r]; arg[r] = c0 + c; }
        }
    }
#pragma unroll
    for (int r = 0; r < RX; r++)
        if (rowid[r] >= 0) atomicMin(&best[rowid[r]], ((unsigned long long)vq_order_bits(bestv[r]) << 32) | (unsigned)arg[r]);
}

struct VtScratch {   // grow-only device scratch of the tensor-core path (operand tiles, norms, undecided list)
    void* p = nullptr;
    size_t bytes = 0;
    int device = -1;
};
inline size_t vt_align(size_t v) { return (v + 1023) / 1024 * 1024; }

}  // namespace
