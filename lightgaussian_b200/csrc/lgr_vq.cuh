// lgr_vq.cuh -- VecTree vector quantisation of the SH features (SURVEY.md section 8f, row N4):
// the importance-weighted EMA k-means of vectree/vq.py:262-306 (EuclideanCodebook.forward) as driven by vectree/vectree.py:166-207,
// and the bit-packing codec of vectree/vectree.py:119-125 / vectree/utils.py:33-39,106-112.
//
// The reference evaluates one k-means iteration (n = 80 000 samples, K = 8192 codes, d = 27 or 48) as torch.cdist (a [n,K] fp32
// matrix, 2.6 GB), argmax, F.one_hot (another 2.6 GB), a broadcast multiply by the weights (2.6 GB more) and an einsum of the
// one-hot matrix with the features (a dense 35 GFLOP GEMM that is all zeros but one entry per row).  Here:
//   vq_assign_kernel      nearest code per sample, score_c = |e_c|^2 - 2 x.e_c (the |x|^2 term of cdist's own expansion is constant
//                         per row), FP32 FFMA with the code tile in shared memory and two sample rows in registers per thread; the
//                         codebook is split over blockIdx.y and the partial winners merged with ONE 64-bit atomicMin per row on
//                         (order-preserving score bits << 32 | code): the smallest code wins ties, as the first-index argmax does.
//                         No [n,K] matrix ever exists: n*d*4 + K*d*4 bytes in, n*8 out.
//   vq_accumulate_kernel  cluster_size_batch[c] += w_i, embed_sum[c,:] += w_i x_i for the winner c of row i (n*(d+1) float atomics
//                         into a K*(d+1) table that lives in L2) -- instead of the one-hot GEMM.
//   vq_ema_kernel(s)      cluster_size <- 0.8 cluster_size + 0.2 batch;  smoothed = (cs + eps) / (sum cs + K eps) * sum cs;
//                         embed <- 0.8 embed + 0.2 embed_sum / smoothed     (vq.py:40-44,286-300; note: the reference updates
//                         `embed` directly, `embed_avg` is never touched again)
//   vq_gather_kernel      quantize[i,:] = embed[idx_i,:]
//   pack / unpack         code indices <-> big-endian bit stream of log2(K) bits per index (dec2bin + np.packbits, MSB first)
#pragma once

#include <cstdint>

namespace {

constexpr int VQ_TC = 64;        // codes per shared-memory tile
constexpr int VQ_THREADS = 128;  // threads per block, RX sample rows each

__device__ __forceinline__ unsigned vq_order_bits(float f)
{
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__global__ void vq_init_best_kernel(int n, unsigned long long* __restrict__ best)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) best[i] = ~0ull;
}

// DP = d padded to a multiple of 4 (28 for d = 27, 48 for d = 48, ...); RX = sample rows held in registers per thread
template <int DP, int RX>
__global__ void __launch_bounds__(VQ_THREADS)
vq_assign_kernel(int n, int d, int K, const float* __restrict__ x, const float* __restrict__ embed, int codes_per_split,
                 unsigned long long* __restrict__ best)
{
    __shared__ __align__(16) float s_e[VQ_TC][DP];
    __shared__ float s_n[VQ_TC];
    const int row0 = blockIdx.x * (RX * VQ_THREADS) + threadIdx.x;
    float xr[RX][DP];
#pragma unroll
    for (int r = 0; r < RX; r++) {
        const int row = row0 + r * VQ_THREADS;
#pragma unroll
        for (int j = 0; j < DP; j++) xr[r][j] = (j < d && row < n) ? -2.0f * x[(size_t)row * d + j] : 0.f;
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
    for (int r = 0; r < RX; r++) {
        const int row = row0 + r * VQ_THREADS;
        if (row < n) atomicMin(&best[row], ((unsigned long long)vq_order_bits(bestv[r]) << 32) | (unsigned)arg[r]);
    }
}

template <int DP>
void vq_launch_assign(int n, int d, int K, const float* x, const float* embed, unsigned long long* best, cudaStream_t stream)
{
    constexpr int RX = DP <= 32 ? 4 : 2;                           // 4 rows x 28 values still fit the register file without spills
    const int rows = RX * VQ_THREADS;
    const int row_tiles = (n + rows - 1) / rows;
    const int code_tiles = (K + VQ_TC - 1) / VQ_TC;
    int splits = (4 * 132 * 3 + row_tiles - 1) / row_tiles;        // aim at >= 4 waves of 132 SMs x 3 resident blocks
    splits = max(1, min(splits, code_tiles));
    const int tiles_per_split = (code_tiles + splits - 1) / splits;
    const int codes_per_split = tiles_per_split * VQ_TC;
    splits = (K + codes_per_split - 1) / codes_per_split;
    vq_assign_kernel<DP, RX><<<dim3(row_tiles, splits), VQ_THREADS, 0, stream>>>(n, d, K, x, embed, codes_per_split, best);
}

// idx[i] = low word of best[i]; optional weighted accumulation for the EMA step.  weight == nullptr: unit weights; otherwise the
// reference's normalisation  w_i * numel / sum(w)  (vq.py:263-264), rounded in that order
__global__ void __launch_bounds__(256)
vq_accumulate_kernel(int n, int d, const unsigned long long* __restrict__ best, const float* __restrict__ x, const float* __restrict__ weight,
                     float weight_numel, const float* __restrict__ weight_sum, int* __restrict__ idx_out, float* __restrict__ cluster_batch,
                     float* __restrict__ embed_sum)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)n * (d + 1);
    if (t >= total) return;
    const int i = (int)(t / (d + 1)), j = (int)(t - (long long)i * (d + 1));
    const int c = (int)(unsigned)best[i];
    const float w = weight ? __fdiv_rn(__fmul_rn(weight[i], weight_numel), weight_sum[0]) : 1.0f;
    if (j == d) {
        if (idx_out) idx_out[i] = c;
        if (cluster_batch) atomicAdd(&cluster_batch[c], w);
    } else if (embed_sum) {
        atomicAdd(&embed_sum[(size_t)c * d + j], __fmul_rn(x[(size_t)i * d + j], w));
    }
}

// ---- deterministic mode: the same sums without float atomics.  A stable radix sort of (code, sample) pairs groups the samples of each
// code in ascending sample order; one warp per code then adds them in that order. ----
__global__ void __launch_bounds__(256)
vq_det_keys_kernel(int n, const unsigned long long* __restrict__ best, int* __restrict__ idx_out, uint32_t* __restrict__ codes,
                   uint32_t* __restrict__ rows)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t c = (uint32_t)best[i];
    if (idx_out) idx_out[i] = (int)c;
    codes[i] = c;
    rows[i] = (uint32_t)i;
}

// block = code c: segment [lower(c), lower(c+1)) of the sorted codes.  Warp w adds the samples a+w, a+w+VQ_SEG_WARPS, ... in that order
// (lane l owns columns l, l+32, l+64 of [embed_sum row | batch], column d being cluster_batch); the warps' partial sums are then added
// in warp order.  The split depends only on the sorted order, so the result is deterministic, and a code that holds every sample is
// added by VQ_SEG_WARPS warps instead of one.  Every code's sums are written, zero for a code no sample chose.
constexpr int VQ_SEG_WARPS = 8;
__global__ void __launch_bounds__(VQ_SEG_WARPS * 32)
vq_det_segsum_kernel(int n, int d, int K, const uint32_t* __restrict__ codes, const uint32_t* __restrict__ rows, const float* __restrict__ x,
                     const float* __restrict__ weight, float weight_numel, const float* __restrict__ weight_sum, float* __restrict__ cluster_batch,
                     float* __restrict__ embed_sum)
{
    __shared__ float part[VQ_SEG_WARPS][96];
    __shared__ int seg[2];
    const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x < 2) {
        const uint32_t key = (uint32_t)c + (uint32_t)threadIdx.x;
        int lo = 0, hi = n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (codes[mid] < key) lo = mid + 1;
            else hi = mid;
        }
        seg[threadIdx.x] = lo;
    }
    __syncthreads();
    const int a = seg[0], b = seg[1];
    float acc[3] = {0.f, 0.f, 0.f};
    for (int k = a + warp; k < b; k += VQ_SEG_WARPS) {
        const int i = (int)rows[k];
        const float w = weight ? __fdiv_rn(__fmul_rn(weight[i], weight_numel), weight_sum[0]) : 1.0f;   // as vq_accumulate_kernel
#pragma unroll
        for (int q = 0; q < 3; q++) {
            const int j = lane + 32 * q;
            if (j < d) acc[q] = __fadd_rn(acc[q], __fmul_rn(x[(size_t)i * d + j], w));
            else if (j == d) acc[q] = __fadd_rn(acc[q], w);
        }
    }
#pragma unroll
    for (int q = 0; q < 3; q++) part[warp][lane + 32 * q] = acc[q];
    __syncthreads();
    for (int j = threadIdx.x; j <= d; j += blockDim.x) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < VQ_SEG_WARPS; w++) v = __fadd_rn(v, part[w][j]);
        if (j < d) {
            if (embed_sum) embed_sum[(size_t)c * d + j] = v;
        } else if (cluster_batch) {
            cluster_batch[c] = v;
        }
    }
}

// one block: cluster_size EMA and its total (fixed summation order -> deterministic given the batch sums)
__global__ void __launch_bounds__(1024)
vq_ema_cluster_kernel(int K, float decay, float one_minus_decay, float* __restrict__ cluster_size, const float* __restrict__ cluster_batch,
                      float* __restrict__ total_out)
{
    __shared__ double s_part[1024];
    double part = 0.0;
    for (int c = threadIdx.x; c < K; c += 1024) {
        const float v = fmaf(cluster_batch[c], one_minus_decay, __fmul_rn(cluster_size[c], decay));   // mul_(decay).add_(new, alpha=1-decay)
        cluster_size[c] = v;
        part += (double)v;
    }
    s_part[threadIdx.x] = part;
    __syncthreads();
    for (int s = 512; s > 0; s >>= 1) {
        if (threadIdx.x < s) s_part[threadIdx.x] += s_part[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) total_out[0] = (float)s_part[0];
}

__global__ void __launch_bounds__(256)
vq_ema_embed_kernel(int K, int d, float decay, float one_minus_decay, float eps, float k_eps, const float* __restrict__ cluster_size,
                    const float* __restrict__ total, const float* __restrict__ embed_sum, float* __restrict__ embed)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= K * d) return;
    const int c = t / d;
    const float tot = total[0];
    // laplace_smoothing(x, K, eps) * x.sum() = (x + eps) / (sum + K*eps) * sum            vq.py:43-44,298
    const float smoothed = __fmul_rn(__fdiv_rn(__fadd_rn(cluster_size[c], eps), __fadd_rn(tot, k_eps)), tot);
    const float target = __fdiv_rn(embed_sum[t], smoothed);
    embed[t] = fmaf(target, one_minus_decay, __fmul_rn(embed[t], decay));
}

__global__ void __launch_bounds__(256) vq_gather_kernel(int n, int d, const int* __restrict__ idx, const float* __restrict__ embed,
                                                        float* __restrict__ out)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * d) return;
    const int i = (int)(t / d), j = (int)(t - (long long)i * d);
    out[t] = embed[(size_t)idx[i] * d + j];
}

// byte b of the stream holds global bits 8b..8b+7, most significant first; global bit g belongs to index g / bits, and is bit
// (bits-1 - g % bits) of it (dec2bin: mask = 2^(bits-1) ... 2^0; np.packbits bitorder 'big'), zero padded at the end
__global__ void __launch_bounds__(256) vq_pack_kernel(long long n, int bits, const int* __restrict__ idx, uint8_t* __restrict__ out,
                                                      long long n_bytes)
{
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_bytes) return;
    unsigned byte = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const long long g = b * 8 + k;
        const long long e = g / bits;
        const int pos = (int)(g - e * bits);
        const unsigned bit = (e < n) ? ((unsigned)idx[e] >> (bits - 1 - pos)) & 1u : 0u;
        byte |= bit << (7 - k);
    }
    out[b] = (uint8_t)byte;
}

__global__ void __launch_bounds__(256) vq_unpack_kernel(long long n, int bits, const uint8_t* __restrict__ in, int* __restrict__ idx)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    unsigned v = 0;
    const long long g0 = e * bits;
    for (int pos = 0; pos < bits; pos++) {
        const long long g = g0 + pos;
        const unsigned bit = (in[g >> 3] >> (7 - (int)(g & 7))) & 1u;
        v = (v << 1) | bit;
    }
    idx[e] = (int)v;
}

}  // namespace
