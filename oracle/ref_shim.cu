// ref_shim.cu -- TEST/BASELINE INFRASTRUCTURE ONLY.
//
// A plain C-ABI around the reference's own, unmodified CudaRasterizer::Rasterizer static API
// (declared in RAST/cuda_rasterizer/rasterizer.h:20-113).  oracle/Makefile compiles the
// reference's forward.cu / backward.cu / rasterizer_impl.cu from the reference checkout together with
// this file into oracle/_ref/libref_rasterizer.so.  It exists so that
//   * tests can compare our kernels with the real reference kernels on the same GPU, and
//   * bench.py --impl reference can time the reference's CUDA path next to ours,
// without torch/pybind in between (the reference's torch binding, RAST/rasterize_points.cu,
// only allocates tensors and forwards raw pointers to this same API).
//
// All pointers are device pointers.  The three state blobs the reference sub-allocates from
// (geometry / binning / image) are kept in a grow-only RefState owned by the caller.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include "cuda_rasterizer/rasterizer.h"
#include "cuda_rasterizer/rasterizer_impl.h"

namespace {
struct Blob {
    char* ptr = nullptr;
    size_t cap = 0;
    char* ensure(size_t n)
    {
        if (n > cap) {
            if (ptr) cudaFree(ptr);
            size_t want = n + n / 4 + 256;
            if (cudaMalloc(&ptr, want) != cudaSuccess) { fprintf(stderr, "ref_shim: cudaMalloc(%zu) failed\n", want); abort(); }
            cap = want;
        }
        return ptr;
    }
    ~Blob() { if (ptr) cudaFree(ptr); }
};
struct RefState {
    Blob geom, binning, img;
    int num_rendered = 0;
    int P = 0;
};
}  // namespace

extern "C" {

void* ref_state_create() { return new RefState(); }
void ref_state_destroy(void* s) { delete static_cast<RefState*>(s); }

// count_mode == 0 -> Rasterizer::forward, else Rasterizer::forwardCount (gaussians_count and
// important_score must be zero-initialised by the caller, as rasterize_points.cu:177-178 does).
int ref_forward(void* state, int count_mode, int P, int D, int M, const float* background, int W, int H, const float* means3D,
                const float* shs, const float* colors_precomp, const float* opacities, const float* scales, float scale_modifier,
                const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                const float* campos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color, int* radii,
                int* gaussians_count, float* important_score)
{
    RefState* st = static_cast<RefState*>(state);
    st->P = P;
    std::function<char*(size_t)> g = [st](size_t n) { return st->geom.ensure(n); };
    std::function<char*(size_t)> b = [st](size_t n) { return st->binning.ensure(n); };
    std::function<char*(size_t)> i = [st](size_t n) { return st->img.ensure(n); };
    int R;
    if (!count_mode)
        R = CudaRasterizer::Rasterizer::forward(g, b, i, P, D, M, background, W, H, means3D, shs, colors_precomp, opacities, scales,
                                                scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx,
                                                tan_fovy, prefiltered != 0, out_color, radii, false);
    else
        R = CudaRasterizer::Rasterizer::forwardCount(g, b, i, P, D, M, background, W, H, means3D, shs, colors_precomp, opacities,
                                                     scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, campos,
                                                     tan_fovx, tan_fovy, prefiltered != 0, out_color, gaussians_count,
                                                     important_score, radii, false);
    st->num_rendered = R;
    return R;
}

// Gradient outputs must be zero-initialised by the caller (rasterize_points.cu:254-262).
void ref_backward(void* state, int P, int D, int M, const float* background, int W, int H, const float* means3D, const float* shs,
                  const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                  const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                  float tan_fovy, const int* radii, const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                  float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot)
{
    RefState* st = static_cast<RefState*>(state);
    CudaRasterizer::Rasterizer::backward(P, D, M, st->num_rendered, background, W, H, means3D, shs, colors_precomp, scales,
                                         scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy,
                                         radii, st->geom.ptr, st->binning.ptr, st->img.ptr, dL_dpix, dL_dmean2D, dL_dconic,
                                         dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, false);
}

void ref_mark_visible(int P, float* means3D, float* viewmatrix, float* projmatrix, bool* present)
{
    CudaRasterizer::Rasterizer::markVisible(P, means3D, viewmatrix, projmatrix, present);
}

// Device addresses of the reference's per-Gaussian intermediates inside the geometry blob of the
// last ref_forward call (layout: rasterizer_impl.cu:155-170), for golden-vector extraction.
// out[0..6] = depths, clamped(bool[3P]), means2D(float2), cov3D(float[6P]), conic_opacity(float4), rgb(float[3P]), tiles_touched
void ref_geom_ptrs(void* state, void** out)
{
    RefState* st = static_cast<RefState*>(state);
    char* chunk = st->geom.ptr;
    CudaRasterizer::GeometryState gs = CudaRasterizer::GeometryState::fromChunk(chunk, st->P);
    out[0] = gs.depths;
    out[1] = gs.clamped;
    out[2] = gs.means2D;
    out[3] = gs.cov3D;
    out[4] = gs.conic_opacity;
    out[5] = gs.rgb;
    out[6] = gs.tiles_touched;
}

// out[0..2] = accum_alpha (final_T, float[N]), n_contrib (u32[N]), ranges (uint2[N])
void ref_image_ptrs(void* state, int N, void** out)
{
    RefState* st = static_cast<RefState*>(state);
    char* chunk = st->img.ptr;
    CudaRasterizer::ImageState is = CudaRasterizer::ImageState::fromChunk(chunk, N);
    out[0] = is.accum_alpha;
    out[1] = is.n_contrib;
    out[2] = is.ranges;
}

// out[0] = point_list (u32[R]) sorted
void ref_binning_ptrs(void* state, void** out)
{
    RefState* st = static_cast<RefState*>(state);
    char* chunk = st->binning.ptr;
    CudaRasterizer::BinningState bs = CudaRasterizer::BinningState::fromChunk(chunk, st->num_rendered);
    out[0] = bs.point_list;
}

// Device -> host copy of `n` bytes (synchronous), so Python can read the intermediates above.
int ref_read(void* host_dst, const void* dev_src, size_t n) { return (int)cudaMemcpy(host_dst, dev_src, n, cudaMemcpyDeviceToHost); }

}  // extern "C"
