// F11: flow colour coding on the GPU -- the repo's flow_utils.flow_to_color (the reference's flow_utils.py:95-121, the
// Middlebury colour wheel of Baker et al.), batched.  Two launches, like metrics.cu: every block takes the maximum radius
// of one fixed chunk of one sample's pixels into the workspace, then one thread per pixel reduces its sample's chunk
// maxima (in its block, through shared memory) and colours the pixel.  The chunks are per sample, so a sample's colours
// do not depend on B or on where it sits in the batch.
//
// Every operation is rounded on its own, in the type numpy computes it in for a float32 flow (no FMA contraction): the
// radius, normalisation, direction and wheel position in fp32, the interpolation and the colours in fp64.  The one
// deliberate difference is arctan2: numpy's float32 arctan2 depends on the machine (its SIMD kernels are not correctly
// rounded), so the direction here is the fp64 atan2 rounded once to fp32.
#include <math.h>

#include "common.cuh"

namespace rb {
namespace {

constexpr int kVizThreads = 256;
constexpr int kVizPerThread = 16;
constexpr int kVizChunk = kVizThreads * kVizPerThread;  // pixels per block of the max-radius launch
constexpr int kWheel = 55;                              // make_colorwheel(): RY 15, YG 6, GC 4, CB 11, BM 13, MR 6

// flow_utils.make_colorwheel(), RGB
__constant__ unsigned char c_wheel[kWheel][3] = {
    {255, 0, 0},   {255, 17, 0},  {255, 34, 0},  {255, 51, 0},  {255, 68, 0},  {255, 85, 0},  {255, 102, 0}, {255, 119, 0},
    {255, 136, 0}, {255, 153, 0}, {255, 170, 0}, {255, 187, 0}, {255, 204, 0}, {255, 221, 0}, {255, 238, 0}, {255, 255, 0},
    {213, 255, 0}, {170, 255, 0}, {128, 255, 0}, {85, 255, 0},  {43, 255, 0},  {0, 255, 0},   {0, 255, 63},  {0, 255, 127},
    {0, 255, 191}, {0, 255, 255}, {0, 232, 255}, {0, 209, 255}, {0, 186, 255}, {0, 163, 255}, {0, 140, 255}, {0, 116, 255},
    {0, 93, 255},  {0, 70, 255},  {0, 47, 255},  {0, 24, 255},  {0, 0, 255},   {19, 0, 255},  {39, 0, 255},  {58, 0, 255},
    {78, 0, 255},  {98, 0, 255},  {117, 0, 255}, {137, 0, 255}, {156, 0, 255}, {176, 0, 255}, {196, 0, 255}, {215, 0, 255},
    {235, 0, 255}, {255, 0, 255}, {255, 0, 213}, {255, 0, 170}, {255, 0, 128}, {255, 0, 85},  {255, 0, 43},
};

// np.clip(x, 0, c): minimum(maximum(x, 0), c) -- negative components become 0 (the reference's quirk)
__device__ __forceinline__ float2 viz_load(const float2* flow, size_t p, int clip, float c) {
  float2 f = flow[p];
  if (clip) {
    f.x = fminf(fmaxf(f.x, 0.f), c);
    f.y = fminf(fmaxf(f.y, 0.f), c);
  }
  return f;
}

__device__ __forceinline__ float viz_radius(float u, float v) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v)));
}

// grid (chunks per sample, B): the maximum radius of one chunk (order-independent, a fixed tree all the same)
__global__ void __launch_bounds__(kVizThreads) flow_color_max_kernel(const float2* __restrict__ flow, int clip, float c,
                                                                     float* __restrict__ partial, size_t npix) {
  __shared__ float red[kVizThreads];
  const size_t base = (size_t)blockIdx.y * npix;
  const size_t c0 = (size_t)blockIdx.x * kVizChunk;
  float m = 0.f;
#pragma unroll 4
  for (int k = 0; k < kVizPerThread; ++k) {
    const size_t q = c0 + (size_t)k * kVizThreads + threadIdx.x;
    if (q >= npix) break;
    const float2 f = viz_load(flow, base + q, clip, c);
    m = fmaxf(m, viz_radius(f.x, f.y));
  }
  red[threadIdx.x] = m;
  __syncthreads();
#pragma unroll
  for (int h = kVizThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = red[0];
}

// grid (pixel blocks per sample, B), one thread per pixel
__global__ void __launch_bounds__(kVizThreads) flow_color_kernel(const float2* __restrict__ flow, int clip, float c,
                                                                 const float* __restrict__ partial, int chunks,
                                                                 int bgr, uint8_t* __restrict__ out, size_t npix) {
  __shared__ float red[kVizThreads];
  const int b = blockIdx.y;
  float m = 0.f;
  for (int i = threadIdx.x; i < chunks; i += kVizThreads) m = fmaxf(m, partial[(size_t)b * chunks + i]);
  red[threadIdx.x] = m;
  __syncthreads();
#pragma unroll
  for (int h = kVizThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  const size_t q = (size_t)blockIdx.x * kVizThreads + threadIdx.x;
  if (q >= npix) return;
  const size_t p = (size_t)b * npix + q;
  const float2 f = viz_load(flow, p, clip, c);
  const float den = __fadd_rn(red[0], 1e-5f);  // fl32(rad_max + fl32(1e-5))
  const float u = __fdiv_rn(f.x, den), v = __fdiv_rn(f.y, den);
  const float rad = viz_radius(u, v);
  // arctan2(-v, -u) / pi: the fp64 atan2 rounded once to fp32, then the fp32 quotient by fl32(pi)
  const float at = __double2float_rn(atan2(-(double)v, -(double)u));
  const float a = __fdiv_rn(at, 3.14159265358979323846f);
  const float fk = __fadd_rn(__fmul_rn(__fdiv_rn(__fadd_rn(a, 1.f), 2.f), (float)(kWheel - 1)), 1.f);
  // k0 = min(floor(fk), 53), clamped into the wheel for any input (a NaN gives 0; its colour is unspecified)
  const float fl = floorf(fk);
  const int k0 = fl >= 0.f ? (fl < (float)(kWheel - 2) ? (int)fl : kWheel - 2) : 0;
  const int k1 = k0 + 1 == kWheel ? 1 : k0 + 1;
  const double fr = __dsub_rn((double)fk, (double)k0);
  const double g = __dsub_rn(1.0, fr);
  uint8_t rgb[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const double c0 = __ddiv_rn((double)c_wheel[k0][ch], 255.0), c1 = __ddiv_rn((double)c_wheel[k1][ch], 255.0);
    double col = __dadd_rn(__dmul_rn(g, c0), __dmul_rn(fr, c1));
    col = rad <= 1.f ? __dsub_rn(1.0, __dmul_rn((double)rad, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    const double q255 = floor(__dmul_rn(255.0, col));
    rgb[ch] = (uint8_t)(q255 >= 0.0 ? (q255 <= 255.0 ? q255 : 255.0) : 0.0);
  }
  uint8_t* o = out + p * 3;
  o[0] = bgr ? rgb[2] : rgb[0];
  o[1] = rgb[1];
  o[2] = bgr ? rgb[0] : rgb[2];
}

size_t viz_chunks(int H, int W) { return ((size_t)H * W + kVizChunk - 1) / kVizChunk; }

}  // namespace
}  // namespace rb

using namespace rb;

extern "C" int rb_flow_to_color_workspace_bytes(int B, int H, int W, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_flow_to_color_workspace_bytes: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_flow_to_color_workspace_bytes: bad shape B=%d H=%d W=%d", B,
             H, W);
  *bytes = (size_t)B * viz_chunks(H, W) * sizeof(float);
  return RB_OK;
}

extern "C" int rb_flow_to_color(const float* flow, int B, int H, int W, int clip, float clip_flow, int convert_to_bgr,
                                uint8_t* out, void* workspace, size_t workspace_bytes, void* stream) {
  RB_REQUIRE(flow && out && workspace, RB_ERR_BAD_ARG, "rb_flow_to_color: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_flow_to_color: bad shape B=%d H=%d W=%d", B, H, W);
  RB_REQUIRE(!clip || isfinite(clip_flow), RB_ERR_BAD_ARG, "rb_flow_to_color: clip_flow must be finite (got %g)",
             (double)clip_flow);
  const size_t npix = (size_t)H * W;
  const size_t chunks = viz_chunks(H, W);
  const size_t blocks = (npix + kVizThreads - 1) / kVizThreads;
  RB_REQUIRE(B <= 65535 && blocks <= 0x7fffffffu, RB_ERR_BAD_SHAPE,
             "rb_flow_to_color: B=%d samples of %zu pixels exceed one grid", B, npix);
  const size_t need = (size_t)B * chunks * sizeof(float);
  RB_REQUIRE(workspace_bytes >= need, RB_ERR_WORKSPACE, "rb_flow_to_color: workspace of %zu bytes, %zu needed",
             workspace_bytes, need);
  const cudaStream_t st = (cudaStream_t)stream;
  const float2* f2 = reinterpret_cast<const float2*>(flow);
  float* partial = static_cast<float*>(workspace);
  flow_color_max_kernel<<<dim3((unsigned)chunks, (unsigned)B), kVizThreads, 0, st>>>(f2, clip, clip_flow, partial, npix);
  RB_CHECK_LAUNCH("flow_color_max_kernel");
  flow_color_kernel<<<dim3((unsigned)blocks, (unsigned)B), kVizThreads, 0, st>>>(f2, clip, clip_flow, partial,
                                                                                (int)chunks, convert_to_bgr != 0, out,
                                                                                npix);
  RB_CHECK_LAUNCH("flow_color_kernel");
  return RB_OK;
}
