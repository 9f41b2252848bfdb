// F27 / F28: video denoising -- each pixel merged with its patch matches in the frames that the chained consecutive flows
// reach consistently (rb_denoise_merge), and the Immerkaer noise estimate behind sigma = "auto" (rb_noise_sums).  Every
// fp32 operation is rounded on its own (__fadd_rn / __fmul_rn / __fsub_rn / __fdiv_rn, no FMA contraction), so a numpy
// restatement reproduces the bits (tests/denoise_oracle.py).  The merge uses no atomics; the noise sums are integers, so
// their int64 atomics are exact in any order.
#include <math.h>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

constexpr int kDenoiseThreads = 256;
constexpr int kSearch = RB_DENOISE_SEARCH;  // candidates at offsets -kSearch .. kSearch per axis
constexpr int kPatch = RB_DENOISE_PATCH;    // patches of (2 kPatch + 1)^2 pixels
constexpr int kReach = kSearch + kPatch;    // samples at integer offsets -kReach .. kReach around a match
constexpr int kSamp = 2 * kReach + 1;       // 5 x 5 samples
constexpr int kTaps = kSamp + 1;            // 6 x 6 taps
constexpr int kSide = 2 * kSearch + 1;
constexpr int kPw = 2 * kPatch + 1;
constexpr float kPatchVals = (float)(kPw * kPw * 3);  // 27: d is the mean over the patch's values

struct MergeAcc {
  float s[3];  // sum of w * centre colour per channel
  float w;     // sum of w
};

// The 9 candidates of one frame img [Hs,Ws,3] around position o (its bilinear weights b): the replicate-padded frame
// sampled at o + delta for the 5 x 5 integer offsets delta (taps clamped into the frame, b's weights), then per search
// offset s (raster order) the patch distance to ref and the weight, added to acc.
__device__ __forceinline__ void merge_frame(const uint8_t* __restrict__ img, int Hs, int Ws, const Bilerp& b,
                                            const float (&ref)[kPw][kPw][3], float two_var, float den, MergeAcc& acc) {
  int col[kTaps];
#pragma unroll
  for (int j = 0; j < kTaps; ++j) col[j] = min(max(b.x0 - kReach + j, 0), Ws - 1) * 3;
  float S[kSamp][kSamp][3];
  float hp[kSamp][3];
#pragma unroll
  for (int i = 0; i < kTaps; ++i) {
    const uint8_t* row = img + (size_t)min(max(b.y0 - kReach + i, 0), Hs - 1) * Ws * 3;
    float v[kTaps][3];
#pragma unroll
    for (int j = 0; j < kTaps; ++j)
#pragma unroll
      for (int c = 0; c < 3; ++c) v[j][c] = (float)__ldg(row + col[j] + c);
#pragma unroll
    for (int j = 0; j < kSamp; ++j)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float h = __fadd_rn(__fmul_rn(b.cx, v[j][c]), __fmul_rn(b.ax, v[j + 1][c]));
        if (i > 0) S[i - 1][j][c] = __fadd_rn(__fmul_rn(hp[j][c], b.cy), __fmul_rn(h, b.ay));
        hp[j][c] = h;
      }
  }
#pragma unroll
  for (int sy = 0; sy < kSide; ++sy)
#pragma unroll
    for (int sx = 0; sx < kSide; ++sx) {
      float d = 0.f;
#pragma unroll
      for (int uy = 0; uy < kPw; ++uy)
#pragma unroll
        for (int ux = 0; ux < kPw; ++ux)
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const float e = __fsub_rn(S[sy + uy][sx + ux][c], ref[uy][ux][c]);
            d = __fadd_rn(d, __fmul_rn(e, e));
          }
      d = __fdiv_rn(d, kPatchVals);
      const float num = fmaxf(__fsub_rn(d, two_var), 0.f);
      const float x = num > 0.f ? __fdiv_rn(num, den) : 0.f;
      const float om = __fsub_rn(1.f, x);
      const float w = x < 1.f ? __fmul_rn(om, om) : 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) acc.s[c] = __fadd_rn(acc.s[c], __fmul_rn(w, S[sy + kPatch][sx + kPatch][c]));
      acc.w = __fadd_rn(acc.w, w);
    }
}

// One side of pixel p (network position p0) of frame t: up to n chain steps (dir = +1 forward, -1 backward); every step
// that stays on the grid and passes the F5 test is a match, merged at its position mapped back to frame pixels.
// Returns the number of matched frames.
__device__ __forceinline__ int denoise_side(const uint8_t* __restrict__ frames, const float2* __restrict__ fw,
                                            const float2* __restrict__ bw, int t, int dir, int n, float2 p, int Hs,
                                            int Ws, int Hn, int Wn, const NetGeom& g, float s, float a1, float a2,
                                            const float (&ref)[kPw][kPw][3], float two_var, float den,
                                            MergeAcc& acc) {
  const size_t nn = (size_t)Hn * Wn, ns = (size_t)Hs * Ws;
  int step = 1;
  for (; step <= n; ++step) {
    const ChainLink l = chain_link(fw, bw, nn, t, dir, step);
    float2 q;
    if (chain_step(l.pull, l.test, Hn, Wn, s, a1, a2, p, q)) break;
    p = q;
    const Bilerp b = bilerp_at(px_remap(p.x, g.rxs, Ws), px_remap(p.y, g.rys, Hs), Hs, Ws);
    merge_frame(frames + (size_t)(t + dir * step) * ns * 3, Hs, Ws, b, ref, two_var, den, acc);
  }
  return step - 1;
}

// One thread per frame pixel, blockIdx.y over the rows (striding); row r = (t, nf, nb).
__global__ void __launch_bounds__(kDenoiseThreads) denoise_merge_kernel(
    const uint8_t* __restrict__ frames, int F, int Hs, int Ws, const float2* __restrict__ fw,
    const float2* __restrict__ bw, int Hn, int Wn, NetGeom g, float s, float a1, float a2,
    const int32_t* __restrict__ rows, int n_rows, float sigma, uint8_t* __restrict__ out,
    uint8_t* __restrict__ support) {
  // the weight's constants, each operation rounded on its own: 2 sigma^2 and (H sigma)^2
  const float two_var = __fmul_rn(2.f, __fmul_rn(sigma, sigma));
  const float hs = __fmul_rn(RB_DENOISE_H, sigma);
  const float den = __fmul_rn(hs, hs);
  const size_t ns = (size_t)Hs * Ws;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ns) return;
  const int x = (int)(q % Ws), y = (int)(q / Ws);
  for (int r = blockIdx.y; r < n_rows; r += gridDim.y) {
    const int t = __ldg(rows + 3 * r), nf = __ldg(rows + 3 * r + 1), nb = __ldg(rows + 3 * r + 2);
    uint8_t* o = out + ((size_t)r * ns + q) * 3;
    uint8_t* sup = support + (size_t)r * ns + q;
    if (t < 0 || t >= F) {  // an absent row
      o[0] = o[1] = o[2] = 0;
      *sup = 0;
      continue;
    }
    const uint8_t* img = frames + (size_t)t * ns * 3;
    float ref[kPw][kPw][3];
#pragma unroll
    for (int uy = 0; uy < kPw; ++uy) {
      const uint8_t* row = img + (size_t)min(max(y - kPatch + uy, 0), Hs - 1) * Ws * 3;
#pragma unroll
      for (int ux = 0; ux < kPw; ++ux) {
        const int cx = min(max(x - kPatch + ux, 0), Ws - 1) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) ref[uy][ux][c] = (float)__ldg(row + cx + c);
      }
    }
    MergeAcc acc = {{0.f, 0.f, 0.f}, 0.f};
    merge_frame(img, Hs, Ws, bilerp_at((float)x, (float)y, Hs, Ws), ref, two_var, den, acc);
    const float2 p = make_float2(px_remap(x, g.rxn, Wn), px_remap(y, g.ryn, Hn));
    const int wf = min(min(max(nf, 0), RB_DENOISE_MAX_WINDOW), F - 1 - t);
    const int wb = min(min(max(nb, 0), RB_DENOISE_MAX_WINDOW), t);
    const int df = denoise_side(frames, fw, bw, t, 1, wf, p, Hs, Ws, Hn, Wn, g, s, a1, a2, ref, two_var, den, acc);
    const int db = denoise_side(frames, fw, bw, t, -1, wb, p, Hs, Ws, Hn, Wn, g, s, a1, a2, ref, two_var, den, acc);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)fminf(fmaxf(rintf(__fdiv_rn(acc.s[c], acc.w)), 0.f), 255.f);
    *sup = (uint8_t)(df + db);
  }
}

// grid: pixel blocks x N.  Each interior pixel's |I * M| per channel (integers <= 16 * 255), summed over the block in
// shared memory, then one int64 atomic per block and channel.
__global__ void __launch_bounds__(kDenoiseThreads) noise_sums_kernel(const uint8_t* __restrict__ frames, int H, int W,
                                                                     unsigned long long* __restrict__ sums) {
  __shared__ int part[3][kDenoiseThreads / 32];
  const size_t np = (size_t)H * W;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint8_t* img = frames + (size_t)blockIdx.y * np * 3;
  int v[3] = {0, 0, 0};
  if (q < np) {
    const int x = (int)(q % W), y = (int)(q / W);
    if (x >= 1 && x <= W - 2 && y >= 1 && y <= H - 2) {
      const uint8_t* c0 = img + q * 3;
      const size_t rs = (size_t)W * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int a = (int)__ldg(c0 - rs - 3 + c) + (int)__ldg(c0 - rs + 3 + c) + (int)__ldg(c0 + rs - 3 + c) +
                      (int)__ldg(c0 + rs + 3 + c);
        const int e = (int)__ldg(c0 - rs + c) + (int)__ldg(c0 + rs + c) + (int)__ldg(c0 - 3 + c) + (int)__ldg(c0 + 3 + c);
        v[c] = abs(a - 2 * e + 4 * (int)__ldg(c0 + c));
      }
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s = __reduce_add_sync(0xffffffffu, v[c]);
    if (lane == 0) part[c][wid] = s;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    long long s = 0;
#pragma unroll
    for (int w = 0; w < kDenoiseThreads / 32; ++w) s += part[threadIdx.x][w];
    if (s) atomicAdd(sums + (size_t)blockIdx.y * 3 + threadIdx.x, (unsigned long long)s);
  }
}

}  // namespace rb

using namespace rb;

extern "C" int rb_denoise_merge(const uint8_t* frames, int F, int Hs, int Ws, const float* flow_fw,
                                const float* flow_bw, int Hn, int Wn, float flow_scale, float alpha1, float alpha2,
                                const int32_t* rows, int n_rows, float sigma, uint8_t* out, uint8_t* support,
                                void* stream) {
  const char* fn = "rb_denoise_merge";
  if (int rc = check_rows_entry(fn, frames && rows && out && support, flow_fw, flow_bw, F, Hs, Ws, Hn, Wn, n_rows))
    return rc;
  if (int rc = check_rows_step(fn, Hs, Ws, flow_scale, alpha1, alpha2)) return rc;
  RB_REQUIRE(sigma > 0.f && isfinite(sigma), RB_ERR_BAD_ARG,
             "rb_denoise_merge: sigma must be finite and > 0 (got %g)", (double)sigma);
  RB_REQUIRE(out != frames, RB_ERR_BAD_ARG, "rb_denoise_merge: out must not alias frames");
  denoise_merge_kernel<<<rows_grid(Hs, Ws, kDenoiseThreads, n_rows), kDenoiseThreads, 0, (cudaStream_t)stream>>>(
      frames, F, Hs, Ws, reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), Hn, Wn,
      net_geom(Hs, Ws, Hn, Wn), flow_scale, alpha1, alpha2, rows, n_rows, sigma, out, support);
  RB_CHECK_LAUNCH("denoise_merge_kernel");
  return RB_OK;
}

extern "C" int rb_noise_sums(const uint8_t* frames, int N, int H, int W, int64_t* sums, void* stream) {
  RB_REQUIRE(frames && sums, RB_ERR_BAD_ARG, "rb_noise_sums: null pointer");
  RB_REQUIRE(N > 0 && H >= 3 && W >= 3, RB_ERR_BAD_SHAPE,
             "rb_noise_sums: bad shape N=%d H=%d W=%d (an interior needs H, W >= 3)", N, H, W);
  RB_REQUIRE(N <= 65535 && (size_t)H * W < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_noise_sums: N=%d frames of %dx%d pixels exceed one grid", N, H, W);
  const cudaStream_t st = (cudaStream_t)stream;
  RB_CHECK_CUDA(cudaMemsetAsync(sums, 0, (size_t)N * 3 * sizeof(int64_t), st));
  const size_t np = (size_t)H * W;
  noise_sums_kernel<<<dim3((unsigned)((np + kDenoiseThreads - 1) / kDenoiseThreads), (unsigned)N), kDenoiseThreads, 0,
                      st>>>(frames, H, W, reinterpret_cast<unsigned long long*>(sums));
  RB_CHECK_LAUNCH("noise_sums_kernel");
  return RB_OK;
}
