// F18 / F19 / F21: keyframe label propagation -- per pixel of every frame, the displacement back to a keyframe accumulated
// through the consecutive flows of forward_sequence_bidirectional (the chained-flow baseline of video object
// segmentation), and the keyframe's labels pulled along it.  Every floating-point operation is rounded on its own
// (__fadd_rn / __fmul_rn / __fsub_rn, no FMA contraction), so an fp32 restatement reproduces the bits
// (tests/propagate_oracle.py); no float atomics.
#include <math.h>

#include "common.cuh"
#include "fb_sample.cuh"
#include "resize_px.cuh"

namespace rb {

// One step of the accumulation, one thread per pixel p = (x, y) of the row it writes.  pull is the flow from this frame to
// the previous one on the chain (flow_bw[r-1] forward, flow_fw[r] backward), test the opposite flow of the same pair;
// prev_acc / prev_st the row already written.  f = s pull(p), q = p + f.  Inside the frame: d = f and the F5 test of f
// against s test(q); outside: q clamped into the frame (replicate border), d = qc - p, status 2.  The row's displacement
// is d plus the bilinear sample of prev_acc at qc, its status the larger of the step's and prev_st's at qc's nearest tap.
__global__ void __launch_bounds__(256) flow_accumulate_step_kernel(
    const float2* __restrict__ pull, const float2* __restrict__ test, const float2* __restrict__ prev_acc,
    const uint8_t* __restrict__ prev_st, float2* __restrict__ acc, uint8_t* __restrict__ st, int H, int W, float s,
    float a1, float a2) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (uint32_t)H * (uint32_t)W) return;
  const int x = (int)(i % (uint32_t)W), y = (int)(i / (uint32_t)W);
  const float2 fr = pull[i];
  const float2 f = make_float2(__fmul_rn(s, fr.x), __fmul_rn(s, fr.y));
  const float qx = __fadd_rn((float)x, f.x), qy = __fadd_rn((float)y, f.y);
  float2 d;
  float cx, cy;
  uint8_t step;
  if (inside_frame(qx, qy, H, W)) {
    cx = qx;
    cy = qy;
    d = f;
    step = fb_inconsistent(f, sample_flow(test, W, bilerp_at(qx, qy, H, W), s), a1, a2);
  } else {  // fminf / fmaxf take the number over a NaN: a NaN coordinate clamps to 0
    cx = fminf(fmaxf(qx, 0.f), (float)(W - 1));
    cy = fminf(fmaxf(qy, 0.f), (float)(H - 1));
    d = make_float2(__fsub_rn(cx, (float)x), __fsub_rn(cy, (float)y));
    step = 2;
  }
  const Bilerp b = bilerp_at(cx, cy, H, W);
  const float2 v00 = prev_acc[(size_t)b.y0 * W + b.x0], v01 = prev_acc[(size_t)b.y0 * W + b.x1];
  const float2 v10 = prev_acc[(size_t)b.y1 * W + b.x0], v11 = prev_acc[(size_t)b.y1 * W + b.x1];
  acc[i] = make_float2(__fadd_rn(d.x, bilerp1(b, v00.x, v01.x, v10.x, v11.x)),
                       __fadd_rn(d.y, bilerp1(b, v00.y, v01.y, v10.y, v11.y)));
  const int nx = b.ax > 0.5f ? b.x1 : b.x0, ny = b.ay > 0.5f ? b.y1 : b.y0;
  const uint8_t carried = prev_st[(size_t)ny * W + nx];
  st[i] = step > carried ? step : carried;
}

// One keyframe side of an output pixel p = (x, y), row r: A' = rb_flow_resize's value of acc's row at p, the origin
// o = p + A' clamped into the key, status = the row's status at the network pixel `near` holding p's centre (2 if the clamp
// moved o), and o's four bilinear taps of the key with their weights in tap order 00, 01, 10, 11.
struct SideTaps {
  uint8_t l[4];
  float w[4];
  uint8_t st;
};

__device__ __forceinline__ SideTaps side_taps(const float* __restrict__ acc, const uint8_t* __restrict__ status,
                                              int H, int W, const uint8_t* __restrict__ key, int Hs, int Ws, int mode,
                                              float su, float sv, int x, int y, size_t near) {
  float a[2];
  resize_f32_px<2>(acc, H, W, Hs, Ws, y, x, mode, a);
  const float ox = __fadd_rn((float)x, __fmul_rn(a[0], su)), oy = __fadd_rn((float)y, __fmul_rn(a[1], sv));
  const float cx = fminf(fmaxf(ox, 0.f), (float)(Ws - 1)), cy = fminf(fmaxf(oy, 0.f), (float)(Hs - 1));
  const bool moved = !(cx == ox && cy == oy);  // a NaN origin counts as moved
  const Bilerp b = bilerp_at(cx, cy, Hs, Ws);
  SideTaps t;
  t.st = moved ? 2 : __ldg(status + near);
  t.l[0] = __ldg(key + (size_t)b.y0 * Ws + b.x0);
  t.l[1] = __ldg(key + (size_t)b.y0 * Ws + b.x1);
  t.l[2] = __ldg(key + (size_t)b.y1 * Ws + b.x0);
  t.l[3] = __ldg(key + (size_t)b.y1 * Ws + b.x1);
  t.w[0] = __fmul_rn(b.cx, b.cy);
  t.w[1] = __fmul_rn(b.ax, b.cy);
  t.w[2] = __fmul_rn(b.cx, b.ay);
  t.w[3] = __fmul_rn(b.ax, b.ay);
  return t;
}

// The label of the largest summed weight among N candidates: each scores the sum (left to right) of the weights of the
// candidates carrying its label; ties go to the smaller label.
template <int N>
__device__ __forceinline__ uint8_t vote(const uint8_t* l, const float* w) {
  uint8_t best = l[0];
  float top = -1.f;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float score = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j)
      if (l[j] == l[i]) score = __fadd_rn(score, w[j]);
    if (score > top || (score == top && l[i] < best)) {
      top = score;
      best = l[i];
    }
  }
  return best;
}

// The keyframe's labels at each output pixel p of Hs x Ws, row blockIdx.y (striding): side_taps of the row and the vote of
// its four taps.
__global__ void __launch_bounds__(256) labels_propagate_kernel(const float* __restrict__ acc,
                                                               const uint8_t* __restrict__ status, int n, int H, int W,
                                                               const uint8_t* __restrict__ key, int Hs, int Ws,
                                                               int mode, float su, float sv,
                                                               uint8_t* __restrict__ labels,
                                                               uint8_t* __restrict__ status_out) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t hw = (uint32_t)Hs * (uint32_t)Ws;
  if (q >= hw) return;
  const int x = (int)(q % (uint32_t)Ws), y = (int)(q / (uint32_t)Ws);
  const size_t lhw = (size_t)H * W;
  const size_t near = near_px(x, y, H, W, Hs, Ws);
  for (uint32_t r = blockIdx.y; r < (uint32_t)n; r += gridDim.y) {
    const SideTaps t = side_taps(acc + (size_t)r * lhw * 2, status + (size_t)r * lhw, H, W, key, Hs, Ws, mode, su, sv,
                                 x, y, near);
    const size_t o = (size_t)r * hw + q;
    labels[o] = vote<4>(t.l, t.w);
    status_out[o] = t.st;
  }
}

// F21: the labels of row r from the keyframes on either side of it.  rows[r] = (slot_a, slot_b, w_a, w_b): side A reads
// acc_a / status_a and key slot_a, side B acc_b / status_b and key slot_b; a slot outside [0, m) is an absent side.  The
// present sides with the smallest status vote: one with its plain bilinear weights (side_taps and vote<4>, so its bits are
// labels_propagate_kernel's), two with side A's weights times w_a and side B's times w_b over the eight taps A00 .. A11,
// B00 .. B11.  Status: the smallest, 3 (label 0) when no side is present.
__global__ void __launch_bounds__(256) labels_propagate_keys_kernel(
    const float* __restrict__ acc_a, const uint8_t* __restrict__ status_a, const float* __restrict__ acc_b,
    const uint8_t* __restrict__ status_b, const int4* __restrict__ rows, int n, int H, int W,
    const uint8_t* __restrict__ keys, int m, int Hs, int Ws, int mode, float su, float sv, uint8_t* __restrict__ labels,
    uint8_t* __restrict__ status_out) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t hw = (uint32_t)Hs * (uint32_t)Ws;
  if (q >= hw) return;
  const int x = (int)(q % (uint32_t)Ws), y = (int)(q / (uint32_t)Ws);
  const size_t lhw = (size_t)H * W;
  const size_t near = near_px(x, y, H, W, Hs, Ws);
  for (uint32_t r = blockIdx.y; r < (uint32_t)n; r += gridDim.y) {
    const int4 row = __ldg(rows + r);
    const bool has_a = row.x >= 0 && row.x < m, has_b = row.y >= 0 && row.y < m;
    const size_t o = (size_t)r * hw + q;
    if (!has_a && !has_b) {
      labels[o] = 0;
      status_out[o] = 3;
      continue;
    }
    SideTaps a, b;
    if (has_a)
      a = side_taps(acc_a + (size_t)r * lhw * 2, status_a + (size_t)r * lhw, H, W, keys + (size_t)row.x * hw, Hs, Ws,
                    mode, su, sv, x, y, near);
    if (has_b)
      b = side_taps(acc_b + (size_t)r * lhw * 2, status_b + (size_t)r * lhw, H, W, keys + (size_t)row.y * hw, Hs, Ws,
                    mode, su, sv, x, y, near);
    if (has_a && has_b && a.st == b.st) {
      const float fa = (float)row.z, fb = (float)row.w;
      uint8_t l[8];
      float w[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        l[i] = a.l[i];
        l[i + 4] = b.l[i];
        w[i] = __fmul_rn(a.w[i], fa);
        w[i + 4] = __fmul_rn(b.w[i], fb);
      }
      labels[o] = vote<8>(l, w);
      status_out[o] = a.st;
    } else {
      const bool use_a = has_a && (!has_b || a.st < b.st);
      uint8_t l[4];
      float w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        l[i] = use_a ? a.l[i] : b.l[i];
        w[i] = use_a ? a.w[i] : b.w[i];
      }
      labels[o] = vote<4>(l, w);
      status_out[o] = use_a ? a.st : b.st;
    }
  }
}

}  // namespace rb

using namespace rb;

namespace {

int accumulate_run(const char* fn, bool backward, const float* flow_fw, const float* flow_bw, int T, int H, int W,
                   int n_steps, float flow_scale, float alpha1, float alpha2, int start, float* acc, uint8_t* status,
                   void* stream) {
  RB_REQUIRE(flow_fw && flow_bw && acc && status, RB_ERR_BAD_ARG, "%s: null pointer", fn);
  RB_REQUIRE(T > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "%s: bad shape T=%d H=%d W=%d", fn, T, H, W);
  RB_REQUIRE((size_t)H * W < (size_t(1) << 31), RB_ERR_BAD_SHAPE, "%s: %dx%d pixels exceed 32-bit indices", fn, H, W);
  RB_REQUIRE(n_steps >= 1 && n_steps <= T, RB_ERR_BAD_SHAPE, "%s: n_steps must be in [1, T=%d] (got %d)", fn, T,
             n_steps);
  RB_REQUIRE(start >= 0 && start <= n_steps, RB_ERR_BAD_ARG, "%s: start must be in [0, n_steps=%d] (got %d)", fn,
             n_steps, start);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "%s: flow_scale must be finite and > 0 (got %g)", fn, (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "%s: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", fn, (double)alpha1, (double)alpha2);
  const size_t npix = (size_t)H * W;
  const unsigned blocks = (unsigned)((npix + 255) / 256);
  const cudaStream_t st = (cudaStream_t)stream;
  const float2* fw = reinterpret_cast<const float2*>(flow_fw);
  const float2* bw = reinterpret_cast<const float2*>(flow_bw);
  float2* a = reinterpret_cast<float2*>(acc);
  // one launch per step: a step reads arbitrary pixels of the row before it
  if (!backward) {
    for (int r = start + 1; r <= n_steps; ++r) {
      const size_t k = (size_t)(r - 1) * npix;
      flow_accumulate_step_kernel<<<blocks, 256, 0, st>>>(bw + k, fw + k, a + k, status + k, a + k + npix,
                                                          status + k + npix, H, W, flow_scale, alpha1, alpha2);
      RB_CHECK_LAUNCH("flow_accumulate_step_kernel");
    }
  } else {
    for (int r = start - 1; r >= 0; --r) {
      const size_t k = (size_t)r * npix;
      flow_accumulate_step_kernel<<<blocks, 256, 0, st>>>(fw + k, bw + k, a + k + npix, status + k + npix, a + k,
                                                          status + k, H, W, flow_scale, alpha1, alpha2);
      RB_CHECK_LAUNCH("flow_accumulate_step_kernel");
    }
  }
  return RB_OK;
}

}  // namespace

extern "C" int rb_flow_accumulate(const float* flow_fw, const float* flow_bw, int T, int H, int W, int n_steps,
                                  float flow_scale, float alpha1, float alpha2, int start, float* acc, uint8_t* status,
                                  void* stream) {
  return accumulate_run("rb_flow_accumulate", false, flow_fw, flow_bw, T, H, W, n_steps, flow_scale, alpha1, alpha2,
                        start, acc, status, stream);
}

extern "C" int rb_flow_accumulate_backward(const float* flow_fw, const float* flow_bw, int T, int H, int W,
                                           int n_steps, float flow_scale, float alpha1, float alpha2, int start,
                                           float* acc, uint8_t* status, void* stream) {
  return accumulate_run("rb_flow_accumulate_backward", true, flow_fw, flow_bw, T, H, W, n_steps, flow_scale, alpha1,
                        alpha2, start, acc, status, stream);
}

extern "C" int rb_labels_propagate(const float* acc, const uint8_t* status, int n, int H, int W, const uint8_t* key,
                                   int Hs, int Ws, uint8_t* labels, uint8_t* status_out, void* stream) {
  RB_REQUIRE(acc && status && key && labels && status_out, RB_ERR_BAD_ARG, "rb_labels_propagate: null pointer");
  RB_REQUIRE(n > 0 && H > 0 && W > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE,
             "rb_labels_propagate: bad shape n=%d H=%d W=%d Hs=%d Ws=%d", n, H, W, Hs, Ws);
  const size_t hw = (size_t)Hs * Ws;
  RB_REQUIRE(hw < (size_t(1) << 32), RB_ERR_BAD_SHAPE, "rb_labels_propagate: %zu pixels per frame exceed 32-bit indices",
             hw);
  const dim3 grid((unsigned)((hw + 255) / 256), (unsigned)std::min(n, 65535));
  labels_propagate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(acc, status, n, H, W, key, Hs, Ws,
                                                                  float_mode(H, W, Hs, Ws), flow_scale_u(W, Ws),
                                                                  flow_scale_v(H, Hs), labels, status_out);
  RB_CHECK_LAUNCH("labels_propagate_kernel");
  return RB_OK;
}

extern "C" int rb_labels_propagate_keys(const float* acc_a, const uint8_t* status_a, const float* acc_b,
                                        const uint8_t* status_b, const int32_t* rows, int n, int H, int W,
                                        const uint8_t* keys, int m, int Hs, int Ws, uint8_t* labels,
                                        uint8_t* status_out, void* stream) {
  RB_REQUIRE(acc_a && status_a && acc_b && status_b && rows && keys && labels && status_out, RB_ERR_BAD_ARG,
             "rb_labels_propagate_keys: null pointer");
  RB_REQUIRE(n > 0 && H > 0 && W > 0 && m > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE,
             "rb_labels_propagate_keys: bad shape n=%d H=%d W=%d m=%d Hs=%d Ws=%d", n, H, W, m, Hs, Ws);
  RB_REQUIRE(reinterpret_cast<uintptr_t>(rows) % alignof(int4) == 0, RB_ERR_BAD_ARG,
             "rb_labels_propagate_keys: rows must be 16-byte aligned");
  const size_t hw = (size_t)Hs * Ws;
  RB_REQUIRE(hw < (size_t(1) << 32), RB_ERR_BAD_SHAPE,
             "rb_labels_propagate_keys: %zu pixels per frame exceed 32-bit indices", hw);
  const dim3 grid((unsigned)((hw + 255) / 256), (unsigned)std::min(n, 65535));
  labels_propagate_keys_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      acc_a, status_a, acc_b, status_b, reinterpret_cast<const int4*>(rows), n, H, W, keys, m, Hs, Ws,
      float_mode(H, W, Hs, Ws), flow_scale_u(W, Ws), flow_scale_v(H, Hs), labels, status_out);
  RB_CHECK_LAUNCH("labels_propagate_keys_kernel");
  return RB_OK;
}
