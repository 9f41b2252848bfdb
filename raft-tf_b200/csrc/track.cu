// F16: point tracking through a video -- the consecutive flows of forward_sequence_bidirectional chained per point, with
// the forward-backward test of F5 at every step (the chained-flow baseline of TAP-Vid, Doersch et al. 2022).
#include <math.h>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

// One thread per query: its position stays in a register across the pass's steps.  No atomics and no shared state, so a
// query's track does not depend on N, on the other queries or on where the passes split the clip.  Row j of tracks /
// status is frame first_frame + j; every row is stored by all threads at once (frame-major), so the stores coalesce.
__global__ void __launch_bounds__(128) track_points_kernel(const float2* __restrict__ flow_fw,
                                                           const float2* __restrict__ flow_bw, int H, int W, int n_steps,
                                                           float s, float a1, float a2, const int* __restrict__ qframe,
                                                           const float2* __restrict__ qpos, int N, int first_frame,
                                                           float2* __restrict__ pos, uint8_t* __restrict__ state,
                                                           float2* __restrict__ tracks, uint8_t* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float nan = __int_as_float(0x7fc00000);
  const long long q0 = (long long)qframe[i] - first_frame;  // the row of the query frame (any value)
  float2 p = make_float2(nan, nan);
  uint8_t st = 3;
  if (q0 < 0) {  // started in an earlier pass: continue from the carried state
    p = pos[i];
    st = state[i];
  }
  const size_t npix = (size_t)H * W;
  for (int j = 0; j <= n_steps; ++j) {
    if (j < q0) {
      p = make_float2(nan, nan);
      st = 3;
    } else if (j == q0) {
      p = qpos[i];
      st = 0;
    } else if (j > 0 && st <= 1) {  // step j-1 -> j; status 2 (and a carried 3) stay as they are
      const size_t k = (size_t)(j - 1) * npix;
      float2 q;
      // only a query position outside the frame fails the first test
      st = inside_frame(p.x, p.y, H, W) ? chain_step(flow_fw + k, flow_bw + k, H, W, s, a1, a2, p, q) : 2;
      p = st == 2 ? make_float2(nan, nan) : q;
    }
    tracks[(size_t)j * N + i] = p;
    status[(size_t)j * N + i] = st;
  }
  pos[i] = p;
  state[i] = st;
}

// F17: the mirror of track_points_kernel, from the query frame back to frame first_frame.  Rows after the query frame are
// not stored, so a launch after track_points_kernel on the same tracks / status completes them in place.  Step j+1 -> j
// is the forward step with the flows' roles swapped at pair j: f from flow_bw[j] at p, the test against flow_fw[j] at p + f.
__global__ void __launch_bounds__(128) track_points_backward_kernel(
    const float2* __restrict__ flow_fw, const float2* __restrict__ flow_bw, int H, int W, int n_steps, float s, float a1,
    float a2, const int* __restrict__ qframe, const float2* __restrict__ qpos, int N, int first_frame,
    float2* __restrict__ pos, uint8_t* __restrict__ state, float2* __restrict__ tracks, uint8_t* __restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const long long q0 = (long long)qframe[i] - first_frame;  // the row of the query frame (any value)
  if (q0 < 0) return;  // the query frame lies in an earlier call's frames: nothing to do here
  const float nan = __int_as_float(0x7fc00000);
  float2 p = make_float2(nan, nan);
  uint8_t st = 3;
  if (q0 > n_steps) {  // the query frame lies in a later call of a reverse sweep: continue from the carried state
    p = pos[i];
    st = state[i];
  }
  const size_t npix = (size_t)H * W;
  for (int j = n_steps; j >= 0; --j) {
    if (j > q0) continue;  // after the query frame: the forward launch's rows
    if (j == q0) {
      p = qpos[i];
      st = 0;
    } else if (j < n_steps && st <= 1) {  // step j+1 -> j; status 2 (and a carried 3) stay as they are
      const size_t k = (size_t)j * npix;
      float2 q;
      // only a query position outside the frame fails the first test
      st = inside_frame(p.x, p.y, H, W) ? chain_step(flow_bw + k, flow_fw + k, H, W, s, a1, a2, p, q) : 2;
      p = st == 2 ? make_float2(nan, nan) : q;
    }
    tracks[(size_t)j * N + i] = p;
    status[(size_t)j * N + i] = st;
  }
  pos[i] = p;
  state[i] = st;
}

}  // namespace rb

using namespace rb;

extern "C" int rb_track_points(const float* flow_fw, const float* flow_bw, int T, int H, int W, int n_steps,
                               float flow_scale, float alpha1, float alpha2, const int32_t* qframe, const float* qpos,
                               int N, int first_frame, float* pos, uint8_t* state, float* tracks, uint8_t* status,
                               void* stream) {
  RB_REQUIRE(flow_fw && flow_bw && qframe && qpos && pos && state && tracks && status, RB_ERR_BAD_ARG,
             "rb_track_points: null pointer");
  RB_REQUIRE(T > 0 && H > 0 && W > 0 && N > 0, RB_ERR_BAD_SHAPE, "rb_track_points: bad shape T=%d H=%d W=%d N=%d", T, H,
             W, N);
  RB_REQUIRE(n_steps >= 1 && n_steps <= T, RB_ERR_BAD_SHAPE, "rb_track_points: n_steps must be in [1, T=%d] (got %d)", T,
             n_steps);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_track_points: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "rb_track_points: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", (double)alpha1, (double)alpha2);
  const unsigned blocks = (unsigned)((N + 127LL) / 128);  // N < 2^31: at most 2^24 blocks, inside one grid
  track_points_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), H, W, n_steps, flow_scale,
      alpha1, alpha2, qframe, reinterpret_cast<const float2*>(qpos), N, first_frame, reinterpret_cast<float2*>(pos),
      state, reinterpret_cast<float2*>(tracks), status);
  RB_CHECK_LAUNCH("track_points_kernel");
  return RB_OK;
}

extern "C" int rb_track_points_backward(const float* flow_fw, const float* flow_bw, int T, int H, int W, int n_steps,
                                        float flow_scale, float alpha1, float alpha2, const int32_t* qframe,
                                        const float* qpos, int N, int first_frame, float* pos, uint8_t* state,
                                        float* tracks, uint8_t* status, void* stream) {
  RB_REQUIRE(flow_fw && flow_bw && qframe && qpos && pos && state && tracks && status, RB_ERR_BAD_ARG,
             "rb_track_points_backward: null pointer");
  RB_REQUIRE(T > 0 && H > 0 && W > 0 && N > 0, RB_ERR_BAD_SHAPE,
             "rb_track_points_backward: bad shape T=%d H=%d W=%d N=%d", T, H, W, N);
  RB_REQUIRE(n_steps >= 1 && n_steps <= T, RB_ERR_BAD_SHAPE,
             "rb_track_points_backward: n_steps must be in [1, T=%d] (got %d)", T, n_steps);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_track_points_backward: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "rb_track_points_backward: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", (double)alpha1,
             (double)alpha2);
  const unsigned blocks = (unsigned)((N + 127LL) / 128);
  track_points_backward_kernel<<<blocks, 128, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), H, W, n_steps, flow_scale,
      alpha1, alpha2, qframe, reinterpret_cast<const float2*>(qpos), N, first_frame, reinterpret_cast<float2*>(pos),
      state, reinterpret_cast<float2*>(tracks), status);
  RB_CHECK_LAUNCH("track_points_backward_kernel");
  return RB_OK;
}
