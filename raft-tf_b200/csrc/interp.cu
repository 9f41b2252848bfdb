// F6: frame interpolation.  rb_flow_reverse is the reference's flow reversal (flow_utils.py:166-274,
// reverse_flow_avg_skip_static) batched and bit for bit; rb_frame_synthesize warps both frames to time t and blends them.
// The *_resized blends do the same at the frames' own size from flows reversed at the network size, resizing each flow
// (resize_px.cuh, rb_flow_resize's arithmetic) inside the kernel.
//
// Reversal: every source pixel of frame 0 is moved by time_step * flow to its nearest target pixel, and each target
// averages -time_step * flow over its sources in source raster order (the reference's loop order).  The fixed order
// rules out float atomics: keys (target index) are radix-sorted with the source index as value -- a stable sort, so
// every target's segment lists its sources in raster order -- and one thread per target sums its segment.  A target hit
// by every source of its frame therefore costs one thread O(H W): inherent to the order the result is defined by.
#define CCCL_DISABLE_NVTX
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <math.h>

#include "resize_px.cuh"

namespace rb {
namespace {

constexpr size_t kAlign = 256;
constexpr int kMaxSteps = RB_INTERP_MAX_STEPS;

// workspace: per-target counts and segment offsets, keys and values before / after the sort, the scaled flow of every
// source, the up/down neighbour count of the hole fill, then CUB's temporary storage
struct ReverseWs {
  size_t counts, offsets, keys_in, keys_out, vals_in, vals_out, fs, nfound, temp, fixed;
};

ReverseWs reverse_layout(size_t n) {
  ReverseWs l;
  size_t o = 0;
  const size_t u32 = round_up(n * sizeof(uint32_t), kAlign);
  l.counts = o, o += u32;
  l.offsets = o, o += u32;
  l.keys_in = o, o += u32;
  l.keys_out = o, o += u32;
  l.vals_in = o, o += u32;
  l.vals_out = o, o += u32;
  l.fs = o, o += round_up(n * sizeof(float2), kAlign);
  l.nfound = o, o += round_up(n, kAlign);
  l.temp = o;
  l.fixed = o;
  return l;
}

int key_bits(size_t n) {  // keys are 0..n (n = skipped source)
  int b = 1;
  while (b < 32 && (size_t(1) << b) <= n) ++b;
  return b;
}

// CUB's temporary storage for the sort and the scan (they run one after the other and share it)
cudaError_t cub_temp_bytes(size_t n, size_t* bytes) {
  size_t sort_b = 0, scan_b = 0;
  const uint32_t* ci = nullptr;
  uint32_t* o = nullptr;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort_b, ci, o, ci, o, (uint32_t)n, 0, key_bits(n));
  if (e != cudaSuccess) return e;
  e = cub::DeviceScan::ExclusiveSum(nullptr, scan_b, ci, o, (uint32_t)n);
  *bytes = round_up(sort_b > scan_b ? sort_b : scan_b, kAlign);
  return e;
}

// Time steps or times of one call, passed by value in the kernel parameters: nothing to copy or allocate.  Sample s of a
// call over B flow rows (or frame pairs) is time v[s / B] on row s % B; an item call (items = 1, launched with B = 1)
// gives every sample its own row: time v[s] on row row[s].
struct Steps {
  float v[kMaxSteps];
  int32_t row[kMaxSteps];
  int items;
};

// One thread per source pixel of every (step, sample): static mask, scaled flow, target key; counts by integer atomics
// (order-free).  Source i belongs to step j = i / n_flow and reads flow[i % n_flow] (an item call, n_flow = H W:
// flow[row[j] n_flow + i % n_flow]); its target lies in its own sample.
__global__ void __launch_bounds__(256) reverse_keys_kernel(const float2* __restrict__ flow, const void* __restrict__ bg,
                                                           const void* __restrict__ im0, int u8, int C, int H, int W,
                                                           uint32_t n, uint32_t n_flow, Steps steps,
                                                           uint32_t* __restrict__ counts, uint32_t* __restrict__ keys,
                                                           uint32_t* __restrict__ vals, float2* __restrict__ fs,
                                                           uint8_t* __restrict__ static_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t hw = (uint32_t)H * W;
  const int x = (int)(i % W), y = (int)((i / W) % H);
  const uint32_t base = i - (i % hw);
  const uint32_t j = i / n_flow;
  const float ts = steps.v[j];
  const size_t src = (steps.items ? (size_t)steps.row[j] * n_flow : 0) + i % n_flow;
  bool st = false;
  if (bg != nullptr) {  // static: every channel differs by < 10 (uint8: the wrapped difference, as numpy computes it)
    st = true;
    for (int c = 0; c < C; ++c) {
      const size_t k = (size_t)i * C + c;
      if (u8) {
        const uint8_t d = (uint8_t)(static_cast<const uint8_t*>(bg)[k] - static_cast<const uint8_t*>(im0)[k]);
        st = st && d < 10;
      } else {
        const float d = fabsf(__fsub_rn(static_cast<const float*>(bg)[k], static_cast<const float*>(im0)[k]));
        st = st && d < 10.f;
      }
    }
  }
  if (static_out != nullptr) static_out[i] = st ? 1 : 0;
  float2 f = st ? make_float2(INFINITY, INFINITY) : flow[src];
  f.x = __fmul_rn(f.x, ts);
  f.y = __fmul_rn(f.y, ts);
  fs[i] = f;
  // float32 + int64 arange promotes to float64 in the reference; +-inf is skipped there, NaN (where the reference
  // raises) is skipped here
  const double px = (double)f.x + x, py = (double)f.y + y;
  uint32_t key = n;
  if (isfinite(px) && isfinite(py)) {
    const int rx = (int)fmin(fmax(rint(px), 0.0), (double)(W - 1));  // rint: half to even, like np.round
    const int ry = (int)fmin(fmax(rint(py), 0.0), (double)(H - 1));
    key = base + (uint32_t)ry * W + rx;
    atomicAdd(&counts[key], 1u);
  }
  keys[i] = key;
  vals[i] = i;
}

// One thread per target: its sources in raster order, -f summed in fp32 from +0.0, divided as the reference does
// (fp32 sum / float64 count, rounded to fp32).
__global__ void __launch_bounds__(256) reverse_average_kernel(const uint32_t* __restrict__ counts,
                                                              const uint32_t* __restrict__ offsets,
                                                              const uint32_t* __restrict__ src,
                                                              const float2* __restrict__ fs, uint32_t n,
                                                              float2* __restrict__ flow_t, uint8_t* __restrict__ empty,
                                                              uint8_t* __restrict__ multi) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t c = counts[k], o = offsets[k];
  float ax = 0.f, ay = 0.f;
  constexpr uint32_t kBatch = 8;  // loads of a batch in flight together; the adds stay in order
  uint32_t j = 0;
  for (; j + kBatch <= c; j += kBatch) {
    float2 f[kBatch];
#pragma unroll
    for (uint32_t u = 0; u < kBatch; ++u) f[u] = fs[src[o + j + u]];
#pragma unroll
    for (uint32_t u = 0; u < kBatch; ++u) {
      ax = __fadd_rn(ax, -f[u].x);
      ay = __fadd_rn(ay, -f[u].y);
    }
  }
  for (; j < c; ++j) {
    const float2 f = fs[src[o + j]];
    ax = __fadd_rn(ax, -f.x);
    ay = __fadd_rn(ay, -f.y);
  }
  if (c > 0) {
    ax = __double2float_rn(__ddiv_rn((double)ax, (double)c));
    ay = __double2float_rn(__ddiv_rn((double)ay, (double)c));
  }
  flow_t[k] = make_float2(ax, ay);
  empty[k] = c == 0 ? 1 : 0;
  multi[k] = c > 1 ? 1 : 0;
}

// Hole fill, pass 1: one thread per (sample, column) walks down (nearest non-empty above) and up (below).  An empty
// pixel's flow_t holds the running sum (+0.0 + up) + down and nfound the neighbours found so far.  Only non-empty
// pixels are read as neighbours, so the sums never see each other.
__global__ void __launch_bounds__(128) fill_columns_kernel(float2* __restrict__ ft, const uint8_t* __restrict__ empty,
                                                           uint8_t* __restrict__ nfound, size_t S, int H, int W) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= S * W) return;
  const size_t b = t / W, x = t % W;
  const size_t col = b * H * W + x;
  bool have = false;
  float2 last = make_float2(0.f, 0.f);
  for (int y = 0; y < H; ++y) {
    const size_t p = col + (size_t)y * W;
    if (!empty[p]) {
      have = true;
      last = ft[p];
    } else {
      ft[p] = have ? make_float2(__fadd_rn(0.f, last.x), __fadd_rn(0.f, last.y)) : make_float2(0.f, 0.f);
      nfound[p] = have ? 1 : 0;
    }
  }
  have = false;
  for (int y = H - 1; y >= 0; --y) {
    const size_t p = col + (size_t)y * W;
    if (!empty[p]) {
      have = true;
      last = ft[p];
    } else if (have) {
      const float2 s = ft[p];
      ft[p] = make_float2(__fadd_rn(s.x, last.x), __fadd_rn(s.y, last.y));
      nfound[p] += 1;
    }
  }
}

// Pass 2: one thread per (sample, row) adds the nearest non-empty pixel on the left, then the right, and divides by the
// number found (fp32, correctly rounded); none found gives +0.0.
__global__ void __launch_bounds__(128) fill_rows_kernel(float2* __restrict__ ft, const uint8_t* __restrict__ empty,
                                                        uint8_t* __restrict__ nfound, size_t S, int H, int W) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= S * H) return;
  const size_t row = t * W;
  bool have = false;
  float2 last = make_float2(0.f, 0.f);
  for (int x = 0; x < W; ++x) {
    const size_t p = row + x;
    if (!empty[p]) {
      have = true;
      last = ft[p];
    } else if (have) {
      const float2 s = ft[p];
      ft[p] = make_float2(__fadd_rn(s.x, last.x), __fadd_rn(s.y, last.y));
      nfound[p] += 1;
    }
  }
  have = false;
  for (int x = W - 1; x >= 0; --x) {
    const size_t p = row + x;
    if (!empty[p]) {
      have = true;
      last = ft[p];
      continue;
    }
    float2 s = ft[p];
    int m = nfound[p];
    if (have) {
      s = make_float2(__fadd_rn(s.x, last.x), __fadd_rn(s.y, last.y));
      ++m;
    }
    // the fp32 quotient through fp64 (double rounding is innocuous for division: 53 >= 2*24 + 2); __fdiv_rn's slow-path
    // call would put this loop's state on the stack
    ft[p] = m > 0 ? make_float2(__double2float_rn(__ddiv_rn((double)s.x, (double)m)),
                                __double2float_rn(__ddiv_rn((double)s.y, (double)m)))
                  : make_float2(0.f, 0.f);
  }
}

// 5x5 minimum of `empty` over the window clipped to the image (cv2.erode's default border)
__global__ void __launch_bounds__(256) erode5_kernel(const uint8_t* __restrict__ empty, uint8_t* __restrict__ out,
                                                     int H, int W, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = (int)(i % W), y = (int)((i / W) % H);
  const uint8_t* img = empty + (i - ((size_t)y * W + x));
  uint8_t m = 1;
  for (int yy = max(y - 2, 0); yy <= min(y + 2, H - 1); ++yy)
    for (int xx = max(x - 2, 0); xx <= min(x + 2, W - 1); ++xx) m &= img[(size_t)yy * W + xx];
  out[i] = m;
}

// One frame of a blend as fp32 values: pixel (y, x), channel c of frame `img`, rows `row` values apart.  CropF32 reads
// fp32 frames (the engine's padded images from the crop's first pixel, or raw frames); RawU8 reads uint8 frames and
// scales them as rb_frames_prepare does (np.float32(u) / 255, from a table of the 256 quotients).
struct CropF32 {
  const float* img;
  size_t row;
  __device__ __forceinline__ float operator()(int y, int x, int c) const { return img[(size_t)y * row + (size_t)x * 3 + c]; }
};
struct RawU8 {
  const uint8_t* img;
  size_t row;
  const float* lut;
  __device__ __forceinline__ float operator()(int y, int x, int c) const {
    return lut[img[(size_t)y * row + (size_t)x * 3 + c]];
  }
};

// One pixel's three channels, in the frames' channel order
struct Rgb {
  float c[3];
};

// The blend of one output pixel (x, y) of an H x W frame: both frames sampled at p + F_k (clamped to the frame; NaN ->
// 0) with the bilinear arithmetic of rb_flow_fb_check, blended by (1-t, t) with empty targets weighted 0.
template <class Frame>
__device__ __forceinline__ Rgb synthesize_px(const Frame& i0, const Frame& i1, int x, int y, int H, int W, float2 F0,
                                             float2 F1, bool empty0, bool empty1, float t) {
  const float s = __fsub_rn(1.f, t);
  float w0 = empty0 ? 0.f : s, w1 = empty1 ? 0.f : t;
  if (w0 == 0.f && w1 == 0.f) w0 = s, w1 = t;
  float v[2][3];
  for (int k = 0; k < 2; ++k) {
    const float2 F = k == 0 ? F0 : F1;
    const Frame& img = k == 0 ? i0 : i1;
    const float qx = fminf(fmaxf(__fadd_rn((float)x, F.x), 0.f), (float)(W - 1));
    const float qy = fminf(fmaxf(__fadd_rn((float)y, F.y), 0.f), (float)(H - 1));
    const int x0 = (int)floorf(qx), y0 = (int)floorf(qy);
    const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const float ax = __fsub_rn(qx, (float)x0), ay = __fsub_rn(qy, (float)y0);
    const float cx = __fsub_rn(1.f, ax), cy = __fsub_rn(1.f, ay);
    for (int c = 0; c < 3; ++c) {
      const float t0 = __fadd_rn(__fmul_rn(cx, img(y0, x0, c)), __fmul_rn(ax, img(y0, x1, c)));
      const float t1 = __fadd_rn(__fmul_rn(cx, img(y1, x0, c)), __fmul_rn(ax, img(y1, x1, c)));
      v[k][c] = __fadd_rn(__fmul_rn(t0, cy), __fmul_rn(t1, ay));
    }
  }
  const float den = __fadd_rn(w0, w1);
  Rgb o;
  for (int c = 0; c < 3; ++c) o.c[c] = __fdiv_rn(__fadd_rn(__fmul_rn(w0, v[0][c]), __fmul_rn(w1, v[1][c])), den);
  return o;
}

// out[p] as fp32, or quantised to uint8 (with bgr: channels reversed)
__device__ __forceinline__ void store_px(const Rgb& o, void* out, size_t p, int out_u8, int bgr) {
  for (int c = 0; c < 3; ++c) {
    const int oc = bgr ? 2 - c : c;
    if (out_u8)
      static_cast<uint8_t*>(out)[p * 3 + oc] = quantise(o.c[c]);
    else
      static_cast<float*>(out)[p * 3 + oc] = o.c[c];
  }
}

// The inputs of the resized blend at output pixel (x, y) of Hs x Ws for reversal sample smp of the H x W flows:
// rb_flow_resize's flow there (resize_f32_px of the low-resolution flow, then u *= su, v *= sv) and the empty mask of
// the network pixel `near` whose area holds the pixel's centre, read through the read-only path.
__device__ __forceinline__ void resized_px(const float* __restrict__ f0, const float* __restrict__ f1,
                                           const uint8_t* __restrict__ e0, const uint8_t* __restrict__ e1, size_t smp,
                                           size_t near, int H, int W, int Hs, int Ws, int y, int x, int mode, float su,
                                           float sv, float2& F0, float2& F1, bool& m0, bool& m1) {
  const size_t lhw = (size_t)H * W;
  float a[2], c[2];
  resize_f32_px<2>(f0 + smp * lhw * 2, H, W, Hs, Ws, y, x, mode, a);
  resize_f32_px<2>(f1 + smp * lhw * 2, H, W, Hs, Ws, y, x, mode, c);
  F0 = make_float2(__fmul_rn(a[0], su), __fmul_rn(a[1], sv));
  F1 = make_float2(__fmul_rn(c[0], su), __fmul_rn(c[1], sv));
  m0 = __ldg(e0 + smp * lhw + near) != 0;
  m1 = __ldg(e1 + smp * lhw + near) != 0;
}

// One thread per output pixel, blockIdx.y striding over the (time, sample) pairs (32-bit pixel indices; a pair is
// (times.v[smp / B], smp % B), or an item's (v[smp], row[smp]), Steps): synthesize_px on the crop of the padded frames
// with the flows and masks of the same pixel.
__global__ void __launch_bounds__(256) frame_synthesize_kernel(const float* __restrict__ frames0,
                                                               const float* __restrict__ frames1, int Hp, int Wp, int top,
                                                               int left, const float2* __restrict__ f0,
                                                               const float2* __restrict__ f1,
                                                               const uint8_t* __restrict__ e0,
                                                               const uint8_t* __restrict__ e1, Steps times, void* out,
                                                               int out_u8, int bgr, int n_t, int B, int H, int W) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t hw = (uint32_t)H * W;
  if (q >= hw) return;
  const int x = (int)(q % W), y = (int)(q / W);
  for (uint32_t smp = blockIdx.y; smp < (uint32_t)n_t * B; smp += gridDim.y) {
    const uint32_t j = smp / (uint32_t)B;
    const int b = times.items ? times.row[j] : (int)(smp % B);
    const size_t p = (size_t)smp * hw + q;
    const size_t crop = ((size_t)b * Hp + top) * Wp * 3 + (size_t)left * 3;
    const CropF32 i0{frames0 + crop, (size_t)Wp * 3}, i1{frames1 + crop, (size_t)Wp * 3};
    store_px(synthesize_px(i0, i1, x, y, H, W, f0[p], f1[p], e0[p] != 0, e1[p] != 0, times.v[j]), out, p, out_u8, bgr);
  }
}

// The blend at the frames' own Hs x Ws from flows and masks at the network's H x W: one thread per output pixel,
// blockIdx.y striding over the (time, sample) pairs as in frame_synthesize_kernel.  Per pixel, F_k is rb_flow_resize's
// value there (resize_f32_px of the sample's low-resolution flow, then u *= su, v *= sv) and the empty mask that of the
// network pixel whose area holds the pixel's centre, (((2x+1) W) div (2 Ws), ((2y+1) H) div (2 Hs)) in 64-bit integers.
// The low-resolution reads go through the read-only path; uint8 frames are read as bytes.
template <bool U8>
__global__ void __launch_bounds__(256) frame_synthesize_resized_kernel(
    const void* __restrict__ frames0, const void* __restrict__ frames1, int Hs, int Ws, const float* __restrict__ f0,
    const float* __restrict__ f1, const uint8_t* __restrict__ e0, const uint8_t* __restrict__ e1, int H, int W,
    int mode, float su, float sv, Steps times, void* out, int out_u8, int bgr, int n_t, int B) {
  __shared__ float lut[256];
  if (U8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = __fdiv_rn((float)i, 255.0f);
    __syncthreads();
  }
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t hw = (uint32_t)Hs * (uint32_t)Ws;
  if (q >= hw) return;
  const int x = (int)(q % (uint32_t)Ws), y = (int)(q / (uint32_t)Ws);
  const size_t near = near_px(x, y, H, W, Hs, Ws);
  const size_t frame = (size_t)hw * 3;
  for (uint32_t smp = blockIdx.y; smp < (uint32_t)n_t * B; smp += gridDim.y) {
    const uint32_t j = smp / (uint32_t)B;
    const int b = times.items ? times.row[j] : (int)(smp % B);
    const size_t p = (size_t)smp * hw + q;
    float2 F0, F1;
    bool m0, m1;
    resized_px(f0, f1, e0, e1, smp, near, H, W, Hs, Ws, y, x, mode, su, sv, F0, F1, m0, m1);
    if (U8) {
      const RawU8 i0{static_cast<const uint8_t*>(frames0) + b * frame, (size_t)Ws * 3, lut};
      const RawU8 i1{static_cast<const uint8_t*>(frames1) + b * frame, (size_t)Ws * 3, lut};
      store_px(synthesize_px(i0, i1, x, y, Hs, Ws, F0, F1, m0, m1, times.v[j]), out, p, out_u8, bgr);
    } else {
      const CropF32 i0{static_cast<const float*>(frames0) + b * frame, (size_t)Ws * 3};
      const CropF32 i1{static_cast<const float*>(frames1) + b * frame, (size_t)Ws * 3};
      store_px(synthesize_px(i0, i1, x, y, Hs, Ws, F0, F1, m0, m1, times.v[j]), out, p, out_u8, bgr);
    }
  }
}

// F32's table (rb_expose_entry / rb_expose_row), by value in the kernel parameters like Steps
struct Expose {
  rb_expose_entry e[kMaxSteps];
  rb_expose_row r[kMaxSteps];
};

// A row's running sum at one pixel: +0.0 when the row opens, else its accumulator
__device__ __forceinline__ Rgb expose_start(const rb_expose_row& r, const float* acc, size_t hw, uint32_t q) {
  Rgb a;
  for (int c = 0; c < 3; ++c)
    a.c[c] = (r.flags & RB_EXPOSE_OPEN) ? 0.f : acc[((size_t)r.acc * hw + q) * 3 + c];
  return a;
}

__device__ __forceinline__ void expose_add(Rgb& a, const Rgb& v) {
  for (int c = 0; c < 3; ++c) a.c[c] = __fadd_rn(a.c[c], v.c[c]);
}

// A row's sum after its entries: closed, the quantised mean acc / m (bgr: channels reversed); else kept in acc
__device__ __forceinline__ void expose_finish(const rb_expose_row& r, Rgb a, float* acc, uint8_t* out, size_t hw,
                                              uint32_t q, int bgr) {
  if (r.flags & RB_EXPOSE_CLOSE) {
    const float m = (float)r.m;
    for (int c = 0; c < 3; ++c) a.c[c] = __fdiv_rn(a.c[c], m);
    store_px(a, out, (size_t)r.out * hw + q, 1, bgr);
  } else {
    for (int c = 0; c < 3; ++c) acc[((size_t)r.acc * hw + q) * 3 + c] = a.c[c];
  }
}

// One thread per (row, pixel), blockIdx.y the row: the row's entries in order, each the blend of its pair at its t
// (synthesize_px on the crops of frames[sample], frames[sample + 1] with the slot's flows and masks) or its input frame.
__global__ void __launch_bounds__(256) frame_expose_kernel(const float* __restrict__ frames, int Hp, int Wp, int top,
                                                           int left, const float2* __restrict__ f0,
                                                           const float2* __restrict__ f1,
                                                           const uint8_t* __restrict__ e0,
                                                           const uint8_t* __restrict__ e1, Expose tab, float* acc,
                                                           uint8_t* out, int bgr, int H, int W) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t hw = (uint32_t)H * W;
  if (q >= hw) return;
  const int x = (int)(q % W), y = (int)(q / W);
  const rb_expose_row& r = tab.r[blockIdx.y];
  Rgb a = expose_start(r, acc, hw, q);
  for (int i = r.first; i < r.first + r.count; ++i) {
    const rb_expose_entry& en = tab.e[i];
    const CropF32 i0{frames + ((size_t)en.sample * Hp + top) * Wp * 3 + (size_t)left * 3, (size_t)Wp * 3};
    Rgb v;
    if (en.slot < 0) {
      for (int c = 0; c < 3; ++c) v.c[c] = i0(y, x, c);
    } else {
      const CropF32 i1{i0.img + (size_t)Hp * Wp * 3, i0.row};
      const size_t p = (size_t)en.slot * hw + q;
      v = synthesize_px(i0, i1, x, y, H, W, f0[p], f1[p], e0[p] != 0, e1[p] != 0, en.t);
    }
    expose_add(a, v);
  }
  expose_finish(r, a, acc, out, hw, q, bgr);
}

// frame_expose_kernel at the frames' own Hs x Ws from flows and masks at H x W (resized_px, as
// frame_synthesize_resized_kernel); uint8 frames are read as bytes and scaled by the table of the 256 quotients.
template <bool U8>
__global__ void __launch_bounds__(256) frame_expose_resized_kernel(const void* __restrict__ frames, int Hs, int Ws,
                                                                   const float* __restrict__ f0,
                                                                   const float* __restrict__ f1,
                                                                   const uint8_t* __restrict__ e0,
                                                                   const uint8_t* __restrict__ e1, int H, int W,
                                                                   int mode, float su, float sv, Expose tab, float* acc,
                                                                   uint8_t* out, int bgr) {
  __shared__ float lut[256];
  if (U8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = __fdiv_rn((float)i, 255.0f);
    __syncthreads();
  }
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t hw = (uint32_t)Hs * (uint32_t)Ws;
  if (q >= hw) return;
  const int x = (int)(q % (uint32_t)Ws), y = (int)(q / (uint32_t)Ws);
  const size_t near = near_px(x, y, H, W, Hs, Ws);
  const size_t frame = (size_t)hw * 3;
  const rb_expose_row& r = tab.r[blockIdx.y];
  Rgb a = expose_start(r, acc, hw, q);
  for (int i = r.first; i < r.first + r.count; ++i) {
    const rb_expose_entry& en = tab.e[i];
    Rgb v;
    float2 F0 = make_float2(0.f, 0.f), F1 = F0;
    bool m0 = false, m1 = false;
    if (en.slot >= 0) resized_px(f0, f1, e0, e1, (size_t)en.slot, near, H, W, Hs, Ws, y, x, mode, su, sv, F0, F1, m0, m1);
    if (U8) {
      const RawU8 i0{static_cast<const uint8_t*>(frames) + en.sample * frame, (size_t)Ws * 3, lut};
      if (en.slot < 0) {
        for (int c = 0; c < 3; ++c) v.c[c] = i0(y, x, c);
      } else {
        const RawU8 i1{i0.img + frame, i0.row, lut};
        v = synthesize_px(i0, i1, x, y, Hs, Ws, F0, F1, m0, m1, en.t);
      }
    } else {
      const CropF32 i0{static_cast<const float*>(frames) + en.sample * frame, (size_t)Ws * 3};
      if (en.slot < 0) {
        for (int c = 0; c < 3; ++c) v.c[c] = i0(y, x, c);
      } else {
        const CropF32 i1{i0.img + frame, i0.row};
        v = synthesize_px(i0, i1, x, y, Hs, Ws, F0, F1, m0, m1, en.t);
      }
    }
    expose_add(a, v);
  }
  expose_finish(r, a, acc, out, hw, q, bgr);
}

}  // namespace
}  // namespace rb

using namespace rb;

namespace {

// checks of the multi-step entries' shapes; n = n_steps * B * H * W keys must stay below 2^32 with the skip key n
int reverse_shape(const char* fn, int n_steps, int B, int H, int W, size_t* n) {
  RB_REQUIRE(n_steps > 0 && n_steps <= kMaxSteps, RB_ERR_BAD_ARG, "%s: %d time steps (1..%d)", fn, n_steps, kMaxSteps);
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "%s: bad shape B=%d H=%d W=%d", fn, B, H, W);
  *n = (size_t)n_steps * B * H * W;
  RB_REQUIRE(*n + 1 < (size_t(1) << 32), RB_ERR_BAD_SHAPE,
             "%s: n_steps*B*H*W = %zu pixels: keys need n_steps*B*H*W + 1 < 2^32", fn, *n);
  return RB_OK;
}

// The reversal of flow01 [B,H,W,2] by n_steps time steps into [n_steps,B,H,W] samples, or with steps.items (B = 1) of
// flow01[steps.row[i]] by step i into sample i (arguments checked by the caller)
int reverse_run(const char* fn, const float* flow01, const void* bg, const void* im0, int img_u8, int img_channels,
                const Steps& steps, int n_steps, float* flow_t, uint8_t* empty, uint8_t* multi, uint8_t* static_mask,
                int B, int H, int W, void* workspace, size_t workspace_bytes, void* stream) {
  const size_t n = (size_t)n_steps * B * H * W;
  const ReverseWs l = reverse_layout(n);
  // the fixed part is known without CUDA; CUB's share needs a device query
  RB_REQUIRE(workspace_bytes >= l.fixed, RB_ERR_WORKSPACE, "%s: workspace of %zu bytes is too small", fn,
             workspace_bytes);
  size_t temp = 0;
  RB_CHECK_CUDA(cub_temp_bytes(n, &temp));
  RB_REQUIRE(workspace_bytes >= l.fixed + temp, RB_ERR_WORKSPACE, "%s: workspace of %zu bytes is too small (need %zu)",
             fn, workspace_bytes, l.fixed + temp);
  char* ws = static_cast<char*>(workspace);
  uint32_t* counts = reinterpret_cast<uint32_t*>(ws + l.counts);
  uint32_t* offsets = reinterpret_cast<uint32_t*>(ws + l.offsets);
  uint32_t* keys_in = reinterpret_cast<uint32_t*>(ws + l.keys_in);
  uint32_t* keys_out = reinterpret_cast<uint32_t*>(ws + l.keys_out);
  uint32_t* vals_in = reinterpret_cast<uint32_t*>(ws + l.vals_in);
  uint32_t* vals_out = reinterpret_cast<uint32_t*>(ws + l.vals_out);
  float2* fs = reinterpret_cast<float2*>(ws + l.fs);
  uint8_t* nfound = reinterpret_cast<uint8_t*>(ws + l.nfound);
  const cudaStream_t st = (cudaStream_t)stream;
  const uint32_t n32 = (uint32_t)n;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  const size_t S = (size_t)n_steps * B;  // samples of the hole fill

  RB_CHECK_CUDA(cudaMemsetAsync(counts, 0, n * sizeof(uint32_t), st));
  reverse_keys_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const float2*>(flow01), bg, im0, img_u8, img_channels, H,
                                              W, n32, (uint32_t)((size_t)B * H * W), steps, counts, keys_in, vals_in, fs,
                                              static_mask);
  RB_CHECK_LAUNCH("reverse_keys_kernel");
  size_t tb = temp;
  RB_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(ws + l.temp, tb, counts, offsets, n32, st));
  tb = temp;
  RB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(ws + l.temp, tb, keys_in, keys_out, vals_in, vals_out, n32, 0,
                                                key_bits(n), st));
  reverse_average_kernel<<<blocks, 256, 0, st>>>(counts, offsets, vals_out, fs, n32, reinterpret_cast<float2*>(flow_t),
                                                 empty, multi);
  RB_CHECK_LAUNCH("reverse_average_kernel");
  fill_columns_kernel<<<(unsigned)((S * W + 127) / 128), 128, 0, st>>>(reinterpret_cast<float2*>(flow_t), empty, nfound,
                                                                       S, H, W);
  RB_CHECK_LAUNCH("fill_columns_kernel");
  fill_rows_kernel<<<(unsigned)((S * H + 127) / 128), 128, 0, st>>>(reinterpret_cast<float2*>(flow_t), empty, nfound, S,
                                                                    H, W);
  RB_CHECK_LAUNCH("fill_rows_kernel");
  return RB_OK;
}

}  // namespace

extern "C" int rb_flow_reverse_workspace_bytes(int B, int H, int W, size_t* bytes) {
  return rb_flow_reverse_multi_workspace_bytes(1, B, H, W, bytes);
}

extern "C" int rb_flow_reverse_multi_workspace_bytes(int n_steps, int B, int H, int W, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_flow_reverse_workspace_bytes: null pointer");
  size_t n = 0;
  const int rc = reverse_shape("rb_flow_reverse_workspace_bytes", n_steps, B, H, W, &n);
  if (rc != RB_OK) return rc;
  size_t temp = 0;
  RB_CHECK_CUDA(cub_temp_bytes(n, &temp));
  *bytes = reverse_layout(n).fixed + temp;
  return RB_OK;
}

extern "C" int rb_flow_reverse(const float* flow01, const void* bg, const void* im0, int img_u8, int img_channels,
                               float time_step, float* flow_t, uint8_t* empty, uint8_t* multi, uint8_t* empty_eroded,
                               uint8_t* static_mask, int B, int H, int W, void* workspace, size_t workspace_bytes,
                               void* stream) {
  RB_REQUIRE(flow01 && flow_t && empty && multi && workspace, RB_ERR_BAD_ARG, "rb_flow_reverse: null pointer");
  RB_REQUIRE((bg == nullptr) == (im0 == nullptr), RB_ERR_BAD_ARG, "rb_flow_reverse: pass both bg and im0, or neither");
  RB_REQUIRE(bg == nullptr || img_channels > 0, RB_ERR_BAD_SHAPE, "rb_flow_reverse: img_channels must be > 0 (got %d)",
             img_channels);
  RB_REQUIRE(isfinite(time_step), RB_ERR_BAD_ARG, "rb_flow_reverse: time_step must be finite (got %g)",
             (double)time_step);
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_flow_reverse: bad shape B=%d H=%d W=%d", B, H, W);
  const size_t n = (size_t)B * H * W;
  RB_REQUIRE(n + 1 < (size_t(1) << 32), RB_ERR_BAD_SHAPE,
             "rb_flow_reverse: B*H*W = %zu pixels: keys need B*H*W + 1 < 2^32", n);
  Steps steps{};
  steps.v[0] = time_step;
  const int rc = reverse_run("rb_flow_reverse", flow01, bg, im0, img_u8, img_channels, steps, 1, flow_t, empty, multi,
                             static_mask, B, H, W, workspace, workspace_bytes, stream);
  if (rc != RB_OK) return rc;
  if (empty_eroded != nullptr) {
    erode5_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(empty, empty_eroded, H, W, (uint32_t)n);
    RB_CHECK_LAUNCH("erode5_kernel");
  }
  return RB_OK;
}

extern "C" int rb_flow_reverse_multi(const float* flow01, const float* time_steps, int n_steps, float* flow_t,
                                     uint8_t* empty, uint8_t* multi, int B, int H, int W, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  RB_REQUIRE(flow01 && time_steps && flow_t && empty && multi && workspace, RB_ERR_BAD_ARG,
             "rb_flow_reverse_multi: null pointer");
  size_t n = 0;
  const int rc = reverse_shape("rb_flow_reverse_multi", n_steps, B, H, W, &n);
  if (rc != RB_OK) return rc;
  Steps steps{};
  for (int i = 0; i < n_steps; ++i) {
    RB_REQUIRE(isfinite(time_steps[i]), RB_ERR_BAD_ARG, "rb_flow_reverse_multi: time_steps[%d] must be finite (got %g)",
               i, (double)time_steps[i]);
    steps.v[i] = time_steps[i];
  }
  return reverse_run("rb_flow_reverse_multi", flow01, nullptr, nullptr, 0, 0, steps, n_steps, flow_t, empty, multi,
                     nullptr, B, H, W, workspace, workspace_bytes, stream);
}

extern "C" int rb_flow_reverse_items(const float* flow01, int B, const int32_t* item_sample, const float* item_step,
                                     int n_items, float* flow_t, uint8_t* empty, uint8_t* multi, int H, int W,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  RB_REQUIRE(flow01 && item_sample && item_step && flow_t && empty && multi && workspace, RB_ERR_BAD_ARG,
             "rb_flow_reverse_items: null pointer");
  RB_REQUIRE(n_items > 0 && n_items <= kMaxSteps, RB_ERR_BAD_ARG, "rb_flow_reverse_items: %d items (1..%d)", n_items,
             kMaxSteps);
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_flow_reverse_items: bad shape B=%d H=%d W=%d", B, H, W);
  const size_t n = (size_t)n_items * H * W;
  RB_REQUIRE(n + 1 < (size_t(1) << 32), RB_ERR_BAD_SHAPE,
             "rb_flow_reverse_items: n_items*H*W = %zu pixels: keys need n_items*H*W + 1 < 2^32", n);
  Steps steps{};
  steps.items = 1;
  for (int i = 0; i < n_items; ++i) {
    RB_REQUIRE(item_sample[i] >= 0 && item_sample[i] < B, RB_ERR_BAD_ARG,
               "rb_flow_reverse_items: item_sample[%d] = %d outside [0, %d)", i, item_sample[i], B);
    RB_REQUIRE(isfinite(item_step[i]), RB_ERR_BAD_ARG, "rb_flow_reverse_items: item_step[%d] must be finite (got %g)", i,
               (double)item_step[i]);
    steps.row[i] = item_sample[i];
    steps.v[i] = item_step[i];
  }
  // one row per item: the kernels read flow01[row[i]] for sample i
  return reverse_run("rb_flow_reverse_items", flow01, nullptr, nullptr, 0, 0, steps, n_items, flow_t, empty, multi,
                     nullptr, 1, H, W, workspace, workspace_bytes, stream);
}

namespace {

// The blend entries after their pointer, count, flag and time checks: the shape, the item rows against the B frame
// pairs, the crop, then one launch over n_t times x B pairs, or over the n_t items (launched with B = 1)
int synthesize_run(const char* fn, const float* frames0, const float* frames1, int Hp, int Wp, int top, int left,
                   const float* flow_t0, const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1,
                   const Steps& times, int n_t, void* out, int out_u8, int bgr, int B, int H, int W, void* stream) {
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "%s: bad shape B=%d H=%d W=%d", fn, B, H, W);
  for (int i = 0; times.items && i < n_t; ++i)
    RB_REQUIRE(times.row[i] >= 0 && times.row[i] < B, RB_ERR_BAD_ARG, "%s: item_sample[%d] = %d outside [0, %d)", fn, i,
               times.row[i], B);
  RB_REQUIRE(top >= 0 && left >= 0 && top + H <= Hp && left + W <= Wp, RB_ERR_BAD_SHAPE,
             "%s: crop (%d, %d) + %dx%d outside the %dx%d frames", fn, top, left, H, W, Hp, Wp);
  const size_t hw = (size_t)H * W;
  const int rows = times.items ? 1 : B;
  RB_REQUIRE(hw < (size_t(1) << 32) && (size_t)n_t * rows < (size_t(1) << 32), RB_ERR_BAD_SHAPE,
             "%s: %zu pixels per frame or %zu frames exceed 32-bit indices", fn, hw, (size_t)n_t * rows);
  const dim3 grid((unsigned)((hw + 255) / 256), (unsigned)std::min<size_t>((size_t)n_t * rows, 65535));
  frame_synthesize_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      frames0, frames1, Hp, Wp, top, left, reinterpret_cast<const float2*>(flow_t0),
      reinterpret_cast<const float2*>(flow_t1), empty0, empty1, times, out, out_u8, bgr, n_t, rows, H, W);
  RB_CHECK_LAUNCH("frame_synthesize_kernel");
  return RB_OK;
}

}  // namespace

extern "C" int rb_frame_synthesize_pairs(const float* frames0, const float* frames1, int Hp, int Wp, int top, int left,
                                         const float* flow_t0, const float* flow_t1, const uint8_t* empty0,
                                         const uint8_t* empty1, const float* ts, int n_t, void* out, int out_u8,
                                         int bgr, int B, int H, int W, void* stream) {
  RB_REQUIRE(frames0 && frames1 && flow_t0 && flow_t1 && empty0 && empty1 && ts && out, RB_ERR_BAD_ARG,
             "rb_frame_synthesize: null pointer");
  RB_REQUIRE(n_t > 0 && n_t <= kMaxSteps, RB_ERR_BAD_ARG, "rb_frame_synthesize: %d times (1..%d)", n_t, kMaxSteps);
  RB_REQUIRE((out_u8 == 0 || out_u8 == 1) && (bgr == 0 || bgr == 1), RB_ERR_BAD_ARG,
             "rb_frame_synthesize: out_u8 and bgr must be 0 or 1 (got %d, %d)", out_u8, bgr);
  Steps times{};
  for (int i = 0; i < n_t; ++i) {
    RB_REQUIRE(ts[i] >= 0.f && ts[i] <= 1.f, RB_ERR_BAD_ARG, "rb_frame_synthesize: t must be in [0, 1] (got %g)",
               (double)ts[i]);
    times.v[i] = ts[i];
  }
  return synthesize_run("rb_frame_synthesize", frames0, frames1, Hp, Wp, top, left, flow_t0, flow_t1, empty0, empty1,
                        times, n_t, out, out_u8, bgr, B, H, W, stream);
}

extern "C" int rb_frame_synthesize_items(const float* frames0, const float* frames1, int Hp, int Wp, int top, int left,
                                         const float* flow_t0, const float* flow_t1, const uint8_t* empty0,
                                         const uint8_t* empty1, const int32_t* item_sample, const float* item_t,
                                         int n_items, void* out, int out_u8, int bgr, int B, int H, int W,
                                         void* stream) {
  RB_REQUIRE(frames0 && frames1 && flow_t0 && flow_t1 && empty0 && empty1 && item_sample && item_t && out,
             RB_ERR_BAD_ARG, "rb_frame_synthesize_items: null pointer");
  RB_REQUIRE(n_items > 0 && n_items <= kMaxSteps, RB_ERR_BAD_ARG, "rb_frame_synthesize_items: %d items (1..%d)",
             n_items, kMaxSteps);
  RB_REQUIRE((out_u8 == 0 || out_u8 == 1) && (bgr == 0 || bgr == 1), RB_ERR_BAD_ARG,
             "rb_frame_synthesize_items: out_u8 and bgr must be 0 or 1 (got %d, %d)", out_u8, bgr);
  Steps times{};
  times.items = 1;
  for (int i = 0; i < n_items; ++i) {
    RB_REQUIRE(item_t[i] >= 0.f && item_t[i] <= 1.f, RB_ERR_BAD_ARG,
               "rb_frame_synthesize_items: item_t[%d] must be in [0, 1] (got %g)", i, (double)item_t[i]);
    times.v[i] = item_t[i];
    times.row[i] = item_sample[i];
  }
  return synthesize_run("rb_frame_synthesize_items", frames0, frames1, Hp, Wp, top, left, flow_t0, flow_t1, empty0,
                        empty1, times, n_items, out, out_u8, bgr, B, H, W, stream);
}

extern "C" int rb_frame_synthesize(const float* frames, int Hp, int Wp, int top, int left, const float* flow_t0,
                                   const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1, float t,
                                   float* out, int B, int H, int W, void* stream) {
  // frames = [I0 | I1]; a bad shape is refused by the call below, with frames1 = frames
  const size_t frame1 = B > 0 && Hp > 0 && Wp > 0 ? (size_t)B * Hp * Wp * 3 : 0;
  return rb_frame_synthesize_pairs(frames, frames == nullptr ? nullptr : frames + frame1, Hp, Wp, top, left, flow_t0,
                                   flow_t1, empty0, empty1, &t, 1, out, 0, 0, B, H, W, stream);
}

namespace {

// The resized blend entries after their pointer, count, flag and time checks: the shapes, the item rows against the B
// frame pairs, then one launch over n_t times x B pairs, or over the n_t items (launched with B = 1)
int synthesize_resized_run(const char* fn, const void* frames0, const void* frames1, int frames_u8, int Hs, int Ws,
                           const float* flow_t0, const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1,
                           int H, int W, const Steps& times, int n_t, void* out, int out_u8, int bgr, int B,
                           void* stream) {
  RB_REQUIRE(B > 0 && H > 0 && W > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE, "%s: bad shape B=%d H=%d W=%d Hs=%d Ws=%d",
             fn, B, H, W, Hs, Ws);
  for (int i = 0; times.items && i < n_t; ++i)
    RB_REQUIRE(times.row[i] >= 0 && times.row[i] < B, RB_ERR_BAD_ARG, "%s: item_sample[%d] = %d outside [0, %d)", fn, i,
               times.row[i], B);
  const size_t hw = (size_t)Hs * Ws;
  const int rows = times.items ? 1 : B;
  RB_REQUIRE(hw < (size_t(1) << 32) && (size_t)n_t * rows < (size_t(1) << 32), RB_ERR_BAD_SHAPE,
             "%s: %zu pixels per frame or %zu frames exceed 32-bit indices", fn, hw, (size_t)n_t * rows);
  const dim3 grid((unsigned)((hw + 255) / 256), (unsigned)std::min<size_t>((size_t)n_t * rows, 65535));
  const int mode = float_mode(H, W, Hs, Ws);
  const float su = flow_scale_u(W, Ws), sv = flow_scale_v(H, Hs);
  const cudaStream_t st = (cudaStream_t)stream;
  if (frames_u8)
    frame_synthesize_resized_kernel<true><<<grid, 256, 0, st>>>(frames0, frames1, Hs, Ws, flow_t0, flow_t1, empty0,
                                                                empty1, H, W, mode, su, sv, times, out, out_u8, bgr, n_t,
                                                                rows);
  else
    frame_synthesize_resized_kernel<false><<<grid, 256, 0, st>>>(frames0, frames1, Hs, Ws, flow_t0, flow_t1, empty0,
                                                                 empty1, H, W, mode, su, sv, times, out, out_u8, bgr,
                                                                 n_t, rows);
  RB_CHECK_LAUNCH("frame_synthesize_resized_kernel");
  return RB_OK;
}

}  // namespace

extern "C" int rb_frame_synthesize_pairs_resized(const void* frames0, const void* frames1, int frames_u8, int Hs, int Ws,
                                                 const float* flow_t0, const float* flow_t1, const uint8_t* empty0,
                                                 const uint8_t* empty1, int H, int W, const float* ts, int n_t,
                                                 void* out, int out_u8, int bgr, int B, void* stream) {
  RB_REQUIRE(frames0 && frames1 && flow_t0 && flow_t1 && empty0 && empty1 && ts && out, RB_ERR_BAD_ARG,
             "rb_frame_synthesize_pairs_resized: null pointer");
  RB_REQUIRE(n_t > 0 && n_t <= kMaxSteps, RB_ERR_BAD_ARG, "rb_frame_synthesize_pairs_resized: %d times (1..%d)", n_t,
             kMaxSteps);
  RB_REQUIRE((frames_u8 == 0 || frames_u8 == 1) && (out_u8 == 0 || out_u8 == 1) && (bgr == 0 || bgr == 1),
             RB_ERR_BAD_ARG, "rb_frame_synthesize_pairs_resized: frames_u8, out_u8 and bgr must be 0 or 1 (got %d, %d, %d)",
             frames_u8, out_u8, bgr);
  Steps times{};
  for (int i = 0; i < n_t; ++i) {
    RB_REQUIRE(ts[i] >= 0.f && ts[i] <= 1.f, RB_ERR_BAD_ARG,
               "rb_frame_synthesize_pairs_resized: ts[%d] must be in [0, 1] (got %g)", i, (double)ts[i]);
    times.v[i] = ts[i];
  }
  return synthesize_resized_run("rb_frame_synthesize_pairs_resized", frames0, frames1, frames_u8, Hs, Ws, flow_t0,
                                flow_t1, empty0, empty1, H, W, times, n_t, out, out_u8, bgr, B, stream);
}

extern "C" int rb_frame_synthesize_items_resized(const void* frames0, const void* frames1, int frames_u8, int Hs, int Ws,
                                                 const float* flow_t0, const float* flow_t1, const uint8_t* empty0,
                                                 const uint8_t* empty1, int H, int W, const int32_t* item_sample,
                                                 const float* item_t, int n_items, void* out, int out_u8, int bgr, int B,
                                                 void* stream) {
  RB_REQUIRE(frames0 && frames1 && flow_t0 && flow_t1 && empty0 && empty1 && item_sample && item_t && out,
             RB_ERR_BAD_ARG, "rb_frame_synthesize_items_resized: null pointer");
  RB_REQUIRE(n_items > 0 && n_items <= kMaxSteps, RB_ERR_BAD_ARG, "rb_frame_synthesize_items_resized: %d items (1..%d)",
             n_items, kMaxSteps);
  RB_REQUIRE((frames_u8 == 0 || frames_u8 == 1) && (out_u8 == 0 || out_u8 == 1) && (bgr == 0 || bgr == 1),
             RB_ERR_BAD_ARG, "rb_frame_synthesize_items_resized: frames_u8, out_u8 and bgr must be 0 or 1 (got %d, %d, %d)",
             frames_u8, out_u8, bgr);
  Steps times{};
  times.items = 1;
  for (int i = 0; i < n_items; ++i) {
    RB_REQUIRE(item_t[i] >= 0.f && item_t[i] <= 1.f, RB_ERR_BAD_ARG,
               "rb_frame_synthesize_items_resized: item_t[%d] must be in [0, 1] (got %g)", i, (double)item_t[i]);
    times.v[i] = item_t[i];
    times.row[i] = item_sample[i];
  }
  return synthesize_resized_run("rb_frame_synthesize_items_resized", frames0, frames1, frames_u8, Hs, Ws, flow_t0,
                                flow_t1, empty0, empty1, H, W, times, n_items, out, out_u8, bgr, B, stream);
}

namespace {

// The checks of F32's tables, shared by both expose entries: every entry and row as include/raft_b200.h states, then
// the table packed into the kernel parameters.  Needs acc / out non-null only when a row reads or stores / closes.
int expose_table(const char* fn, const rb_expose_entry* entries, int n_entries, const rb_expose_row* rows, int n_rows,
                 int n_slots, int B, const float* acc, int n_acc, const uint8_t* out, int n_out, int bgr, Expose* tab) {
  RB_REQUIRE(entries && rows, RB_ERR_BAD_ARG, "%s: null pointer", fn);
  RB_REQUIRE(n_entries > 0 && n_entries <= kMaxSteps, RB_ERR_BAD_ARG, "%s: %d entries (1..%d)", fn, n_entries,
             kMaxSteps);
  RB_REQUIRE(n_rows > 0 && n_rows <= n_entries, RB_ERR_BAD_ARG, "%s: %d rows (1..%d entries)", fn, n_rows, n_entries);
  RB_REQUIRE(bgr == 0 || bgr == 1, RB_ERR_BAD_ARG, "%s: bgr must be 0 or 1 (got %d)", fn, bgr);
  RB_REQUIRE(B > 0, RB_ERR_BAD_SHAPE, "%s: B = %d pairs", fn, B);
  for (int i = 0; i < n_entries; ++i) {
    const rb_expose_entry& e = entries[i];
    RB_REQUIRE(e.slot >= RB_EXPOSE_FRAME && e.slot < n_slots, RB_ERR_BAD_ARG, "%s: entry %d: slot %d outside [-1, %d)",
               fn, i, e.slot, n_slots);
    const int hi = e.slot < 0 ? B : B - 1;
    RB_REQUIRE(e.sample >= 0 && e.sample <= hi, RB_ERR_BAD_ARG, "%s: entry %d: sample %d outside [0, %d]", fn, i,
               e.sample, hi);
    RB_REQUIRE(e.slot < 0 || (e.t >= 0.f && e.t <= 1.f), RB_ERR_BAD_ARG, "%s: entry %d: t must be in [0, 1] (got %g)",
               fn, i, (double)e.t);
    tab->e[i] = e;
  }
  bool reads_acc = false, closes = false;
  for (int r = 0; r < n_rows; ++r) {
    const rb_expose_row& w = rows[r];
    RB_REQUIRE(w.count >= 1 && w.first >= 0 && w.first <= n_entries - w.count, RB_ERR_BAD_ARG,
               "%s: row %d: entries %d + %d outside the %d of the table", fn, r, w.first, w.count, n_entries);
    RB_REQUIRE(w.m >= 1 && w.m <= (1 << 24), RB_ERR_BAD_ARG, "%s: row %d: m = %d samples (1..2^24)", fn, r, w.m);
    RB_REQUIRE((w.flags & ~(RB_EXPOSE_OPEN | RB_EXPOSE_CLOSE)) == 0, RB_ERR_BAD_ARG, "%s: row %d: flags %d", fn, r,
               w.flags);
    const bool uses_acc = w.flags != (RB_EXPOSE_OPEN | RB_EXPOSE_CLOSE), close = (w.flags & RB_EXPOSE_CLOSE) != 0;
    RB_REQUIRE(!uses_acc || (w.acc >= 0 && w.acc < n_acc), RB_ERR_BAD_ARG, "%s: row %d: acc %d outside [0, %d)", fn, r,
               w.acc, n_acc);
    RB_REQUIRE(!close || (w.out >= 0 && w.out < n_out), RB_ERR_BAD_ARG, "%s: row %d: out %d outside [0, %d)", fn, r,
               w.out, n_out);
    for (int o = 0; o < r; ++o) {  // rows run concurrently: none may touch another's accumulator or output frame
      const rb_expose_row& v = rows[o];
      RB_REQUIRE(!(uses_acc && v.flags != (RB_EXPOSE_OPEN | RB_EXPOSE_CLOSE) && v.acc == w.acc), RB_ERR_BAD_ARG,
                 "%s: rows %d and %d share acc %d", fn, o, r, w.acc);
      RB_REQUIRE(!(close && (v.flags & RB_EXPOSE_CLOSE) && v.out == w.out), RB_ERR_BAD_ARG,
                 "%s: rows %d and %d share out %d", fn, o, r, w.out);
    }
    reads_acc = reads_acc || uses_acc;
    closes = closes || close;
    tab->r[r] = w;
  }
  RB_REQUIRE((!reads_acc || acc) && (!closes || out), RB_ERR_BAD_ARG, "%s: null acc or out", fn);
  return RB_OK;
}

}  // namespace

extern "C" int rb_frame_expose_items(const float* frames, int Hp, int Wp, int top, int left, const float* flow_t0,
                                     const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1, int n_slots,
                                     const rb_expose_entry* entries, int n_entries, const rb_expose_row* rows,
                                     int n_rows, float* acc, int n_acc, uint8_t* out, int n_out, int bgr, int B, int H,
                                     int W, void* stream) {
  const char* fn = "rb_frame_expose_items";
  RB_REQUIRE(frames && (n_slots == 0 || (flow_t0 && flow_t1 && empty0 && empty1)), RB_ERR_BAD_ARG, "%s: null pointer",
             fn);
  Expose tab;
  const int rc = expose_table(fn, entries, n_entries, rows, n_rows, n_slots, B, acc, n_acc, out, n_out, bgr, &tab);
  if (rc != RB_OK) return rc;
  RB_REQUIRE(H > 0 && W > 0, RB_ERR_BAD_SHAPE, "%s: bad shape H=%d W=%d", fn, H, W);
  RB_REQUIRE(top >= 0 && left >= 0 && top + H <= Hp && left + W <= Wp, RB_ERR_BAD_SHAPE,
             "%s: crop (%d, %d) + %dx%d outside the %dx%d frames", fn, top, left, H, W, Hp, Wp);
  const size_t hw = (size_t)H * W;
  RB_REQUIRE(hw < (size_t(1) << 32), RB_ERR_BAD_SHAPE, "%s: %zu pixels per frame exceed 32-bit indices", fn, hw);
  const dim3 grid((unsigned)((hw + 255) / 256), (unsigned)n_rows);
  frame_expose_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      frames, Hp, Wp, top, left, reinterpret_cast<const float2*>(flow_t0), reinterpret_cast<const float2*>(flow_t1),
      empty0, empty1, tab, acc, out, bgr, H, W);
  RB_CHECK_LAUNCH("frame_expose_kernel");
  return RB_OK;
}

extern "C" int rb_frame_expose_items_resized(const void* frames, int frames_u8, int Hs, int Ws, const float* flow_t0,
                                             const float* flow_t1, const uint8_t* empty0, const uint8_t* empty1, int H,
                                             int W, int n_slots, const rb_expose_entry* entries, int n_entries,
                                             const rb_expose_row* rows, int n_rows, float* acc, int n_acc,
                                             uint8_t* out, int n_out, int bgr, int B, void* stream) {
  const char* fn = "rb_frame_expose_items_resized";
  RB_REQUIRE(frames && (n_slots == 0 || (flow_t0 && flow_t1 && empty0 && empty1)), RB_ERR_BAD_ARG, "%s: null pointer",
             fn);
  RB_REQUIRE(frames_u8 == 0 || frames_u8 == 1, RB_ERR_BAD_ARG, "%s: frames_u8 must be 0 or 1 (got %d)", fn, frames_u8);
  Expose tab;
  const int rc = expose_table(fn, entries, n_entries, rows, n_rows, n_slots, B, acc, n_acc, out, n_out, bgr, &tab);
  if (rc != RB_OK) return rc;
  RB_REQUIRE(H > 0 && W > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE, "%s: bad shape H=%d W=%d Hs=%d Ws=%d", fn, H, W, Hs,
             Ws);
  const size_t hw = (size_t)Hs * Ws;
  RB_REQUIRE(hw < (size_t(1) << 32), RB_ERR_BAD_SHAPE, "%s: %zu pixels per frame exceed 32-bit indices", fn, hw);
  const dim3 grid((unsigned)((hw + 255) / 256), (unsigned)n_rows);
  const int mode = float_mode(H, W, Hs, Ws);
  const float su = flow_scale_u(W, Ws), sv = flow_scale_v(H, Hs);
  const cudaStream_t st = (cudaStream_t)stream;
  if (frames_u8)
    frame_expose_resized_kernel<true><<<grid, 256, 0, st>>>(frames, Hs, Ws, flow_t0, flow_t1, empty0, empty1, H, W, mode,
                                                            su, sv, tab, acc, out, bgr);
  else
    frame_expose_resized_kernel<false><<<grid, 256, 0, st>>>(frames, Hs, Ws, flow_t0, flow_t1, empty0, empty1, H, W,
                                                             mode, su, sv, tab, acc, out, bgr);
  RB_CHECK_LAUNCH("frame_expose_resized_kernel");
  return RB_OK;
}
