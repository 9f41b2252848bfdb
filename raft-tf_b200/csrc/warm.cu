// F10: warm start.  rb_flow_forward_interpolate is upstream RAFT's forward_interpolate (core/utils/utils.py): every source
// pixel is moved by its own 1/8-resolution flow, and every grid point takes the flow of the nearest source that landed
// strictly inside the frame (scipy.interpolate.griddata(method='nearest') in upstream, on the host).
//
// The valid sources of each sample are bucketed by integer cell (floor(x1), floor(y1)) -- the cells are the grid points
// themselves -- by integer-atomic counts, a per-sample block scan and a placement pass; then one thread per grid point
// scans Chebyshev rings of cells around it and keeps the minimum of (d, source index).  A source in ring r is more than
// r - 1 away along one axis, so the scan stops before ring r once (r - 1)^2 > d_best.  The order in which the placement
// lists a cell's sources depends on the atomics, but the result does not: the minimum of (d, index) is unique.
#define CCCL_DISABLE_NVTX
#include <cub/block/block_scan.cuh>
#include <math.h>

#include "common.cuh"

namespace rb {
namespace {

constexpr size_t kAlign = 256;
constexpr uint32_t kNone = 0xffffffffu;
constexpr int kScanThreads = 1024;

// workspace: per-cell counts and list offsets, each source's slot in its cell, the cell lists, per-sample valid counts
struct WarmWs {
  size_t counts, offsets, rank, list, nvalid, total;
};

WarmWs warm_layout(size_t n, int B) {
  WarmWs l;
  size_t o = 0;
  const size_t u32 = round_up(n * sizeof(uint32_t), kAlign);
  l.counts = o, o += u32;
  l.offsets = o, o += u32;
  l.rank = o, o += u32;
  l.list = o, o += u32;
  l.nvalid = o, o += round_up((size_t)B * sizeof(uint32_t), kAlign);
  l.total = o;
  return l;
}

// the target of source i (sample-local pixel (x, y)): numpy's int64 + float32 -> float64 sums are exact
__device__ __forceinline__ bool source_cell(float2 f, int x, int y, int h, int w, uint32_t* cell) {
  const double x1 = (double)x + (double)f.x, y1 = (double)y + (double)f.y;
  if (!(x1 > 0.0 && x1 < (double)w && y1 > 0.0 && y1 < (double)h)) return false;  // NaN fails every comparison
  *cell = (uint32_t)y1 * (uint32_t)w + (uint32_t)x1;  // positive: truncation is floor
  return true;
}

// One thread per source: its cell and its slot in that cell's list (integer atomics; the slot order is irrelevant).
__global__ void __launch_bounds__(256) warm_bucket_kernel(const float2* __restrict__ flow, int h, int w, uint32_t n,
                                                          uint32_t* __restrict__ counts, uint32_t* __restrict__ rank) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t hw = (uint32_t)h * w, local = i % hw;
  uint32_t cell, r = kNone;
  if (source_cell(flow[i], (int)(local % w), (int)(local / w), h, w, &cell)) r = atomicAdd(&counts[i - local + cell], 1u);
  rank[i] = r;
}

// One block per sample: exclusive scan of the sample's cell counts into list offsets (the sample's list starts at
// b*h*w), and the sample's number of valid sources.
__global__ void __launch_bounds__(kScanThreads) warm_scan_kernel(const uint32_t* __restrict__ counts,
                                                                 uint32_t* __restrict__ offsets,
                                                                 uint32_t* __restrict__ nvalid, uint32_t hw) {
  using Scan = cub::BlockScan<uint32_t, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const size_t base = (size_t)blockIdx.x * hw;
  const uint32_t chunk = (hw + kScanThreads - 1) / kScanThreads;
  const uint32_t lo = min(threadIdx.x * chunk, hw), hi = min(lo + chunk, hw);
  uint32_t sum = 0;
  for (uint32_t k = lo; k < hi; ++k) sum += counts[base + k];
  uint32_t run, total;
  Scan(tmp).ExclusiveSum(sum, run, total);
  run += (uint32_t)base;
  for (uint32_t k = lo; k < hi; ++k) {
    offsets[base + k] = run;
    run += counts[base + k];
  }
  if (threadIdx.x == 0) nvalid[blockIdx.x] = total;
}

__global__ void __launch_bounds__(256) warm_place_kernel(const float2* __restrict__ flow, int h, int w, uint32_t n,
                                                         const uint32_t* __restrict__ offsets,
                                                         const uint32_t* __restrict__ rank, uint32_t* __restrict__ list) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t r = rank[i];
  if (r == kNone) return;
  const uint32_t hw = (uint32_t)h * w, local = i % hw;
  uint32_t cell;
  source_cell(flow[i], (int)(local % w), (int)(local / w), h, w, &cell);
  list[offsets[i - local + cell] + r] = i;
}

// One thread per grid point: rings r = 0, 1, ... of cells around it, the minimum of (d, source index) over their lists;
// d = fl64(fl64((qx - x1)^2) + fl64((qy - y1)^2)) without FMA contraction (cKDTree's squared distance).
__global__ void __launch_bounds__(256) warm_query_kernel(const float2* __restrict__ flow, int h, int w, uint32_t n,
                                                         const uint32_t* __restrict__ counts,
                                                         const uint32_t* __restrict__ offsets,
                                                         const uint32_t* __restrict__ list,
                                                         const uint32_t* __restrict__ nvalid, float2* __restrict__ out) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const uint32_t hw = (uint32_t)h * w, local = g % hw, base = g - local;
  const int qx = (int)(local % w), qy = (int)(local / w);
  double best = INFINITY;
  uint32_t bi = kNone;
  if (nvalid[g / hw] > 0) {
    const int rmax = max(max(qx, w - 1 - qx), max(qy, h - 1 - qy));
    for (int r = 0; r <= rmax; ++r) {
      if (r > 0 && bi != kNone && (double)(r - 1) * (double)(r - 1) > best) break;
      for (int dy = -r; dy <= r; ++dy) {
        const int cy = qy + dy;
        if (cy < 0 || cy >= h) continue;
        const int step = (dy == -r || dy == r) ? 1 : 2 * r;  // full top / bottom rows, the two side cells otherwise
        for (int dx = -r; dx <= r; dx += step) {
          const int cx = qx + dx;
          if (cx < 0 || cx >= w) continue;
          const uint32_t c = base + (uint32_t)cy * w + (uint32_t)cx;
          const uint32_t o = offsets[c], e = o + counts[c];
          for (uint32_t j = o; j < e; ++j) {
            const uint32_t s = list[j], sl = s - base;
            const float2 f = flow[s];
            const double tx = __dsub_rn((double)qx, __dadd_rn((double)(sl % w), (double)f.x));
            const double ty = __dsub_rn((double)qy, __dadd_rn((double)(sl / w), (double)f.y));
            const double d = __dadd_rn(__dmul_rn(tx, tx), __dmul_rn(ty, ty));
            if (d < best || (d == best && s < bi)) best = d, bi = s;
          }
        }
      }
    }
  }
  out[g] = bi == kNone ? make_float2(0.f, 0.f) : flow[bi];
}

}  // namespace
}  // namespace rb

using namespace rb;

extern "C" int rb_flow_forward_interpolate_workspace_bytes(int B, int h, int w, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_flow_forward_interpolate_workspace_bytes: null pointer");
  RB_REQUIRE(B > 0 && h > 0 && w > 0, RB_ERR_BAD_SHAPE,
             "rb_flow_forward_interpolate_workspace_bytes: bad shape B=%d h=%d w=%d", B, h, w);
  const size_t n = (size_t)B * h * w;
  RB_REQUIRE(n < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_flow_forward_interpolate_workspace_bytes: B*h*w = %zu must be < 2^31", n);
  *bytes = warm_layout(n, B).total;
  return RB_OK;
}

extern "C" int rb_flow_forward_interpolate(const float* flow, float* out, int B, int h, int w, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  RB_REQUIRE(flow && out && workspace, RB_ERR_BAD_ARG, "rb_flow_forward_interpolate: null pointer");
  RB_REQUIRE(B > 0 && h > 0 && w > 0, RB_ERR_BAD_SHAPE, "rb_flow_forward_interpolate: bad shape B=%d h=%d w=%d", B, h,
             w);
  const size_t n = (size_t)B * h * w;
  RB_REQUIRE(n < (size_t(1) << 31), RB_ERR_BAD_SHAPE, "rb_flow_forward_interpolate: B*h*w = %zu must be < 2^31", n);
  const WarmWs l = warm_layout(n, B);
  RB_REQUIRE(workspace_bytes >= l.total, RB_ERR_WORKSPACE,
             "rb_flow_forward_interpolate: workspace of %zu bytes is too small (need %zu)", workspace_bytes, l.total);
  char* ws = static_cast<char*>(workspace);
  uint32_t* counts = reinterpret_cast<uint32_t*>(ws + l.counts);
  uint32_t* offsets = reinterpret_cast<uint32_t*>(ws + l.offsets);
  uint32_t* rank = reinterpret_cast<uint32_t*>(ws + l.rank);
  uint32_t* list = reinterpret_cast<uint32_t*>(ws + l.list);
  uint32_t* nvalid = reinterpret_cast<uint32_t*>(ws + l.nvalid);
  const float2* f = reinterpret_cast<const float2*>(flow);
  const cudaStream_t st = (cudaStream_t)stream;
  const uint32_t n32 = (uint32_t)n;
  const unsigned blocks = (unsigned)((n + 255) / 256);

  RB_CHECK_CUDA(cudaMemsetAsync(counts, 0, n * sizeof(uint32_t), st));
  warm_bucket_kernel<<<blocks, 256, 0, st>>>(f, h, w, n32, counts, rank);
  RB_CHECK_LAUNCH("warm_bucket_kernel");
  warm_scan_kernel<<<B, kScanThreads, 0, st>>>(counts, offsets, nvalid, (uint32_t)h * w);
  RB_CHECK_LAUNCH("warm_scan_kernel");
  warm_place_kernel<<<blocks, 256, 0, st>>>(f, h, w, n32, offsets, rank, list);
  RB_CHECK_LAUNCH("warm_place_kernel");
  warm_query_kernel<<<blocks, 256, 0, st>>>(f, h, w, n32, counts, offsets, list, nvalid, reinterpret_cast<float2*>(out));
  RB_CHECK_LAUNCH("warm_query_kernel");
  return RB_OK;
}
