// F15: scene-cut scores of a frame sequence -- one minus the intersection of consecutive frames' joint colour histograms
// (8 levels per channel, RB_SCENE_BINS bins).  Counts are integers, so the histograms and the scores are exact and do not
// depend on the launch order: a memset, one histogram launch and one score launch, no allocation, graph-capturable.
#include "common.cuh"

namespace rb {

constexpr int kSceneThreads = 256;
constexpr int kScenePerThread = 16;
constexpr int kSceneChunk = kSceneThreads * kScenePerThread;  // pixels per block
constexpr int kSceneBins = RB_SCENE_BINS;

// grid: chunks per frame x N (flattened).  Thread t takes pixels chunk_start + i * 256 + t, i = 0..15 (coalesced), loads
// all of them first, then adds them to the block's shared histogram one pixel per lane at a time: __match_any_sync groups
// the lanes of a warp whose pixels share a bin and the lowest lane of each group adds the group's size, so a frame of one
// colour costs one shared atomic per warp and pixel step, not 32 on one address.  The block's nonzero bins are then added
// to the frame's global histogram (integer atomics: exact in any order).
__global__ void __launch_bounds__(kSceneThreads) scene_hist_kernel(const uint8_t* __restrict__ frames, int chunks,
                                                                  size_t npix, int* __restrict__ hist) {
  __shared__ int sh[kSceneBins];
  const int t = threadIdx.x, lane = t & 31;
  const int n = (int)(blockIdx.x / (unsigned)chunks), c = (int)(blockIdx.x % (unsigned)chunks);
  for (int b = t; b < kSceneBins; b += kSceneThreads) sh[b] = 0;
  const size_t c0 = (size_t)c * kSceneChunk;
  const uint8_t* src = frames + ((size_t)n * npix) * 3;
  int bins[kScenePerThread];
#pragma unroll
  for (int i = 0; i < kScenePerThread; ++i) {
    const size_t p = c0 + (size_t)i * kSceneThreads + t;
    bins[i] = -1;  // past the frame: a key no pixel has, never added
    if (p < npix) {
      const uint8_t* px = src + p * 3;
      bins[i] = ((__ldg(px) >> 5) << 6) | ((__ldg(px + 1) >> 5) << 3) | (__ldg(px + 2) >> 5);
    }
  }
  __syncthreads();  // sh zeroed
#pragma unroll
  for (int i = 0; i < kScenePerThread; ++i) {
    const unsigned peers = __match_any_sync(0xffffffffu, bins[i]);
    if (bins[i] >= 0 && lane == __ffs(peers) - 1) atomicAdd(&sh[bins[i]], __popc(peers));
  }
  __syncthreads();
  int* dst = hist + (size_t)n * kSceneBins;
  for (int b = t; b < kSceneBins; b += kSceneThreads)
    if (sh[b]) atomicAdd(dst + b, sh[b]);
}

// one block of RB_SCENE_BINS threads per pair k: thread b takes min(hist[k][b], hist[k+1][b]); the sum is exact in int
// (at most H*W < 2^31), and the score is the fp32 rounding of the exact-in-fp64 quotient (H*W - sum) / (H*W).
__global__ void __launch_bounds__(kSceneBins) scene_score_kernel(const int* __restrict__ hist, int npix,
                                                                float* __restrict__ scores) {
  __shared__ unsigned part[kSceneBins / 32];
  const int k = blockIdx.x, b = threadIdx.x;
  const int* h0 = hist + (size_t)k * kSceneBins;
  const unsigned m = (unsigned)min(h0[b], h0[kSceneBins + b]);
  const unsigned s = __reduce_add_sync(0xffffffffu, m);
  if ((b & 31) == 0) part[b >> 5] = s;
  __syncthreads();
  if (b == 0) {
    unsigned sum = 0;
#pragma unroll
    for (int w = 0; w < kSceneBins / 32; ++w) sum += part[w];
    scores[k] = (float)((double)(npix - (int)sum) / (double)npix);
  }
}

}  // namespace rb

using namespace rb;

extern "C" int rb_scene_cut_scores(const uint8_t* frames, int N, int H, int W, int32_t* hist, float* scores,
                                   void* stream) {
  RB_REQUIRE(frames && hist && scores, RB_ERR_BAD_ARG, "rb_scene_cut_scores: null pointer");
  RB_REQUIRE(N >= 2, RB_ERR_BAD_SHAPE, "rb_scene_cut_scores: a score needs two frames at least (N=%d)", N);
  RB_REQUIRE(H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_scene_cut_scores: bad shape N=%d H=%d W=%d", N, H, W);
  const size_t npix = (size_t)H * W;
  RB_REQUIRE(npix < (size_t(1) << 31), RB_ERR_BAD_SHAPE, "rb_scene_cut_scores: H*W = %zu must be < 2^31", npix);
  const size_t chunks = (npix + kSceneChunk - 1) / kSceneChunk;
  RB_REQUIRE((size_t)N * chunks <= 0x7fffffffu, RB_ERR_BAD_SHAPE,
             "rb_scene_cut_scores: N=%d frames of %zu pixels exceed one grid", N, npix);
  const cudaStream_t st = (cudaStream_t)stream;
  RB_CHECK_CUDA(cudaMemsetAsync(hist, 0, (size_t)N * kSceneBins * sizeof(int32_t), st));
  scene_hist_kernel<<<(unsigned)((size_t)N * chunks), kSceneThreads, 0, st>>>(frames, (int)chunks, npix, hist);
  RB_CHECK_LAUNCH("scene_hist_kernel");
  scene_score_kernel<<<N - 1, kSceneBins, 0, st>>>(hist, (int)npix, scores);
  RB_CHECK_LAUNCH("scene_score_kernel");
  return RB_OK;
}
