// wgmma implicit-GEMM convolution / GEMM over split fp16 operands (the RB_MATH_TC back end), and its single-pass variant
// over the hi planes only (RB_MATH_TC_FP16).
//
// One CTA computes a 128-pixel x BLOCK_N-channel output tile.  The 128 pixels are a BH x BW box of
// one image, so for every filter tap the A operand is ONE TMA box load from the NHWC activation
// at a shifted coordinate -- out-of-image pixels are zero-filled by TMA, which is exactly TF 'SAME'
// zero padding for the stride-1 odd kernels of the update block (SURVEY A14).  Per (tap, 64-channel
// chunk) a pipeline stage holds A_hi, A_lo (128x64 fp16 each) and B_hi, B_lo (BLOCK_N x 64 each),
// all 128-byte swizzled K-major.  Per 16-wide k-slice each consumer warpgroup issues
//     HH += A_hi x B_hi^T,   X += A_hi x B_lo^T,   X += A_lo x B_hi^T
// (m64nBLOCK_Nk16, fp32 accumulators in registers); the epilogue forms HH + 2^-11 * X in fp32 and applies the fused
// epilogue of common.cuh.
// SINGLE (RB_MATH_TC_FP16, ConvParams::single_pass): a stage holds A_hi and B_hi only, each k-slice issues HH += A_hi x B_hi^T
// alone, and the epilogue consumes HH -- fp16(a) * fp16(b) with fp32 accumulation, in the same K order.
// Warpgroup roles: 0 = TMA producer (one elected thread), 1 and 2 = consumers: wgmma on tile rows [0,64) / [64,128),
// then the epilogue of those rows.  The accumulator fragments are staged through shared memory in slabs of 32 columns
// so that every epilogue thread owns one pixel and 16 consecutive channels (the layout the epilogues and the fused
// instance-norm statistics are written for).
// Programmatic dependent launch: the prologue (barrier init, descriptor prefetch) and the first weight tiles run
// before griddepcontrol.wait, i.e. overlapped with the tail of the previous kernel in the stream.
#include <stdlib.h>
#include <unordered_map>
#include <string.h>

#include "tc_common.cuh"

namespace rb {
using namespace tc;

constexpr int kTileM = 128;
constexpr int kChunkK = 64;               // fp16 elements per 128-byte swizzled row
constexpr int kATileBytes = kTileM * 128;  // 16 KB
constexpr int kTcThreads = 384;            // 3 warpgroups: TMA producer, 2 x wgmma + epilogue
constexpr int kSlabCols = 32;              // epilogue staging: 64 rows x 32 fp32 columns per consumer warpgroup
constexpr int kSlabPitch = kSlabCols + 4;  // floats per staged row: 16-byte aligned rows, rows spread over the banks
constexpr int kStagingBytes = 2 * 64 * kSlabPitch * 4;
constexpr int kMaxSmem = 227 * 1024;       // opt-in shared memory per block on sm_90
// operand rings: everything but the alignment slack, the epilogue staging, the barriers and the split-K partials
constexpr int kRingBytes = kMaxSmem - 1024 /*align slack*/ - kStagingBytes - 256 /*barriers*/ - 1024 /*split-K partials*/;
constexpr int kSmemOverhead = 1024 + kStagingBytes + 256 + 1024;

// Halo A operand (ConvParams::halo, kh > 1): the A ring holds kHaloSlots slots of one (BH + kh - 1) x BW box (hi | lo)
// per (channel chunk, kx); the B ring holds one weight tile (hi | lo) per (chunk, kx, ky), as before.  Tap ky of the box is
// the rows [ky BW, ky BW + 128): a ky BW x 128-byte offset, a whole number of 1024-byte SW128 atoms for BW >= 8, so the
// wgmma descriptor is the canonical one at that address.  Two slots let the producer load the next group's halo while
// the consumers work through the current one (with one, the producer would wait for a release that needs its own load).
constexpr int kHaloSlots = 2;
// B ring depth next to the A ring: 0 when the two slots do not leave room for two B stages (the conv then keeps one
// A box per tap)
constexpr int halo_b_stages(int block_n, int planes, int halo_rows) {
  return (kRingBytes - kHaloSlots * planes * halo_rows * 128) / (planes * block_n * 128) < 2 ? 0
         : (kRingBytes - kHaloSlots * planes * halo_rows * 128) / (planes * block_n * 128) > 6
             ? 6
             : (kRingBytes - kHaloSlots * planes * halo_rows * 128) / (planes * block_n * 128);
}
// the geometries choose_geom picks for the update block at 55 x 128 (3x3 and 5x1 on 8 x 16 boxes), the 2 x 64 / 4 x 32
// boxes, and the widest tile
static_assert(halo_b_stages(128, 2, 10 * 16) == 3 && halo_b_stages(128, 2, 12 * 16) == 3, "3x3 / 5x1 halo at N = 128");
static_assert(halo_b_stages(96, 2, 10 * 16) == 5 && halo_b_stages(96, 2, 12 * 16) == 4, "3x3 / 5x1 halo at N = 96");
static_assert(halo_b_stages(128, 2, 4 * 64) == 2 && halo_b_stages(128, 2, 8 * 32) == 2, "2x64 3x3 / 4x32 5x1 halo at N = 128");
static_assert(halo_b_stages(128, 2, 3 * 128) == 0, "a 1x128 3x3 halo does not fit beside two N = 128 stages");

// PERSISTENT kernel: each CTA walks tiles t = blockIdx.x, blockIdx.x + gridDim.x, ... (n-tile fastest, so CTAs that
// run side by side share the same activation tile in L2).  The smem ring and its mbarrier phases simply continue across
// tiles, so the producer streams the next tile's operands while the consumers run the epilogue of the current one.
template <int BLOCK_N, bool SINGLE = false>
struct TcCfg {
  static constexpr int kBTileBytes = BLOCK_N * 128;
  static constexpr int kPlanes = SINGLE ? 1 : 2;          // hi (| lo) per operand
  static constexpr int kBOff = kPlanes * kATileBytes;      // B_hi inside a stage: A_hi | A_lo | B_hi | B_lo, or A_hi | B_hi
  static constexpr int kStageBytes = kPlanes * (kATileBytes + kBTileBytes);
  static constexpr int kStages = kRingBytes / kStageBytes > 6 ? 6 : kRingBytes / kStageBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + kSmemOverhead;
  static constexpr int kSlab = BLOCK_N < kSlabCols ? BLOCK_N : kSlabCols;  // columns staged at a time
  static constexpr int kAcc = BLOCK_N / 2;  // fp32 accumulator registers per thread and accumulator
};

__device__ __forceinline__ void consumer_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// EXTRAS: phase timestamps (p.dbg) and fused instance-norm statistics (p.stat_part) -- a separate instantiation, so that
// the kernel the update block runs carries none of their registers.
// SINGLE: the single-pass variant (tmA_lo / tmB_lo are not read).
// HALO: the halo A operand (g.halo_rows > 0) -- a separate instantiation, so that the one-box-per-tap kernel of every
// other conv carries none of its ring bookkeeping.
template <int BLOCK_N, bool EXTRAS, bool SINGLE, bool HALO>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
               const ConvParams p, const TileGeom g, const int STAGES) {
  using Cfg = TcCfg<BLOCK_N, SINGLE>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // STAGES: depth of the B ring (one A | B stage per k-iteration without the halo).  Layout: [A slots] B ring | staging |
  // barriers | split-K partials.
  constexpr bool halo = HALO;
  const int a_plane = halo ? g.halo_rows * 128 : kATileBytes;  // A_lo behind A_hi
  const int a_slot_bytes = Cfg::kPlanes * a_plane;
  const int b_stage_bytes = halo ? Cfg::kPlanes * Cfg::kBTileBytes : Cfg::kStageBytes;
  const int b_off = halo ? 0 : Cfg::kBOff;  // B_hi inside a stage
  uint8_t* bring = smem + (halo ? kHaloSlots * a_slot_bytes : 0);
  float* staging = reinterpret_cast<float*>(smem + g.ring_bytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + g.ring_bytes + kStagingBytes);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* a_full = empty_bar + STAGES;   // halo: A slot loaded / released by both consumer warpgroups
  uint64_t* a_empty = a_full + kHaloSlots;
  uint64_t* red_bar = a_empty + kHaloSlots;  // split-K: the peer's partial sums have arrived (128 pixel arrivals)
  float2* red_buf = reinterpret_cast<float2*>(smem + g.ring_bytes + kStagingBytes + 256);  // [128 pixels] ch 0, 1

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  long long* dbg = (EXTRAS && p.dbg) ? p.dbg + (size_t)blockIdx.x * 8 : nullptr;
  const bool wide = epilogue_wide_ok(p);
  if (dbg && threadIdx.x == 0) dbg[0] = gtime_ns();
  // Split-K (p.split_k, 16-wide tiles with <= 2 real channels: the flow head's last conv, update.cu).  The sum over K is
  // ALWAYS formed as (first half of the channel chunks) + (second half), each half in its own accumulator, so that the
  // result does not depend on how it is executed:
  //  * p.split_cluster = 1 (one wave of CTA pairs, batch 1): clusters of two CTAs share one pixel tile, CTA r multiplies
  //    half r; CTA 1 hands its partial sums to CTA 0 through distributed shared memory, CTA 0 runs the epilogue on r0 + r1;
  //  * else one CTA runs both halves back to back into two accumulators and its epilogue adds them the same way.
  const bool halves = BLOCK_N == 16 && p.split_k;
  const bool splitk = halves && p.split_cluster;
  const int chunks = splitk ? conv_chunks(p) / 2 : conv_chunks(p);
  const int taps = p.kh * p.kw;
  const int kiters = taps * chunks;
  const int tiles_per_img = g.tiles_x * g.tiles_y;

  if (threadIdx.x == 0) {
    if constexpr (SINGLE) {
      prefetch_tmap(&tmA_hi); prefetch_tmap(&tmB_hi);
    } else {
      prefetch_tmap(&tmA_hi); prefetch_tmap(&tmA_lo); prefetch_tmap(&tmB_hi); prefetch_tmap(&tmB_lo);
    }
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }  // one arrival per consumer warpgroup
    for (int s = 0; s < kHaloSlots; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 2); }
    mbar_init(red_bar, 128);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncthreads();
  if (splitk) cluster_sync_all();  // the peer's barriers must be initialised before anything of ours can reach them
  const int krank = splitk ? (int)cluster_ctarank() : 0;
  const int first = splitk ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;  // first work item of this CTA (pair)
  const int stride = splitk ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  if (dbg && threadIdx.x == 0) dbg[1] = gtime_ns();
  // Programmatic dependent launch: this kernel may have been started while its predecessor is still running.  Everything
  // up to here and the WEIGHT tiles of the first ring stages are independent of it; `griddepcontrol.wait` (no-op without
  // the launch attribute) is executed by the producer before its first activation load and by the consumers before
  // their first global access.

  if (warp < 4) {
    if (warp == 0 && elect_one()) {
      const int ph = conv_pad_y(p), pw = conv_pad_x(p), csx = conv_sx(p), csy = conv_sy(p);
      int s = 0;          // ring slot and its phase; both continue across tiles.  No integer division in this loop:
      uint32_t phase = 0;  // the k-iteration -> (chunk, kx, ky) mapping is advanced incrementally.
      int as = 0;            // halo: A slot and its phase, likewise
      uint32_t a_phase = 0;
      bool waited = false;
      for (int tile = first; tile < g.total_tiles; tile += stride) {
        const int mt = tile / g.n_tiles, nt = tile - mt * g.n_tiles;
        const int b = mt / tiles_per_img, trem = mt - b * tiles_per_img;
        const int ty = trem / g.tiles_x, tx = trem - ty * g.tiles_x;
        const int y0 = ty << g.bh_log2, x0 = tx << g.bw_log2, n0 = nt * BLOCK_N;
        const int xs = x0 * csx - pw, ys = y0 * csy - ph;  // input coordinates of tap (0, 0) of the tile's first pixel
        const int wb = p.w_per_batch ? min(b, p.B - 1) : 0;
        // K order: channel chunk outermost, then kx, then ky, whatever the tile geometry, so that a batched run equals
        // the per-sample runs bit for bit.
        struct KIter {
          int cki, kx, ky, ck;
        };
        auto k_next = [&](KIter& k) {
          if (++k.ky == p.kh) {
            k.ky = 0;
            if (++k.kx == p.kw) { k.kx = 0; k.ck = conv_chunk(p, ++k.cki); }
          }
        };
        auto load_a = [&](const KIter& k, int slot) {
          uint8_t* st = smem + slot * Cfg::kStageBytes;
          const int c0 = p.in_choff + k.ck * kChunkK;
          tma_load_4d(&tmA_hi, &full_bar[slot], st, c0, xs + k.kx, ys + k.ky, b);
          if constexpr (!SINGLE) tma_load_4d(&tmA_lo, &full_bar[slot], st + kATileBytes, c0, xs + k.kx, ys + k.ky, b);
        };
        auto load_b = [&](const KIter& k, int slot) {
          uint8_t* st = bring + slot * b_stage_bytes + b_off;
          const int kcol = (k.ky * p.kw + k.kx) * p.cin_pad + k.ck * kChunkK;
          tma_load_3d(&tmB_hi, &full_bar[slot], st, kcol, n0, wb);
          if constexpr (!SINGLE) tma_load_3d(&tmB_lo, &full_bar[slot], st + Cfg::kBTileBytes, kcol, n0, wb);
        };
        // halo: the (BH + kh - 1) x BW box of all kh taps of (chunk, kx), from input row ys (TMA zero fill = SAME padding)
        auto load_halo = [&](const KIter& k, int slot) {
          uint8_t* st = smem + slot * a_slot_bytes;
          const int c0 = p.in_choff + k.ck * kChunkK;
          tma_load_4d(&tmA_hi, &a_full[slot], st, c0, xs + k.kx, ys, b);
          if constexpr (!SINGLE) tma_load_4d(&tmA_lo, &a_full[slot], st + a_plane, c0, xs + k.kx, ys, b);
        };
        KIter k = {krank * chunks, 0, 0, conv_chunk(p, krank * chunks)};
        int it0 = 0;
        if (!waited) {
          // first tile of the kernel: weight tiles of the first ring stages, then wait for the predecessor kernel, then
          // the activation tiles of the same stages (the ring is empty here: slots 0.., phase 0)
          // (not when the B operand is itself an activation produced by an earlier kernel: corr build, w_per_batch)
          // (halo: the B stages only; the halo boxes follow in the loop below)
          const int pre = p.w_per_batch ? 0 : (kiters < STAGES ? kiters : STAGES);
          KIter kb = k;
          for (int it = 0; it < pre; ++it) {
            mbar_arrive_expect_tx(&full_bar[it], b_stage_bytes);
            load_b(kb, it);
            k_next(kb);
          }
          asm volatile("griddepcontrol.wait;" ::: "memory");
          if (dbg) dbg[2] = gtime_ns();
          if (!halo) {
            for (int it = 0; it < pre; ++it) {
              load_a(k, s);
              k_next(k);
              if (++s == STAGES) { s = 0; phase ^= 1; }
            }
          }
          it0 = pre;
          waited = true;
        }
        if constexpr (halo) {
          // per (chunk, kx): one halo box into the A ring, then the kh weight tiles into the B ring (those of the first
          // it0 k-iterations are already in flight)
          for (int it = 0; it < kiters; ++it) {
            if (k.ky == 0) {
              mbar_wait(&a_empty[as], a_phase ^ 1);
              mbar_arrive_expect_tx(&a_full[as], a_slot_bytes);
              load_halo(k, as);
            }
            if (it >= it0) {
              mbar_wait(&empty_bar[s], phase ^ 1);
              mbar_arrive_expect_tx(&full_bar[s], b_stage_bytes);
              load_b(k, s);
            }
            const bool group_end = k.ky == p.kh - 1;
            k_next(k);
            if (++s == STAGES) { s = 0; phase ^= 1; }
            if (group_end && ++as == kHaloSlots) { as = 0; a_phase ^= 1; }
          }
        } else {
          for (int it = it0; it < kiters; ++it) {
            mbar_wait(&empty_bar[s], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
            load_a(k, s);
            load_b(k, s);
            k_next(k);
            if (++s == STAGES) { s = 0; phase ^= 1; }
          }
        }
      }
    }
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  } else {
    // ---- consumers: warpgroup cw = 0, 1 owns tile rows [64 cw, 64 cw + 64) ----
    const int cw = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127;
    const int wi = t >> 5;                   // warp inside the warpgroup: fragment rows 16 wi + lane/4 + {0, 8}
    // Epilogue lanes.  Default: thread t owns pixel t % 64 and the 16 columns [16 h, 16 h + 16) of a 32-column slab,
    // h = t / 64 -- one pixel per lane, the layout of the fused instance-norm statistics (32 pixels per warp).
    // PAIRED (every other 16-channel epilogue): lanes 2i, 2i + 1 own pixel i of the warpgroup's 64 and the 8-column groups
    // {8 h, 16 + 8 h} of the slab, h = t % 2, so that each 16-byte fp16 store of a lane pair fills a whole 32-byte sector
    // instead of half of one (the split-plane stores are most of the epilogue's memory traffic).  Same arithmetic per
    // element.  Needs whole 32-channel slabs: cout, and hidden of the GRU epilogues, multiples of 32.
    const bool paired = BLOCK_N >= 32 && wide && (p.cout & 31) == 0 && !(EXTRAS && p.stat_part) &&
                        ((p.epi != EPI_ZR && p.epi != EPI_Q) || (p.hidden & 31) == 0);
    const int prow = paired ? (t >> 1) : (t & 63);  // pixel of this lane among the warpgroup's 64 tile rows
    const int r = 64 * cw + prow;            // epilogue: tile row = pixel index inside the box
    const int half = paired ? (t & 1) : (t >> 6);  // epilogue: 16-column half (paired: 8-column groups) of a staged slab
    const int gofs = paired ? 8 : 16;        // column of this lane's first group inside the slab: gofs * half
    const int gsep = paired ? 16 : 8;        // columns between its two 8-column groups
    float* stg = staging + cw * 64 * kSlabPitch;
    asm volatile("griddepcontrol.wait;" ::: "memory");  // addend / z / h reads and all stores come after the predecessor
    constexpr int kNumAcc = BLOCK_N == 16 ? 2 : 1;  // the split-K halves of a 16-wide tile on one CTA
    float hh[kNumAcc][Cfg::kAcc], xx[kNumAcc][SINGLE ? 1 : Cfg::kAcc];  // SINGLE: no cross-term accumulators
    int s = 0, pend = -1, li = 0;
    uint32_t phase = 0;
    int as = 0, apend = -1, ky = 0;  // halo: A slot, the slot to hand back after the next wgmma_wait<1>, tap row
    uint32_t a_phase = 0;
    // k-iterations [it0, it1) into (H, X); the wgmma group of a stage stays in flight while the next stage is issued, the
    // stage before it is handed back to the producer
    auto mma_range = [&](float* H, float* X, int it0, int it1) {
      for (int it = it0; it < it1; ++it) {
        if (halo && ky == 0) mbar_wait(&a_full[as], a_phase);
        mbar_wait(&full_bar[s], phase);
        if (dbg && li == 0 && it == 0 && t == 0) dbg[3] = gtime_ns();
        const uint32_t st = smem_u32(bring + s * b_stage_bytes);
        // halo: tap row ky starts ky box rows into the slot
        const uint32_t sa = halo ? smem_u32(smem + as * a_slot_bytes) + ((uint32_t)ky << g.bw_log2) * 128u : st;
        const uint64_t a_hi = wgmma_desc_sw128(sa + cw * 64 * 128);
        const uint64_t a_lo = wgmma_desc_sw128(sa + a_plane + cw * 64 * 128);
        const uint64_t b_hi = wgmma_desc_sw128(st + b_off);
        const uint64_t b_lo = wgmma_desc_sw128(st + b_off + Cfg::kBTileBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kChunkK / 16; ++k) {
          const uint64_t koff = (uint64_t)(k * 2);  // 32 bytes per k-slice, in 16-byte units
          wgmma_f16<BLOCK_N>(H, a_hi + koff, b_hi + koff);
          if constexpr (!SINGLE) {
            wgmma_f16<BLOCK_N>(X, a_hi + koff, b_lo + koff);
            wgmma_f16<BLOCK_N>(X, a_lo + koff, b_hi + koff);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (pend >= 0 && t == 0) mbar_arrive(&empty_bar[pend]);
        if (apend >= 0 && t == 0) mbar_arrive(&a_empty[apend]);
        apend = -1;
        pend = s;
        if (++s == STAGES) { s = 0; phase ^= 1; }
        if (halo && ++ky == p.kh) {  // the group's last tap: its slot goes back once this wgmma group has completed
          ky = 0;
          apend = as;
          if (++as == kHaloSlots) { as = 0; a_phase ^= 1; }
        }
      }
    };
    for (int tile = first; tile < g.total_tiles; tile += stride, ++li) {
      const int mt = tile / g.n_tiles, nt = tile - mt * g.n_tiles;
      const int b = mt / tiles_per_img, trem = mt - b * tiles_per_img;
      const int ty = trem / g.tiles_x, tx = trem - ty * g.tiles_x;
      const int y0 = ty << g.bh_log2, x0 = tx << g.bw_log2, n0 = nt * BLOCK_N;
      const int py = y0 + (r >> g.bw_log2), px = x0 + (r & ((1 << g.bw_log2) - 1));
      const bool valid = (py < p.h) && (px < p.w) && (mt < g.m_tiles);
      const int pix = (b * p.h + py) * p.w + px;
#pragma unroll
      for (int a = 0; a < kNumAcc; ++a)
#pragma unroll
        for (int i = 0; i < Cfg::kAcc; ++i) {
          hh[a][i] = 0.f;
          fence_operand(hh[a][i]);  // zeroed before the first wgmma, not between stages
          if constexpr (!SINGLE) { xx[a][i] = 0.f; fence_operand(xx[a][i]); }
        }
      const int it_half = (halves && !splitk) ? kiters / 2 : kiters;  // first k-iteration of the second accumulator
      mma_range(hh[0], xx[0], 0, it_half);
      if constexpr (BLOCK_N == 16) mma_range(hh[1], xx[1], it_half, kiters);
      wgmma_wait<0>();
#pragma unroll
      for (int a = 0; a < kNumAcc; ++a)
#pragma unroll
        for (int i = 0; i < Cfg::kAcc; ++i) {
          fence_operand(hh[a][i]);
          if constexpr (!SINGLE) fence_operand(xx[a][i]);
        }
      if (t == 0) mbar_arrive(&empty_bar[pend]);
      if (apend >= 0 && t == 0) mbar_arrive(&a_empty[apend]);
      pend = -1;
      apend = -1;
      if (li == 0) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        if (dbg && t == 0 && cw == 0) dbg[4] = gtime_ns();
      }
      if (dbg && li == 0 && t == 0 && cw == 0) dbg[5] = gtime_ns();  // epilogue of the first tile begins
#pragma unroll
      for (int i = 0; i < Cfg::kAcc; ++i) {
        if constexpr (SINGLE) {
          if constexpr (BLOCK_N == 16) {
            if (halves && !splitk) hh[0][i] += hh[1][i];  // second accumulator of the same CTA
          }
        } else {
          hh[0][i] = hh[0][i] + xx[0][i] * kLoInv;
          if constexpr (BLOCK_N == 16) {
            if (halves && !splitk) hh[0][i] += hh[1][i] + xx[1][i] * kLoInv;  // second accumulator of the same CTA
          }
        }
      }
#pragma unroll
      for (int c0 = 0; c0 < BLOCK_N; c0 += Cfg::kSlab) {
        // fragments of columns [c0, c0 + kSlab) -> staging rows
        const int row = 16 * wi + (lane >> 2), col = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < Cfg::kSlab / 8; ++j) {
          const int i = (c0 / 8 + j) * 4;
          *reinterpret_cast<float2*>(stg + row * kSlabPitch + 8 * j + col) = make_float2(hh[0][i], hh[0][i + 1]);
          *reinterpret_cast<float2*>(stg + (row + 8) * kSlabPitch + 8 * j + col) = make_float2(hh[0][i + 2], hh[0][i + 3]);
        }
        consumer_bar_sync(1 + cw);
        if (Cfg::kSlab == 32 || half == 0) {  // warp-uniform
          const int c = c0 + gofs * half;  // first column of this lane (multiple of 8; 16 when not paired)
          float v[16];
          const float* srow = stg + prow * kSlabPitch + c - c0;
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const float4 f = *reinterpret_cast<const float4*>(srow + (q4 >> 1) * gsep + 4 * (q4 & 1));
            v[4 * q4] = f.x; v[4 * q4 + 1] = f.y; v[4 * q4 + 2] = f.z; v[4 * q4 + 3] = f.w;
          }
          bool store = valid && n0 + c < p.cout;
          if constexpr (BLOCK_N == 16) {
            if (splitk) {
              if (krank != 0) {  // partial sums of channels 0, 1 -> CTA 0 of the cluster; nothing else to do here
                st_cluster_f32x2(mapa_u32(smem_u32(red_buf + r), 0), v[0], v[1]);
                mbar_arrive_remote(mapa_u32(smem_u32(red_bar), 0));
                store = false;
              } else {
                mbar_wait_cluster(red_bar, 0);
                const float2 pr = red_buf[r];
                v[0] += pr.x;
                v[1] += pr.y;
              }
            }
          }
          if (store) {
            if (wide) {
              epilogue_wide16(p, pix, n0 + c, n0 + c + gsep, v);
            } else {
              epilogue_store<8>(p, pix, n0 + c, v);
              epilogue_store<8>(p, pix, n0 + c + 8, v + 8);
            }
          }
          if (EXTRAS && p.stat_part && n0 + c < p.cout) {  // instance-norm statistics of the values just stored (v was finalised in place; host: wide only)
            if (!valid) {
#pragma unroll
              for (int i = 0; i < 16; ++i) v[i] = 0.f;
            }
            double s1, s2;
            int ch;
            warp_stats16(v, s1, s2, ch);
            if ((lane & 1) == 0 && mt < g.m_tiles) {
              double* dst = p.stat_part + ((size_t)(b * p.stat_strips + trem * 4 + (r >> 5)) * 2) * p.cout + n0 + c + ch;
              dst[0] = s1;
              dst[p.cout] = s2;
            }
          }
        }
        consumer_bar_sync(1 + cw);  // the slab is overwritten next
      }
    }
    if (dbg && t == 0 && cw == 0) dbg[6] = gtime_ns();
  }
  __syncthreads();
  // Split-K: CTA 0 cannot exit before CTA 1's partial sums have landed in its shared memory -- it waited for them
  // (mbarrier, release.cluster / acquire.cluster) -- so no closing cluster barrier is needed.  compute-sanitizer's racecheck
  // cannot see that ("block that might have already exited"); p.split_close adds the barrier it wants.
  if (splitk && p.split_close) cluster_sync_all();
  if (dbg && threadIdx.x == 0) dbg[7] = gtime_ns();
}

// ---- host side -------------------------------------------------------------------------------------
namespace tc {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, int kind, const uint32_t* elem_strides) {
  EncodeTiledFn fn = encode_fn();
  RB_REQUIRE(fn, RB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = elem_strides ? elem_strides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  const CUtensorMapDataType dt = kind == TMAP_F16_SW128 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const CUtensorMapSwizzle sw = kind == TMAP_F16_SW128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = fn(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RB_REQUIRE(r == CUDA_SUCCESS, RB_ERR_CUDA,
             "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu,%llu] box [%u,%u,%u,%u]", (int)r, rank,
             (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
             rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
  return RB_OK;
}
}  // namespace tc

// Tensor maps depend only on (pointer, geometry); cache them per thread so steady-state launches
// (and CUDA-graph capture, which bakes kernel parameters) pay nothing for the encode.
struct TmapKey {
  const void* base;
  uint64_t kind;
  uint64_t d[4];
  uint64_t s[4];
  uint32_t b[4];
  uint32_t e[4];
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    size_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) h = (h ^ w[i]) * 1099511628211ull;
    return h;
  }
};

int cached_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                const uint32_t* box, int kind, const uint32_t* elem_strides) {
  static thread_local std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  TmapKey k;
  memset(&k, 0, sizeof(k));
  k.base = base;
  k.kind = (uint64_t)kind;
  for (int i = 0; i < rank; ++i) {
    k.d[i] = dims[i]; k.s[i] = (i + 1 < rank) ? strides[i] : 0; k.b[i] = box[i]; k.e[i] = elem_strides ? elem_strides[i] : 1;
  }
  auto it = cache.find(k);
  if (it != cache.end()) { *out = it->second; return RB_OK; }
  int rc = make_tmap(out, base, rank, dims, strides, box, kind, elem_strides);
  if (rc) return rc;
  if (cache.size() > 4096) cache.clear();
  cache.emplace(k, *out);
  return RB_OK;
}

// Test hook (rb_debug_conv_override / rb_debug_conv_last): a forced configuration and the record of the last launch, per
// thread.  0 = automatic.
struct ConvOverride {
  int block_n, bw_log2, max_ctas, stages;
};
struct ConvRecord {
  int block_n, bw_log2, grid, stages, total_tiles;
  int launched;     // a tensor-core conv has been launched on this thread
  int fused_stats;  // convs since the last rb_debug_conv_override() call that wrote fused instance-norm statistics
  int passes;       // wgmma per product: 3 (split operands) or 1 (single pass)
};
static thread_local ConvOverride g_override = {0, 0, 0, 0};
static thread_local ConvRecord g_record = {0, 0, 0, 0, 0, 0, 0, 0};
// Test hook (rb_debug_conv_halo): -1 = no conv uses the halo A operand, 0 = as ConvParams::halo says, 1 = every conv
// that can.  And the launch log of rb_debug_conv_log: the first kLogLen launches since the last rb_debug_conv_override().
static thread_local int g_halo_mode = 0;
constexpr int kLogLen = 64, kLogFields = 10;
static thread_local int g_log[kLogLen][kLogFields];
static thread_local int g_log_n = 0;

// Ring depth of a launch: the test hook may lower it, but never below 2 -- a consumer hands a stage back only after it has
// issued the next one (wgmma_wait<1>), so a one-stage ring deadlocks any conv with two k-iterations.
static int ring_stages(int max_stages) {
  const int req = g_override.stages;
  if (req <= 0) return max_stages;
  return req < 2 ? 2 : req > max_stages ? max_stages : req;
}

// halo_kh > 1: a conv with the halo A operand.  Every geometry streams the same weight tiles per pixel tile, and the
// classic rule (fewest tiles) picks one-row boxes, whose halo is as large as the kh per-tap boxes it replaces; so these
// convs take the box with the fewest rows streamed per (chunk, kx) over the whole image: the tiles times the
// (BH + kh - 1) x BW halo plus kh weight tiles of up to 128 rows.  At 55 x 128 that is 8 x 16 (56 tiles against 55) for
// 3x3 and 5x1 alike.
static TileGeom choose_geom(int h, int w, int halo_kh = 0) {
  TileGeom best{};
  if (g_override.bw_log2 > 0) {
    const int bwl = g_override.bw_log2, bw = 1 << bwl, bh = kTileM >> bwl;
    best.bw_log2 = bwl; best.bh_log2 = 7 - bwl;
    best.tiles_x = (w + bw - 1) / bw; best.tiles_y = (h + bh - 1) / bh;
    return best;
  }
  long best_tiles = -1;
  for (int bwl = 7; bwl >= 3; --bwl) {
    int bw = 1 << bwl, bh = kTileM >> bwl;
    if (bw > w && bwl > 3) continue;  // keep the box inside the row when possible
    long tiles = (long)((w + bw - 1) / bw) * ((h + bh - 1) / bh);
    if (halo_kh > 1) tiles *= (long)((bh + halo_kh - 1) << bwl) + halo_kh * 128;  // rows streamed per (chunk, kx)
    if (best_tiles < 0 || tiles < best_tiles) {
      best_tiles = tiles;
      best.bw_log2 = bwl; best.bh_log2 = 7 - bwl;
      best.tiles_x = (w + bw - 1) / bw; best.tiles_y = (h + bh - 1) / bh;
    }
  }
  return best;
}

// Pixel tiles per image of the tensor-core conv (strip count of the fused instance-norm statistics = 4x this).
int conv_tc_tiles_per_image(int h, int w) {
  const TileGeom g = choose_geom(h, w);
  return g.tiles_x * g.tiles_y;
}
// The conv can produce the statistics itself: tensor-core back end, 16-channel epilogue (see epilogue_wide_ok()).
bool conv_tc_fused_stats_ok(const ConvParams& p) {
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 31) == 0; };
  return math_mode_tc() && p.epi == EPI_F32 && (p.cout & 15) == 0 && al(p.bias) && al(p.addend) && al(p.f0) &&
         p.cin_pad % kChunkK == 0;
}

// relative cost of a 16-wide k-slice of an n-wide tile: max(tensor math, shared-memory operand reads) -- a heuristic that
// only ranks tile widths against the wave count.  Its constants are carried over from the B200 version of this kernel and
// have not been re-measured on H100 (only the wave count uses the device's SM count).
static int slice_cycles(int n) {
  int math = n + n / 2;
  int smem = 64 + (3 * n) / 4;
  return math > smem ? math : smem;
}

static int choose_block_n(int cout, long m_tiles, int ctas) {  // ctas: persistent CTAs the launch may use (SMs or cta_limit)
  if (cout <= 16) return 16;
  const int cand[4] = {128, 96, 64, 32};
  int best = 128;
  long best_cost = -1;
  for (int i = 0; i < 4; ++i) {
    int n = cand[i];
    long tiles = m_tiles * ((cout + n - 1) / n);
    long waves = (tiles + ctas - 1) / ctas;
    long cost = waves * slice_cycles(n);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = n; }
  }
  return best;
}

template <int BLOCK_N, bool SINGLE>
static int launch_cfg(const ConvParams& p_in, TileGeom g, const CUtensorMap* maps, cudaStream_t s) {
  using Cfg = TcCfg<BLOCK_N, SINGLE>;
  int dev = 0, rc;
  if ((rc = current_device(&dev))) return rc;
  const int num_sms = device_sm_count(dev);
  ConvParams p = p_in;
  g.n_tiles = (p.cout + BLOCK_N - 1) / BLOCK_N;
  g.m_tiles = p.B * g.tiles_x * g.tiles_y;
  g.total_tiles = g.m_tiles * g.n_tiles;
  // split-K: only when every pixel tile gets its own CTA pair in one wave (batch 1), else the plain persistent grid
  if (p.split_k && !(BLOCK_N == 16 && p.cout <= 2 && p.epi == EPI_DELTA && !p.w_per_batch && conv_chunks(p) % 2 == 0))
    p.split_k = 0;
  static const bool close_barrier = getenv("RAFT_B200_SPLITK_CLOSING_BARRIER") != nullptr;  // for compute-sanitizer runs
  p.split_close = close_barrier ? 1 : 0;
  const int max_ctas = g_override.max_ctas;  // test hook: a capped grid walks more tiles per CTA (no CTA pairs then)
  p.split_cluster = (p.split_k && 2 * g.total_tiles <= num_sms && p.cta_limit <= 0 && max_ctas <= 0) ? 1 : 0;
  const bool cluster2 = p.split_cluster;
  int units = cluster2 ? num_sms / 2 : num_sms;  // persistent: at most one CTA (pair) per SM (pair)
  if (!cluster2 && p.cta_limit > 0 && p.cta_limit < units) units = p.cta_limit;  // leave SMs to a concurrent conv (update.cu)
  if (max_ctas > 0 && max_ctas < units) units = max_ctas;
  const dim3 grid((g.total_tiles < units ? g.total_tiles : units) * (cluster2 ? 2 : 1));
  // halo: a B ring beside the kHaloSlots A slots; a forced ring depth applies to the B ring (the A ring stays at two)
  const int stages = ring_stages(g.halo_rows ? halo_b_stages(BLOCK_N, Cfg::kPlanes, g.halo_rows) : Cfg::kStages);
  g.ring_bytes = g.halo_rows ? kHaloSlots * Cfg::kPlanes * g.halo_rows * 128 + stages * Cfg::kPlanes * Cfg::kBTileBytes
                             : stages * Cfg::kStageBytes;
  const int smem = g.halo_rows ? g.ring_bytes + kSmemOverhead : Cfg::kSmemBytes;
  // Programmatic dependent launch: the dependent conv's prologue and its first weight tiles overlap the tail of this one.
  // Both EXTRAS instantiations get their shared-memory limit at the first launch of either.
  constexpr auto plain = conv_tc_kernel<BLOCK_N, false, SINGLE, false>;
  constexpr auto extras = conv_tc_kernel<BLOCK_N, true, SINGLE, false>;
  constexpr auto plain_halo = conv_tc_kernel<BLOCK_N, false, SINGLE, true>;
  constexpr auto extras_halo = conv_tc_kernel<BLOCK_N, true, SINGLE, true>;
  const int cluster = cluster2 ? 2 : 1;
  if (!g.halo_rows) {
    if (p.dbg || p.stat_part)
      rc = launch_pdl<extras, plain>(grid, dim3(kTcThreads), smem, cluster, s, maps[0], maps[1], maps[2], maps[3], p, g, stages);
    else
      rc = launch_pdl<plain, extras>(grid, dim3(kTcThreads), smem, cluster, s, maps[0], maps[1], maps[2], maps[3], p, g, stages);
  } else {
    // the halo layouts take up to the whole ring budget: the limit is raised to it, for both instantiations, at the first
    // launch of either
    if ((rc = set_max_dyn_smem<plain_halo>(dev, kMaxSmem)) || (rc = set_max_dyn_smem<extras_halo>(dev, kMaxSmem))) return rc;
    if (p.dbg || p.stat_part)
      rc = launch_pdl<extras_halo>(grid, dim3(kTcThreads), smem, cluster, s, maps[0], maps[1], maps[2], maps[3], p, g, stages);
    else
      rc = launch_pdl<plain_halo>(grid, dim3(kTcThreads), smem, cluster, s, maps[0], maps[1], maps[2], maps[3], p, g, stages);
  }
  if (rc) return rc;
  RB_CHECK_LAUNCH("conv_tc_kernel");
  g_record.block_n = BLOCK_N; g_record.bw_log2 = g.bw_log2; g_record.grid = (int)grid.x; g_record.stages = stages;
  g_record.total_tiles = g.total_tiles; g_record.launched = 1; g_record.passes = SINGLE ? 1 : 3;
  if (p.stat_part) ++g_record.fused_stats;
  if (g_log_n < kLogLen) {
    const int rec[kLogFields] = {BLOCK_N, g.bw_log2, (int)grid.x, stages, g.total_tiles, g.halo_rows, p.kh, p.kw,
                                 conv_chunks(p), SINGLE ? 1 : 3};
    memcpy(g_log[g_log_n++], rec, sizeof(rec));
  }
  return RB_OK;
}

int launch_conv_tc(const ConvParams& p, cudaStream_t s) {
  RB_REQUIRE(p.cin_pad % kChunkK == 0 && p.in_stride % 8 == 0 && p.in_choff % 8 == 0, RB_ERR_BAD_SHAPE,
             "conv_tc: channel padding (cin_pad=%d stride=%d off=%d)", p.cin_pad, p.in_stride, p.in_choff);
  // the halo A operand: stride-1 convs over the default view with a vertical filter extent (not the split-K pair)
  const bool want_halo = (g_halo_mode > 0 || (g_halo_mode == 0 && p.halo)) && p.kh > 1 && conv_default_view(p) &&
                         !p.w_per_batch && !p.split_k;
  TileGeom g = choose_geom(p.h, p.w, want_halo ? p.kh : 0);
  const long m_tiles = (long)p.B * g.tiles_x * g.tiles_y;
  int dev = 0, rc_dev;
  if ((rc_dev = current_device(&dev))) return rc_dev;
  const int num_sms = device_sm_count(dev);
  int bn = choose_block_n(p.cout, m_tiles, p.cta_limit > 0 && p.cta_limit < num_sms ? p.cta_limit : num_sms);
  if (g_override.block_n > 0 && bn != 16) bn = g_override.block_n;  // the 16-wide (split-K) convs keep theirs
  const bool single = p.single_pass != 0;
  g.halo_rows = 0;
  if (want_halo) {  // one A box per tap when the halo box is too tall for TMA or the two slots leave no room for the B ring
    const int box_h = (1 << g.bh_log2) + p.kh - 1, rows = box_h << g.bw_log2;
    if (box_h <= 256 && halo_b_stages(bn, single ? 1 : 2, rows) >= 2) g.halo_rows = rows;
  }
  CUtensorMap maps[4];
  {
    // the input view (common.cuh): strided convs traverse it with TMA element strides -- a box of bw*sx x bh*sy input
    // pixels delivers every sx-th / sy-th one, i.e. the bw x bh taps of the output tile
    const int iw = conv_in_w(p), ih = conv_in_h(p), sx = conv_sx(p), sy = conv_sy(p);
    const uint64_t rowpitch = (uint64_t)conv_rowpitch(p);
    RB_REQUIRE(sx <= 2 && sy <= 2 && rowpitch % 8 == 0, RB_ERR_BAD_SHAPE, "conv_tc: stride (%d,%d) / row pitch %llu", sx, sy,
               (unsigned long long)rowpitch);
    uint64_t dims[4] = {(uint64_t)(p.in_cext > 0 ? p.in_cext : p.in_stride), (uint64_t)iw, (uint64_t)ih, (uint64_t)p.B};
    uint64_t str[3] = {(uint64_t)p.in_stride * 2, rowpitch * 2, rowpitch * 2 * ih};
    const uint32_t box_h = g.halo_rows ? (uint32_t)(g.halo_rows >> g.bw_log2) : (1u << g.bh_log2) * sy;
    uint32_t box[4] = {(uint32_t)kChunkK, (1u << g.bw_log2) * sx, box_h, 1};
    uint32_t es[4] = {1, (uint32_t)sx, (uint32_t)sy, 1};
    int rc;
    if ((rc = cached_tmap(&maps[0], p.in_hi, 4, dims, str, box, tc::TMAP_F16_SW128, es))) return rc;
    if (single) maps[1] = maps[0];  // not read by the single-pass kernel
    else if ((rc = cached_tmap(&maps[1], p.in_lo, 4, dims, str, box, tc::TMAP_F16_SW128, es))) return rc;
  }
  {
    const uint64_t ktot = (uint64_t)p.kh * p.kw * p.cin_pad;
    uint64_t dims[3] = {ktot, (uint64_t)p.cout_pad, (uint64_t)(p.w_per_batch ? p.B : 1)};
    uint64_t str[2] = {ktot * 2, ktot * 2 * p.cout_pad};
    uint32_t box[3] = {(uint32_t)kChunkK, (uint32_t)bn, 1};
    int rc;
    if ((rc = cached_tmap(&maps[2], p.w_hi, 3, dims, str, box))) return rc;
    if (single) maps[3] = maps[2];
    else if ((rc = cached_tmap(&maps[3], p.w_lo, 3, dims, str, box))) return rc;
  }
  if (single) {
    switch (bn) {
      case 16: return launch_cfg<16, true>(p, g, maps, s);
      case 32: return launch_cfg<32, true>(p, g, maps, s);
      case 64: return launch_cfg<64, true>(p, g, maps, s);
      case 96: return launch_cfg<96, true>(p, g, maps, s);
      default: return launch_cfg<128, true>(p, g, maps, s);
    }
  }
  switch (bn) {
    case 16: return launch_cfg<16, false>(p, g, maps, s);
    case 32: return launch_cfg<32, false>(p, g, maps, s);
    case 64: return launch_cfg<64, false>(p, g, maps, s);
    case 96: return launch_cfg<96, false>(p, g, maps, s);
    default: return launch_cfg<128, false>(p, g, maps, s);
  }
}

}  // namespace rb

namespace rb {
// ring depth of the forced width, or the deepest ring of any width (0: block_n is not a width)
template <bool SINGLE>
static int ring_max_of(int block_n) {
  switch (block_n) {
    case 0: return TcCfg<16, SINGLE>::kStages > TcCfg<32, SINGLE>::kStages ? TcCfg<16, SINGLE>::kStages : TcCfg<32, SINGLE>::kStages;
    case 16: return TcCfg<16, SINGLE>::kStages;
    case 32: return TcCfg<32, SINGLE>::kStages;
    case 64: return TcCfg<64, SINGLE>::kStages;
    case 96: return TcCfg<96, SINGLE>::kStages;
    case 128: return TcCfg<128, SINGLE>::kStages;
    default: return 0;
  }
}
}  // namespace rb

extern "C" int rb_debug_conv_override(int block_n, int bw_log2, int max_ctas, int stages) {
  using namespace rb;
  // the ring of the kernel the thread's math mode launches
  const int ring_max = math_mode() == RB_MATH_TC_FP16 ? ring_max_of<true>(block_n) : ring_max_of<false>(block_n);
  RB_REQUIRE(ring_max > 0, RB_ERR_BAD_ARG, "rb_debug_conv_override: block_n %d not in {0,16,32,64,96,128}", block_n);
  RB_REQUIRE(bw_log2 == 0 || (bw_log2 >= 3 && bw_log2 <= 7), RB_ERR_BAD_ARG, "rb_debug_conv_override: bw_log2 %d not 0 or in [3,7]",
             bw_log2);
  RB_REQUIRE(max_ctas >= 0, RB_ERR_BAD_ARG, "rb_debug_conv_override: max_ctas %d < 0", max_ctas);
  RB_REQUIRE(stages == 0 || (stages >= 2 && stages <= ring_max), RB_ERR_BAD_ARG,
             "rb_debug_conv_override: stages %d not 0 or in [2,%d]", stages, ring_max);
  g_override = {block_n, bw_log2, max_ctas, stages};
  g_record.fused_stats = 0;
  g_log_n = 0;
  return RB_OK;
}

extern "C" int rb_debug_conv_halo(int mode) {
  using namespace rb;
  RB_REQUIRE(mode >= -1 && mode <= 1, RB_ERR_BAD_ARG, "rb_debug_conv_halo: mode %d not in {-1, 0, 1}", mode);
  g_halo_mode = mode;
  return RB_OK;
}

extern "C" int rb_debug_conv_log(int i, int* rec) {
  using namespace rb;
  RB_REQUIRE(i >= 0 && i < g_log_n && rec, RB_ERR_BAD_ARG, "rb_debug_conv_log: launch %d of %d logged", i, g_log_n);
  memcpy(rec, g_log[i], sizeof(g_log[i]));
  return g_log_n;
}

extern "C" int rb_debug_conv_last(int* block_n, int* bw_log2, int* grid, int* stages, int* total_tiles) {
  using namespace rb;
  RB_REQUIRE(g_record.launched, RB_ERR_BAD_ARG, "rb_debug_conv_last: no tensor-core conv has been launched on this thread");
  if (block_n) *block_n = g_record.block_n;
  if (bw_log2) *bw_log2 = g_record.bw_log2;
  if (grid) *grid = g_record.grid;
  if (stages) *stages = g_record.stages;
  if (total_tiles) *total_tiles = g_record.total_tiles;
  return g_record.fused_stats;
}

extern "C" int rb_debug_conv_last_passes(void) {
  using namespace rb;
  RB_REQUIRE(g_record.launched, RB_ERR_BAD_ARG,
             "rb_debug_conv_last_passes: no tensor-core conv has been launched on this thread");
  return g_record.passes;
}
