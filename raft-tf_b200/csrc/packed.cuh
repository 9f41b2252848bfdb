// Host side of the conv operands: the one definition of the packed conv-weight format, the workspace arena every
// *_workspace_bytes query and layout carves with, and the ConvParams builder.
//
// Packed conv (DESIGN §3): split fp16 planes [cout_pad][kh*kw][cin_pad] (K-major, hi then lo) and an fp32 bias of
// cout_pad entries, each starting at a 256-byte boundary of the blob; cout_pad = round_up(cout, 16), the padding is zero.
#pragma once
#include <string.h>

#include <vector>

#include "common.cuh"

namespace rb {

// Hands out consecutive regions of a buffer, each starting at a multiple of its alignment and padded to one (workspace
// regions: 1024 bytes).  base == nullptr: offsets and the size only (the size queries), the pointers are null.
struct Arena {
  char* base;
  size_t size = 0;
  explicit Arena(void* b = nullptr) : base(reinterpret_cast<char*>(b)) {}
  size_t reserve(size_t bytes, size_t align = 1024) {  // byte offset of the region
    const size_t off = round_up(size, align);
    size = round_up(off + bytes, align);
    return off;
  }
  template <typename T>
  T* take(size_t count) {
    const size_t off = reserve(count * sizeof(T));
    return base ? reinterpret_cast<T*>(base + off) : nullptr;
  }
  SplitPtr split(size_t count) {  // hi plane, then lo plane, of `count` fp16 each
    SplitPtr s;
    s.hi = take<__half>(count);
    s.lo = take<__half>(count);
    return s;
  }
};

// One packed conv inside a weight blob: byte offsets of its planes and its geometry.  All zero: no such conv.
struct PackedConv {
  size_t hi, lo, bias;
  int kh, kw, cin_pad, cout, cout_pad;
};

// Reserves a packed conv at the blob's running offset: hi, lo, bias, each 256-byte aligned.
inline PackedConv reserve_conv(Arena& blob, int kh, int kw, int cin_pad, int cout) {
  PackedConv c;
  c.kh = kh; c.kw = kw; c.cin_pad = cin_pad; c.cout = cout; c.cout_pad = round_up(cout, 16);
  const size_t plane = (size_t)c.cout_pad * kh * kw * cin_pad * sizeof(__half);
  c.hi = blob.reserve(plane, 256);
  c.lo = blob.reserve(plane, 256);
  c.bias = blob.reserve((size_t)c.cout_pad * sizeof(float), 256);
  return c;
}

// Host: element (co, row, k) of packed conv c in a host image of its blob; row = tap index (ky * kw + kx), k < cin_pad.
inline void put_weight(const PackedConv& c, void* blob, int co, int row, int k, float v) {
  char* b = reinterpret_cast<char*>(blob);
  const size_t o = ((size_t)co * c.kh * c.kw + row) * c.cin_pad + k;
  split_f32(v, reinterpret_cast<__half*>(b + c.hi)[o], reinterpret_cast<__half*>(b + c.lo)[o]);
}
inline void put_bias(const PackedConv& c, void* blob, int co, float v) {
  reinterpret_cast<float*>(reinterpret_cast<char*>(blob) + c.bias)[co] = v;
}

// Host: a HWIO filter [kh*kw][cin][cout] as output channels [co_base, co_base + cout) of packed conv c.  scale (optional,
// one per output channel) multiplies each weight in double precision (batch norm folded at pack time).
inline void pack_hwio(const PackedConv& c, void* blob, const float* W, int cin, int cout, int co_base = 0,
                      const double* scale = nullptr) {
  const int taps = c.kh * c.kw;
  for (int t = 0; t < taps; ++t)
    for (int ci = 0; ci < cin; ++ci)
      for (int co = 0; co < cout; ++co) {
        const float v = W[((size_t)t * cin + ci) * cout + co];
        put_weight(c, blob, co_base + co, t, ci, scale ? (float)(v * scale[co]) : v);
      }
}

// Packs a weight blob of `bytes` bytes in host memory with pack(host) (zeroed first) and uploads it to `dst`.  Weight
// packing is an init-time call: it returns once the copy is complete.
template <typename F>
int upload_packed(void* dst, size_t bytes, cudaStream_t s, F pack) {
  std::vector<char> host(bytes, 0);
  const int rc = pack(host.data());
  if (rc) return rc;
  RB_CHECK_CUDA(cudaMemcpyAsync(dst, host.data(), bytes, cudaMemcpyHostToDevice, s));
  RB_CHECK_CUDA(cudaStreamSynchronize(s));
  return RB_OK;
}

// The weight operand of a conv as the kernels read it ([cout_pad][kh*kw][cin_pad] split planes and an fp32 bias).
struct ConvWeights {
  const __half* hi;
  const __half* lo;
  const float* bias;
  int kh, kw, cin_pad, cout, cout_pad;
};
inline ConvWeights conv_weights(const PackedConv& c, const void* blob) {
  const char* b = reinterpret_cast<const char*>(blob);
  return {reinterpret_cast<const __half*>(b + c.hi), reinterpret_cast<const __half*>(b + c.lo),
          reinterpret_cast<const float*>(b + c.bias), c.kh, c.kw, c.cin_pad, c.cout, c.cout_pad};
}

// A zeroed ConvParams for the stride-1 'same' conv of `wt` over in ([B][h][w][in_stride], first channel in_choff), scale 1;
// the caller adds the input view, the epilogue and its operands.
inline ConvParams conv_params(const ConvWeights& wt, SplitPtr in, int in_stride, int in_choff, int B, int h, int w) {
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.in_hi = in.hi; p.in_lo = in.lo; p.in_stride = in_stride; p.in_choff = in_choff;
  p.cin_pad = wt.cin_pad;
  p.w_hi = wt.hi; p.w_lo = wt.lo; p.bias = wt.bias;
  p.cout = wt.cout; p.cout_pad = wt.cout_pad; p.kh = wt.kh; p.kw = wt.kw;
  p.B = B; p.h = h; p.w = w;
  p.scale = 1.f;
  return p;
}

}  // namespace rb
