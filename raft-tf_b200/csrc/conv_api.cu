// A14: stand-alone 'same' convolution with bias (+ReLU), i.e. the tensorpack Conv2D call every hot-path layer is made
// of (stride 1: model_utils.py:112-118,123-128,133-134,142-153,162-166,181-182; stride 2: the encoders' strided layers,
// model_utils.py:21,39,68,92), on fp32 NHWC tensors.  Same kernels as the fused update block: the input is split to fp16 hi/lo planes, the
// HWIO kernel is packed K-major, and the selected back end (wgmma or CUDA-core) runs the implicit
// GEMM.  Used by the parity tests to exercise every filter shape / tile geometry in isolation.
#include "packed.cuh"

namespace rb {

// the split input, then the packed conv (a blob of one conv)
struct ConvWs {
  SplitPtr in;
  PackedConv wt;  // offsets inside `blob`
  char* blob;
  size_t blob_bytes, total;
};

static ConvWs conv_ws_layout(int B, int h, int w, int cin, int cout, int kh, int kw, void* base) {
  ConvWs W;
  Arena a(base), blob;
  W.wt = reserve_conv(blob, kh, kw, round_up(cin, 64), cout);
  W.blob_bytes = blob.size;
  W.in = a.split((size_t)B * h * w * W.wt.cin_pad);
  W.blob = a.take<char>(W.blob_bytes);
  W.total = a.size;
  return W;
}

__global__ void split_pad_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo,
                                 size_t npix, int cin, int cin_pad) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * cin_pad) return;
  size_t pix = i / cin_pad;
  int c = i % cin_pad;
  float v = c < cin ? src[pix * cin + c] : 0.f;
  __half hh, ll;
  split_f32(v, hh, ll);
  hi[i] = hh;
  lo[i] = ll;
}

}  // namespace rb

using namespace rb;

extern "C" int rb_conv2d_workspace_bytes(int B, int h, int w, int cin, int cout, int kh, int kw, size_t* bytes) {
  RB_REQUIRE(bytes && B > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && kh > 0 && kw > 0, RB_ERR_BAD_ARG,
             "rb_conv2d_workspace_bytes: bad argument");
  *bytes = conv_ws_layout(B, h, w, cin, cout, kh, kw, nullptr).total;
  return RB_OK;
}

extern "C" int rb_conv2d(const float* x, const float* W_host, const float* b_host, float* y, int B, int h, int w,
                         int cin, int cout, int kh, int kw, int relu, void* workspace, size_t workspace_bytes,
                         void* stream) {
  return rb_conv2d_strided(x, W_host, b_host, y, B, h, w, cin, cout, kh, kw, 1, relu, workspace, workspace_bytes, stream);
}

extern "C" int rb_conv2d_strided(const float* x, const float* W_host, const float* b_host, float* y, int B, int h, int w,
                                 int cin, int cout, int kh, int kw, int stride, int relu, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  RB_REQUIRE(x && W_host && y && workspace, RB_ERR_BAD_ARG, "rb_conv2d: null pointer");
  RB_REQUIRE(B > 0 && h > 0 && w > 0 && cin > 0 && cout > 0, RB_ERR_BAD_SHAPE, "rb_conv2d: bad shape");
  RB_REQUIRE((kh & 1) && (kw & 1) && kh <= 7 && kw <= 7, RB_ERR_UNSUPPORTED,
             "rb_conv2d: only odd kernels up to 7 ('same'), got %dx%d", kh, kw);
  RB_REQUIRE(stride == 1 || stride == 2, RB_ERR_UNSUPPORTED, "rb_conv2d: stride %d (1 and 2 are what the reference uses)", stride);
  ConvWs L = conv_ws_layout(B, h, w, cin, cout, kh, kw, workspace);
  RB_REQUIRE(workspace_bytes >= L.total, RB_ERR_WORKSPACE, "rb_conv2d: workspace has %zu bytes, need %zu", workspace_bytes,
             L.total);
  cudaStream_t s = (cudaStream_t)stream;
  const PackedConv& wt = L.wt;
  int rc = upload_packed(L.blob, L.blob_bytes, s, [&](void* host) {
    pack_hwio(wt, host, W_host, cin, cout);
    for (int co = 0; b_host && co < cout; ++co) put_bias(wt, host, co, b_host[co]);
    return RB_OK;
  });
  if (rc) return rc;
  size_t npix = (size_t)B * h * w;
  size_t n = npix * wt.cin_pad;
  split_pad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, L.in.hi, L.in.lo, npix, cin, wt.cin_pad);
  RB_CHECK_LAUNCH("split_pad_kernel");
  ConvParams p = conv_params(conv_weights(wt, L.blob), L.in, wt.cin_pad, 0, B, h, w);
  if (stride != 1) {  // strided input view (ConvParams, common.cuh): y is [B, ceil(h/s), ceil(w/s), cout]
    int pt, pl, oh, ow;
    conv_pad_before(h, kh, stride, semantics(), &pt, &oh);
    conv_pad_before(w, kw, stride, semantics(), &pl, &ow);
    p.in_h = h; p.in_w = w; p.h = oh; p.w = ow;
    p.sx = p.sy = stride;
    p.pad_explicit = 1; p.pad_x = pl; p.pad_y = pt;
  }
  p.epi = EPI_F32; p.act = relu ? ACT_RELU : ACT_NONE; p.f0 = y;
  return launch_conv(p, s);
}
