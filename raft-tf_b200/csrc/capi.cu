// Library-level entry points: version, thread-local error string, back-end selection, launch counter.
#include <stdarg.h>

#include "common.cuh"

namespace rb {
static thread_local char g_err[512] = "";
static thread_local int g_mode = RB_MATH_TC;
static thread_local int g_semantics = RB_SEMANTICS_REFERENCE;
static thread_local long long g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch() { ++g_launches; }
int math_mode() { return g_mode; }
int semantics() { return g_semantics; }

int current_device(int* dev) {
  RB_CHECK_CUDA(cudaGetDevice(dev));
  return RB_OK;
}
int device_sm_count(int dev) {
  constexpr int kDefaultSms = 132;  // H100 SXM: only if the device cannot be queried
  static int cache[256];  // 0 = not queried yet; racing first calls write the same value
  if (dev < 0 || dev >= 256) return kDefaultSms;
  int n = __atomic_load_n(&cache[dev], __ATOMIC_RELAXED);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kDefaultSms;
    __atomic_store_n(&cache[dev], n, __ATOMIC_RELAXED);
  }
  return n;
}
}  // namespace rb

extern "C" int rb_version(void) { return 100; }
extern "C" const char* rb_last_error(void) { return rb::g_err; }
extern "C" int rb_set_math_mode(int mode) {
  if (mode != RB_MATH_TC && mode != RB_MATH_SIMT && mode != RB_MATH_TC_FP16) {
    rb::set_error("rb_set_math_mode: unknown mode %d", mode);
    return RB_ERR_BAD_ARG;
  }
  rb::g_mode = mode;
  return RB_OK;
}
extern "C" int rb_get_math_mode(void) { return rb::g_mode; }
extern "C" int rb_set_semantics(int semantics) {
  if (semantics != RB_SEMANTICS_REFERENCE && semantics != RB_SEMANTICS_UPSTREAM) {
    rb::set_error("rb_set_semantics: unknown semantics %d", semantics);
    return RB_ERR_BAD_ARG;
  }
  rb::g_semantics = semantics;
  return RB_OK;
}
extern "C" int rb_get_semantics(void) { return rb::g_semantics; }
// The library links its own (static) CUDA runtime, whose per-thread "current device" is independent of the host
// framework's: a caller that drives several GPUs from one thread tells the library which one the following calls (and their
// stream handles -- stream 0 means "the current device's default stream") belong to.  raft_b200/capi.py does this in stream().
extern "C" int rb_set_device(int device) {
  RB_CHECK_CUDA(cudaSetDevice(device));
  return RB_OK;
}
extern "C" long long rb_launch_count(void) { return rb::g_launches; }
extern "C" void rb_launch_count_reset(void) { rb::g_launches = 0; }
