/*
 * cuda_emu.h -- just enough of the CUDA execution model to run a SCALAR kernel (no warp-level primitives, no shared
 * memory, no inline PTX on its path) on the host, one thread after the other.  Test infrastructure: it lets a CPU
 * test execute the very source of such a kernel (gigapaxos_b200/csrc/gpx_phase1b.cuh) against the oracle without
 * a GPU.  The product never includes this file.
 *
 * <cuda_runtime.h> is host-compilable (g++): it brings int4 / make_int4 / uint3 and defines __device__, __global__,
 * __forceinline__ ... away.  What is left: the built-in index variables (declared `extern const` there, so they are
 * renamed to mutable globals), the few device-only names gpx_dev.cuh mentions in functions the emulated kernels never
 * call, and the atomics (atomicAdd, atomicMax, atomicMin, atomicCAS).
 *
 * A launch runs its threads one after the other in the order GPX_EMU_ORDER names (see emu_launch): the device runs
 * them in no fixed order, so an emulated kernel's output must not depend on the order of the threads of a launch.
 */
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

using std::max;
using std::min;

static uint3 emu_threadIdx, emu_blockIdx;
static dim3 emu_blockDim, emu_gridDim;
#define threadIdx emu_threadIdx
#define blockIdx emu_blockIdx
#define blockDim emu_blockDim
#define gridDim emu_gridDim

#ifndef __noinline__
#define __noinline__
#endif
#ifndef __launch_bounds__
#define __launch_bounds__(...)
#endif
#ifndef __grid_constant__
#define __grid_constant__
#endif
#define __cvta_generic_to_shared(p) ((size_t)(p)) /* only inside the TMA helpers, never executed here */

template <class T>
static inline T atomicAdd(T* p, T v) { /* one thread at a time */
  T old = *p;
  *p = (T)(old + v);
  return old;
}

template <class T>
static inline T atomicMax(T* p, T v) {
  T old = *p;
  if (v > old) *p = v;
  return old;
}

template <class T>
static inline T atomicMin(T* p, T v) {
  T old = *p;
  if (v < old) *p = v;
  return old;
}

template <class T>
static inline T atomicCAS(T* p, T cmp, T v) {
  T old = *p;
  if (old == cmp) *p = v;
  return old;
}

/* The order of a launch's (block, thread) pairs, from GPX_EMU_ORDER or emu_set_order:
 *   asc            block by block, thread by thread (the default);
 *   desc           the whole grid reversed;
 *   shuffle:<seed> one permutation of all pairs of the launch, blocks mixed in with threads (the device orders neither).
 * The atomics above stay one thread at a time, so the order of the threads is also the order of the atomics.  A
 * shuffle's permutation follows from the seed, the pytest test phase the launch runs in (PYTEST_CURRENT_TEST, when
 * set) and the number of launches since that phase began, so `GPX_EMU_ORDER=shuffle:<seed> pytest <file> -k <test>`
 * replays a failing test's launches in the same orders. */
enum { EMU_ASC = 0, EMU_DESC = 1, EMU_SHUFFLE = 2 };
struct EmuOrder {
  int mode = -1; /* -1: read GPX_EMU_ORDER at the next launch */
  uint64_t seed = 0;
  uint64_t launches = 0; /* since the current test phase began */
  std::string phase;     /* PYTEST_CURRENT_TEST at the last launch */
};
static EmuOrder emu_order;

static int emu_parse_order(const char* s, int* mode, uint64_t* seed) {
  if (!s || !*s || !strcmp(s, "asc")) {
    *mode = EMU_ASC;
    return 0;
  }
  if (!strcmp(s, "desc")) {
    *mode = EMU_DESC;
    return 0;
  }
  if (!strncmp(s, "shuffle:", 8) && s[8] >= '0' && s[8] <= '9') {
    char* end;
    const unsigned long long v = strtoull(s + 8, &end, 10);
    if (!*end) {
      *mode = EMU_SHUFFLE;
      *seed = v;
      return 0;
    }
  }
  return -1;
}

/* the order of the following launches of this library: "asc", "desc", "shuffle:<seed>", or null to go back to
 * GPX_EMU_ORDER.  Restarts the launch count.  Returns 0, or -1 (order unchanged) for a spec it does not know. */
extern "C" int emu_set_order(const char* spec) {
  int mode;
  uint64_t seed = 0;
  if (!spec) {
    emu_order.mode = -1;
    return 0;
  }
  if (emu_parse_order(spec, &mode, &seed)) return -1;
  emu_order.mode = mode;
  emu_order.seed = seed;
  emu_order.launches = 0;
  return 0;
}

static uint64_t emu_mix(uint64_t x) { /* splitmix64's finaliser */
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

/* run kernel(args...) over grid x block threads, one thread at a time, in the order above */
template <class K, class... Args>
static void emu_launch(K kernel, unsigned grid, unsigned block, Args... args) {
  if (emu_order.mode < 0) {
    const char* env = getenv("GPX_EMU_ORDER");
    if (emu_parse_order(env, &emu_order.mode, &emu_order.seed)) {
      fprintf(stderr, "GPX_EMU_ORDER=%s: want asc, desc or shuffle:<seed>\n", env);
      abort();
    }
  }
  const char* test = getenv("PYTEST_CURRENT_TEST");
  if (emu_order.phase != (test ? test : "")) {
    emu_order.phase = test ? test : "";
    emu_order.launches = 0;
  }
  uint64_t h = 0xcbf29ce484222325ull; /* FNV-1a of the test phase */
  for (const char c : emu_order.phase) h = (h ^ (uint8_t)c) * 0x100000001b3ull;
  uint64_t r = emu_mix(emu_order.seed ^ emu_mix(h ^ emu_mix(emu_order.launches++)));

  emu_gridDim = dim3(grid, 1, 1);
  emu_blockDim = dim3(block, 1, 1);
  const uint64_t n = (uint64_t)grid * block;
  std::vector<uint64_t> perm;
  if (emu_order.mode == EMU_SHUFFLE) {
    perm.resize(n);
    for (uint64_t i = 0; i < n; i++) perm[i] = i;
    for (uint64_t i = n; i > 1; i--) { /* Fisher-Yates */
      r = emu_mix(r);
      std::swap(perm[i - 1], perm[r % i]);
    }
  }
  for (uint64_t i = 0; i < n; i++) {
    const uint64_t k = emu_order.mode == EMU_SHUFFLE ? perm[i] : emu_order.mode == EMU_DESC ? n - 1 - i : i;
    emu_blockIdx = {(unsigned)(k / block), 0, 0};
    emu_threadIdx = {(unsigned)(k % block), 0, 0};
    kernel(args...);
  }
}
