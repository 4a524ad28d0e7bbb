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
 */
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>

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

/* run kernel(args...) over grid x block threads, block by block, thread by thread */
template <class K, class... Args>
static void emu_launch(K kernel, unsigned grid, unsigned block, Args... args) {
  emu_gridDim = dim3(grid, 1, 1);
  emu_blockDim = dim3(block, 1, 1);
  for (unsigned b = 0; b < grid; b++)
    for (unsigned t = 0; t < block; t++) {
      emu_blockIdx = {b, 0, 0};
      emu_threadIdx = {t, 0, 0};
      kernel(args...);
    }
}
