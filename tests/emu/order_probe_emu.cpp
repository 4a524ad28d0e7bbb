/*
 * order_probe_emu.cpp -- two kernels whose output follows the order emu_launch runs threads in (cuda_emu.h), so
 * tests/test_emu_orders.py can check that GPX_EMU_ORDER and emu_set_order reach a launch.  Both are wrong on a device
 * on purpose; they exist only to make the order visible.  Test infrastructure only.
 */
#include "cuda_emu.h"

/* thread i copies what thread i - 1 wrote, plus one: out = 0, 1, 2, ... only when every thread runs after its
 * predecessor */
__global__ void k_probe_chain(uint32_t* out, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i ? out[i - 1] + 1 : 0;
}

/* each thread appends its index at the next free place: out = 0, 1, 2, ... only in ascending order */
__global__ void k_probe_append(uint32_t* out, uint32_t* count, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[atomicAdd(count, 1u)] = i;
}

/* out[0..n) zeroed, then the chain */
extern "C" void emu_probe_chain(uint32_t* out, uint32_t n, uint32_t block) {
  memset(out, 0, (size_t)n * sizeof *out);
  emu_launch(k_probe_chain, (n + block - 1) / block, block, out, n);
}

extern "C" void emu_probe_append(uint32_t* out, uint32_t n, uint32_t block) {
  uint32_t count = 0;
  emu_launch(k_probe_append, (n + block - 1) / block, block, out, &count, n);
}
