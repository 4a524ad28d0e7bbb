/*
 * wire_exec.h -- the CPU executor of gigapaxos_b200/csrc/gpx_wire_seq.h and gpx_state_seq.h, so that the CPU tests run
 * the product's own host sequences (argument checks, scratch layouts, passes, sorts, scans, capacity decisions, early
 * exits) over the kernels compiled for the host by cuda_emu.h.  Only what the CUDA executor does with CUB and the CUDA
 * runtime is done here with the standard library.  Test infrastructure only.
 */
#pragma once
#include "cuda_emu.h"

#include <cstdlib>
#include <memory>
#include <numeric>
#include <string>
#include <vector>

static std::string emu_err; /* the message of the last refusal */
static int fail(int code, const std::string& msg) {
  emu_err = msg;
  return code;
}
extern "C" const char* emu_last_error() { return emu_err.c_str(); }

#include "gpx_wire_seq.h"

/* a scan's row total passed its bound: the kernels would have written past the arrays the host sized (the JSON
 * decoder's events and members) */
enum { EMU_EBOUND = -100 };

struct EmuExec {
  uint32_t block; /* every kernel runs in blocks of the test's size */
  void* buf = nullptr;
  size_t bytes = 0;
  ~EmuExec() { free(buf); }
  WireEnv env(const DevState& S, const WireNames& W) { return WireEnv{S, W, &buf, &bytes}; }

  template <class K, class... A>
  int launch(K kernel, uint32_t n, uint32_t, const A&... a) {
    emu_launch(kernel, (n + block - 1) / block, block, a...);
    return GPX_OK;
  }
  /* as CUB's radix sort: stable, on the low `bits` bits only, the whole keys out */
  template <typename K>
  int sort(const K* key, K* skey, const uint32_t* val, uint32_t* perm, uint32_t n, int bits, void*, size_t) {
    const K mask = bits >= (int)(8 * sizeof(K)) ? ~(K)0 : (K)(((K)1 << bits) - 1);
    std::vector<uint32_t> idx(n);
    std::iota(idx.begin(), idx.end(), 0u);
    std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return (key[a] & mask) < (key[b] & mask); });
    for (uint32_t i = 0; i < n; i++) {
      skey[i] = key[idx[i]];
      perm[i] = val[idx[i]];
    }
    return GPX_OK;
  }
  int scan(const uint32_t* cnt, uint32_t* off, uint32_t n, uint32_t rows, const WireScan&, uint64_t bound = ~0ull) {
    for (uint32_t j = 0; j < rows; j++) {
      uint64_t s = 0;
      for (uint32_t i = 0; i < n; i++) {
        off[(size_t)j * n + i] = (uint32_t)s;
        s += cnt[(size_t)j * n + i];
      }
      if (s > bound) return EMU_EBOUND;
    }
    return GPX_OK;
  }
  int totals(const uint32_t* cnt, const uint32_t* off, uint32_t n, uint32_t rows, uint32_t* tot) {
    for (uint32_t j = 0; j < rows; j++) tot[j] = off[(size_t)j * n + n - 1] + cnt[(size_t)j * n + n - 1];
    return GPX_OK;
  }
  int scan_by_key(const uint32_t* key, const JsonSum* sum, JsonSum* pre, uint32_t n, const WireScan&) {
    JsonSum acc = json_identity();
    for (uint32_t i = 0; i < n; i++) {
      if (i == 0 || key[i] != key[i - 1]) acc = json_identity();
      pre[i] = acc;
      acc = JsonCompose()(acc, sum[i]);
    }
    return GPX_OK;
  }
  int sum_by_key(const unsigned long long* key, const uint32_t* val, uint32_t* start, uint32_t n, const WireScan&) {
    for (uint32_t j = 0, s = 0; j < n; j++) {
      if (j == 0 || key[j] != key[j - 1]) s = 0;
      start[j] = s;
      s += val[j];
    }
    return GPX_OK;
  }
  int fill(void* p, int byte, size_t n) {
    memset(p, byte, n);
    return GPX_OK;
  }
  int upload(void* dst, const void* host, size_t n) {
    memcpy(dst, host, n);
    return GPX_OK;
  }
  int column(uint32_t* dst, const void* src, size_t pitch, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) memcpy(dst + i, (const uint8_t*)src + i * pitch, 4);
    return GPX_OK;
  }
  int read(void* host, const void* src, size_t n) { return upload(host, src, n); }
  int sync() { return GPX_OK; }
  int settle() { return GPX_OK; } /* no lockstep records here */
  /* a fresh buffer on every layout, its bytes past `keep` garbage: a pass that reads what an earlier one wrote finds it
   * only if the layout kept it */
  int grow(void** b, size_t* cap, size_t need, size_t keep) {
    const size_t alloc = (need + 255) / 256 * 256 + 256;
    void* q = aligned_alloc(256, alloc);
    memset(q, 0xa5, alloc);
    if (keep) memcpy(q, *b, keep);
    free(*b);
    *b = q;
    *cap = need;
    return GPX_OK;
  }
  size_t scan_bytes(uint32_t) { return 0; }
  size_t sort_bytes(uint32_t, int) { return 0; }
  size_t sort64_bytes(uint32_t, int) { return 0; }
  size_t scan_by_key_bytes(uint32_t) { return 0; }
  size_t sum_by_key_bytes(uint32_t) { return 0; }
};

/* no other calls to order with */
struct EmuCall {
  int begin() { return GPX_OK; }
  int end() { return GPX_OK; }
};

/* a capacity of the tests' uint64_t sizes[] as the C ABI's uint32_t one */
static uint32_t cap32(uint64_t c) { return (uint32_t)std::min<uint64_t>(c, 0xffffffffu); }
