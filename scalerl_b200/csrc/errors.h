// The error channel of a library's C-ABI entry points and the argument checks they share (internal, not part of the C ABI).
// Every entry point reports through one message per calling thread: srl_last_error() in the product library, srl_test_last_error()
// in the test-hook library.
#pragma once
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <cuda_runtime.h>
#include "../../include/scalerl_b200.h"

namespace srl {

// The calling thread's message, one per shared object: hidden, so a process that loads both libraries keeps the two apart.
constexpr int ERROR_MESSAGE_BYTES = 512;
__attribute__((visibility("hidden"))) inline char* error_message() {
  static thread_local char msg[ERROR_MESSAGE_BYTES] = "";
  return msg;
}
// sets the message and returns code.  No argument may point into the message itself (vsnprintf must not overlap its output).
__attribute__((format(printf, 2, 3))) static inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(error_message(), ERROR_MESSAGE_BYTES, fmt, ap);
  va_end(ap);
  return code;
}
static inline int cuda_fail(cudaError_t e, const char* what) {
  return fail((int)e, "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
}

static inline bool misaligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

// One argument of a call: outputs may overlap nothing, inputs may overlap each other.  A NULL pointer (an optional argument) is skipped.
struct Span { const void* p; int64_t bytes; bool out; const char* name; };
// SRL_EINVAL, "<what>: <later argument> overlaps <earlier argument>", on the first overlap that involves an output
static inline int check_spans(const Span* s, int n, const char* what) {
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j) {
      if (!s[i].p || !s[j].p || !(s[i].out || s[j].out)) continue;
      const uintptr_t x = reinterpret_cast<uintptr_t>(s[i].p), y = reinterpret_cast<uintptr_t>(s[j].p);
      if (x < y + (uintptr_t)s[j].bytes && y < x + (uintptr_t)s[i].bytes) return fail(SRL_EINVAL, "%s: %s overlaps %s", what, s[i].name, s[j].name);
    }
  return 0;
}
static const char* const kW8[8] = {"weights8[0]", "weights8[1]", "weights8[2]", "weights8[3]", "weights8[4]", "weights8[5]", "weights8[6]", "weights8[7]"};
static const char* const kG8[8] = {"grads8[0]", "grads8[1]", "grads8[2]", "grads8[3]", "grads8[4]", "grads8[5]", "grads8[6]", "grads8[7]"};

}  // namespace srl

#define CU(x, what) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return srl::cuda_fail(e_, what); } while (0)
#define REQ(c, ...) do { if (!(c)) return srl::fail(SRL_EINVAL, __VA_ARGS__); } while (0)
