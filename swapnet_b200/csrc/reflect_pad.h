// swapnet_b200 — index fan-out of ReflectionPad2d(1) along one axis.
//
// Interior index i of an axis of n >= 2 elements appears in the padded axis (n + 2 elements) at i + 1, and also at 0
// when i == 1 and at n + 1 when i == n - 2.  For n == 3 both mirrors copy i = 1, so that index owns three padded
// positions.  The forward writers scatter a value to every position; the backward gathers fold them back.
//
// Plain C++ with no CUDA includes, so that the CPU suite can compile it on the host and compare it with torch.
// The positions are computed, not stored: an array indexed by a loop counter would live in local memory.
#pragma once

#ifdef __CUDACC__
#define SN_REFLECT_FN __host__ __device__ __forceinline__
#else
#define SN_REFLECT_FN inline
#endif

// how many padded positions interior index i has (1..3)
SN_REFLECT_FN int reflect_pad1_count(int i, int n) { return 1 + (i == 1) + (i == n - 2); }

// the k-th of them, k < reflect_pad1_count(i, n): i + 1, then 0 when i == 1, then n + 1 when i == n - 2
SN_REFLECT_FN int reflect_pad1_position(int i, int n, int k) {
  return k == 0 ? i + 1 : (k == 1 && i == 1 ? 0 : n + 1);
}
