// rng.cuh -- the counter-based generator of libcogdl_b200 (host and device).
//
// Every random decision the library makes is a pure function of (seed, i, k): two rounds of the splitmix64
// finaliser, no state, no sequence.  Users:
//   * the neighbour sampler (sampler.cu): i = batch slot, k = draw index;
//   * the GAT attention dropout (edge_softmax.cu): i = CSR edge position, k = head; the (edge, head) is kept iff
//     draw(seed, p, h) >= drop_below, drop_below = floor(p_drop * 2^64).
// cogdl_b200_sample_draw exports draw() to the host; the CPU oracle (oracle_sample_draw) and the tests restate it.
#pragma once
#include <stdint.h>

namespace cogdl_b200 {

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// draw k of counter i
__host__ __device__ __forceinline__ uint64_t draw(uint64_t seed, int64_t i, int64_t k) {
  return mix64(mix64(seed + (uint64_t)i * 0xD1342543DE82EF95ull) + (uint64_t)k);
}

}  // namespace cogdl_b200
