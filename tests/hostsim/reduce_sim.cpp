// tests/hostsim/reduce_sim.cpp — TEST INFRASTRUCTURE, never part of the product library.
//
// CPU stand-in for swgpu::launch_reduce (starway_b200/csrc/gpu.h), linked into libstarway_hostsim.so next to
// gpu_sim.cpp so that the CPU suite drives the engine's reducing receives (landing blocks, host-path routing, FIN,
// cancel, close) without a GPU.  dst += src element by element, synchronously on the calling thread.  f16 / bf16
// go through float and are rounded to nearest even, as one rounded add on the device is; loads and stores go
// through memcpy (a source may sit at any byte offset).
#include <stdio.h>
#include <string.h>

#include <cmath>

#include "../../starway_b200/csrc/gpu.h"

namespace swgpu {
namespace {

float f16_to_f32(uint16_t h) {
  const uint32_t sign = (uint32_t)(h & 0x8000) << 16, exp = (h >> 10) & 0x1f, man = h & 0x3ff;
  uint32_t u;
  if (exp == 0x1f) {
    u = sign | 0x7f800000u | (man << 13);
  } else if (exp) {
    u = sign | ((exp + 112) << 23) | (man << 13);
  } else {
    float f = (float)man * (1.0f / 16777216.0f);   // subnormal: man * 2^-24
    memcpy(&u, &f, 4);
    u |= sign;
  }
  float f;
  memcpy(&f, &u, 4);
  return f;
}
uint16_t f32_to_f16(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  const uint16_t sign = (uint16_t)((u >> 16) & 0x8000);
  const uint32_t a = u & 0x7fffffffu;
  if (a >= 0x7f800000u) return sign | 0x7c00 | (a > 0x7f800000u ? 0x200 : 0);   // inf / nan
  if (a >= 0x477ff000u) return sign | 0x7c00;                                    // rounds past 65504: inf
  if (a < 0x38800000u) {                                                          // below 2^-14: subnormal or zero
    float m;
    memcpy(&m, &a, 4);
    return sign | (uint16_t)std::nearbyint(m * 16777216.0f);                      // exact scaling, current mode: RNE
  }
  const uint32_t r = a + 0xfffu + ((a >> 13) & 1);                                // round mantissa to 10 bits, ties to even
  return sign | (uint16_t)((r - 0x38000000u) >> 13);
}
float bf16_to_f32(uint16_t h) {
  const uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
uint16_t f32_to_bf16(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1)) >> 16);
}
template <class T, class Add>
void reduce_seg(const SwSeg& g, Add add) {
  for (uint64_t off = 0; off + sizeof(T) <= g.len; off += sizeof(T)) {
    T d, v;
    memcpy(&d, (const void*)(uintptr_t)(g.dst + off), sizeof(T));
    memcpy(&v, (const void*)(uintptr_t)(g.src + off), sizeof(T));
    d = add(d, v);
    memcpy((void*)(uintptr_t)(g.dst + off), &d, sizeof(T));
  }
}

}  // namespace

int launch_reduce(stream_t, const SwSeg* segs, uint32_t nseg, int dtype, const BulkTuning* t) {
  for (uint32_t i = 0; i < nseg; i++) {
    const SwSeg& g = segs[i];
    const uint32_t isz = sw_dtype_size(dtype);
    // the same rule the CUDA kernels rely on: a segment the engine routed wrongly is reported, not summed
    if (!isz || ((g.dst | g.len) % isz) || (t->mode == 0 && ((g.src | g.dst | g.len) & 15))) {
      fprintf(stderr, "hostsim launch_reduce: segment %u breaks the kernel's alignment rule\n", i);
      return -1;
    }
    switch (dtype) {
      case SW_DT_F32: reduce_seg<float>(g, [](float a, float b) { return a + b; }); break;
      case SW_DT_F64: reduce_seg<double>(g, [](double a, double b) { return a + b; }); break;
      case SW_DT_I32: reduce_seg<uint32_t>(g, [](uint32_t a, uint32_t b) { return a + b; }); break;
      case SW_DT_I64: reduce_seg<uint64_t>(g, [](uint64_t a, uint64_t b) { return a + b; }); break;
      case SW_DT_F16: reduce_seg<uint16_t>(g, [](uint16_t a, uint16_t b) { return f32_to_f16(f16_to_f32(a) + f16_to_f32(b)); }); break;
      case SW_DT_BF16: reduce_seg<uint16_t>(g, [](uint16_t a, uint16_t b) { return f32_to_bf16(bf16_to_f32(a) + bf16_to_f32(b)); }); break;
    }
  }
  return 0;
}

}  // namespace swgpu
