// host_emu_ray_batch.cpp — host build of pnr_ray_batch_row (csrc/ray_math.h), the per-ray routine of
// pnr_sample_ray_batch, so the CPU tests can compare it with the numpy oracle (tests/oracle_ray_batch.py) bit for bit
// without a GPU.  emu_sample_ray_batch is ray_batch_kernel's loop over the routine; the other two exports expose the
// generator and the pixel pick for the known-answer tests.
// Built by the `emu_rb` fixture of tests/oracle_ray_batch.py with: g++ -O2 -ffp-contract=off -shared -fPIC.
#include <cstdint>
#include "../panopticnerf_b200/csrc/ray_math.h"

extern "C" {

// rows r0 .. r1-1 with host pointers (no argument checks: the tests pass valid sets)
void emu_sample_ray_batch(const pnr_ray_batch_args* a) {
  for (int64_t r = a->r0; r < a->r1; ++r) pnr_ray_batch_row(*a, a->pix_offset, r);
}

// one Philox4x32-10 block
void emu_philox4x32_10(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  pnr_philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1], out);
}

uint64_t emu_mulhi64(uint64_t a, uint64_t b) { return pnr_mulhi64(a, b); }
}
