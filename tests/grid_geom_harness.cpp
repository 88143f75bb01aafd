// TEST-ONLY host build of the grid geometry rule of locus_b200/csrc/grid.h (what the index build evaluates on the device
// and on the host): tests/test_grid_geom_cpu.py compares it bit for bit with a numpy restatement.
#include "../locus_b200/csrc/grid.h"

using namespace lb;

extern "C" {

// geom8: ox, oy, oz, inv_h, h as float bits, then nx, ny, nz
static void pack(const GridGeom& g, int32_t* geom8) {
  geom8[0] = float_to_bits(g.ox); geom8[1] = float_to_bits(g.oy); geom8[2] = float_to_bits(g.oz);
  geom8[3] = float_to_bits(g.inv_h); geom8[4] = float_to_bits(g.h);
  geom8[5] = g.nx; geom8[6] = g.ny; geom8[7] = g.nz;
}

void gg_auto_geom(const float* mn, const float* mx, uint32_t n, int32_t* geom8, int* key_bits) {
  const GridGeom g = grid_auto_geom(mn, mx, n);
  pack(g, geom8);
  *key_bits = grid_key_bits((uint64_t)g.nx * g.ny * g.nz);
}

void gg_make_geom(const float* mn, const float* mx, float cell, int32_t* geom8) {
  const float ext[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};
  pack(grid_make_geom(mn, ext, cell), geom8);
}

int gg_probe_accept(uint32_t n, uint32_t n_occ, float h, float* next_cell) {
  return grid_probe_accept(n, n_occ, h, next_cell) ? 1 : 0;
}

}
