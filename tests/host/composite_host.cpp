// Host run of the composite walks (hold_b200/csrc/composite_phases.h): hold_composite and hold_composite_bwd with one loop
// iteration per ray in place of one thread, the same argument set-up, no argument checks.
#include <string.h>

#include "../../hold_b200/csrc/composite_phases.h"

using namespace hold;

extern "C" void composite_host(int n, int R, int S, const hold_factors* factors, const int32_t* cls, const hold_render_out* comp,
                               const hold_render_out* per_node) {
  if (comp != nullptr) {
    CompositeArgs a;
    memset(&a, 0, sizeof(a));
    a.n = n, a.R = R, a.S = S;
    for (int k = 0; k < n; ++k) {
      a.color[k] = factors[k].color, a.normal[k] = factors[k].normal, a.density[k] = factors[k].density, a.z[k] = factors[k].z_vals;
      a.class_id[k] = cls[k];
    }
    a.out = *comp, a.drop_head = n - 1, a.drop_tail = n, a.single_zmax_last = 0;
    for (int r = 0; r < R; ++r) composite_ray(a, r);
  }
  if (per_node != nullptr) {
    for (int k = 0; k < n; ++k) {
      CompositeArgs b;
      memset(&b, 0, sizeof(b));
      b.n = 1, b.R = R, b.S = S;
      b.color[0] = factors[k].color, b.normal[0] = factors[k].normal, b.density[0] = factors[k].density, b.z[0] = factors[k].z_vals;
      b.class_id[0] = cls[k];
      b.out = per_node[k], b.drop_head = 0, b.drop_tail = 0, b.single_zmax_last = 1;
      for (int r = 0; r < R; ++r) composite_ray(b, r);
    }
  }
}

extern "C" void composite_bwd_host(int n, int R, int S, const hold_factors* factors, const int32_t* cls, const hold_render_out* g_comp,
                                   const hold_render_out* g_per_node, const hold_factors* d_factors) {
  bool written = false;
  if (g_comp != nullptr) {
    CompositeBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.n = n, a.R = R, a.S = S;
    for (int k = 0; k < n; ++k) {
      a.color[k] = factors[k].color, a.normal[k] = factors[k].normal, a.density[k] = factors[k].density, a.z[k] = factors[k].z_vals;
      a.class_id[k] = cls[k];
      a.d_color[k] = d_factors[k].color, a.d_normal[k] = d_factors[k].normal, a.d_density[k] = d_factors[k].density;
    }
    a.g = *g_comp, a.drop_head = n - 1, a.drop_tail = n, a.single_zmax_last = 0, a.accumulate = 0;
    for (int r = 0; r < R; ++r) composite_bwd_ray(a, r);
    written = true;
  }
  if (g_per_node != nullptr) {
    for (int k = 0; k < n; ++k) {
      CompositeBwdArgs b;
      memset(&b, 0, sizeof(b));
      b.n = 1, b.R = R, b.S = S;
      b.color[0] = factors[k].color, b.normal[0] = factors[k].normal, b.density[0] = factors[k].density, b.z[0] = factors[k].z_vals;
      b.class_id[0] = cls[k];
      b.d_color[0] = d_factors[k].color, b.d_normal[0] = d_factors[k].normal, b.d_density[0] = d_factors[k].density;
      b.g = g_per_node[k], b.drop_head = 0, b.drop_tail = 0, b.single_zmax_last = 1, b.accumulate = written ? 1 : 0;
      for (int r = 0; r < R; ++r) composite_bwd_ray(b, r);
    }
  }
}
