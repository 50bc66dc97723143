// Host build of hold_b200/csrc/embed_phases.h for tests/test_cpu_embed.py.
#include "../../hold_b200/csrc/embed_phases.h"

extern "C" {
// out[P][n_groups * 8], ok[n_groups] (mask per group): embedding (deriv = 0) or its derivative w.r.t. the element's own coordinate
void embed_groups(int D, int deriv, int n_embed, int P, const float* x, const float* ew, int n_groups, const int* e0, float* out, unsigned* ok) {
  for (int p = 0; p < P; ++p)
    for (int g = 0; g < n_groups; ++g) {
      float v[8];
      const float* q = x + (size_t)p * D;
      unsigned m;
      if (D == 3) m = deriv ? hold::embedn_inl<3, true>(e0[g], n_embed, q[0], q[1], q[2], 0.f, ew, v) : hold::embedn_inl<3, false>(e0[g], n_embed, q[0], q[1], q[2], 0.f, ew, v);
      else m = deriv ? hold::embedn_inl<4, true>(e0[g], n_embed, q[0], q[1], q[2], q[3], ew, v) : hold::embedn_inl<4, false>(e0[g], n_embed, q[0], q[1], q[2], q[3], ew, v);
      for (int i = 0; i < 8; ++i) out[((size_t)p * n_groups + g) * 8 + i] = v[i];
      if (p == 0) ok[g] = m;
    }
}
void sincos_host(int n, const float* x, float* s, float* c) {
  for (int i = 0; i < n; ++i) hold::sincos_cw(x[i], s[i], c[i]);
}
}
