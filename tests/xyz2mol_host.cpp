// Host build of dig_b200/csrc/xyz2mol.cuh for the CPU tests (tests/test_xyz2mol_cpu.py compiles it with a host C++
// compiler and calls it through ctypes).  Test-only: the library has no CPU path.
#include <stdint.h>

#include "../dig_b200/csrc/xyz2mol.cuh"

extern "C" {

// The matching xyz2mol computes on an n-atom graph whose atoms are all unsaturated: adj[i] is atom i's neighbour mask.
// mate[i] = the matched atom, or -1.  Returns 0, or kInternalError.
int x2m_host_match(int n, const uint64_t* adj, int8_t* mate) {
  static x2m::Matcher m;
  m.nv = 0;
  for (int i = 0; i < n; ++i) m.local[i] = -1;
  for (int i = 0; i < n; ++i) {
    const uint64_t up = adj[i] & ~((2ull << i) - 1);
    if (!up) continue;
    if (m.local[i] < 0) m.local[i] = (int8_t)m.nv++;
    for (uint64_t u = up; u; u &= u - 1) {
      const int j = x2m::ctz64(u);
      if (m.local[j] < 0) m.local[j] = (int8_t)m.nv++;
    }
  }
  int8_t atom[x2m::kMaxAtoms];
  for (int i = 0; i < n; ++i)
    if (m.local[i] >= 0) {
      m.nbr[m.local[i]] = adj[i];
      atom[m.local[i]] = (int8_t)i;
    }
  m.solve();
  if (m.err) return x2m::kInternalError;
  for (int i = 0; i < n; ++i) mate[i] = m.local[i] >= 0 && m.mate[m.local[i]] >= 0 ? atom[m.mate[m.local[i]]] : -1;
  return 0;
}

// xyz2mol_one over n_mols molecules of n_atoms atoms, laid out as the kernel reads them.
void x2m_host_xyz2mol(const int64_t* z, const double* pos, int64_t n_mols, int n_atoms, int8_t* bo, int8_t* valid) {
  static x2m::Matcher m;
  for (int64_t k = 0; k < n_mols; ++k)
    valid[k] = (int8_t)x2m::xyz2mol_one(n_atoms, z + k * n_atoms, pos + k * n_atoms * 3,
                                        bo + k * (int64_t)n_atoms * n_atoms, m);
}

}  // extern "C"
