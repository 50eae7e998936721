// xyz2mol on the GPU (reference dig/ggraph3D/utils/eval_validity_utils.py:382-405 with use_graph=True): the bond-order
// matrix and validity flag of every molecule of a batch with one atom count, one thread per molecule.  The per-molecule
// work (greedy adjacency, blossom matching) is sequential; the parallelism is the molecules of an evaluation.  The
// algorithm is in xyz2mol.cuh, shared with the host build the CPU tests check against networkx.
#include "common.cuh"
#include "xyz2mol.cuh"

using namespace dig3d;

namespace {

constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads) xyz2mol_kernel(const int64_t* __restrict__ z, const double* __restrict__ pos,
                                                           int64_t n_mols, int n_atoms, int8_t* __restrict__ bo,
                                                           int8_t* __restrict__ valid) {
  const int64_t m = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (m >= n_mols) return;
  x2m::Matcher st;
  valid[m] = (int8_t)x2m::xyz2mol_one(n_atoms, z + m * n_atoms, pos + m * n_atoms * 3,
                                      bo + m * (int64_t)n_atoms * n_atoms, st);
}

}  // namespace

extern "C" {

int dig3d_xyz2mol(const int64_t* z, const double* pos, int64_t n_mols, int32_t n_atoms, int8_t* bo, int8_t* valid,
                  void* stream) {
  DIG3D_REQUIRE(n_mols >= 0 && n_atoms >= 1 && n_atoms <= x2m::kMaxAtoms && (n_mols == 0 || (z && pos && bo && valid)),
                "xyz2mol: bad arguments (1 <= n_atoms <= %d, n_mols >= 0)", x2m::kMaxAtoms);
  DIG3D_REQUIRE((n_mols + kThreads - 1) / kThreads < (1ll << 31), "xyz2mol: too many molecules (%lld)",
                (long long)n_mols);
  if (n_mols == 0) return DIG3D_OK;
  xyz2mol_kernel<<<ceil_div(n_mols, kThreads), kThreads, 0, (cudaStream_t)stream>>>(z, pos, n_mols, n_atoms, bo, valid);
  DIG3D_LAUNCH_CHECK();
  return DIG3D_OK;
}

}  // extern "C"
