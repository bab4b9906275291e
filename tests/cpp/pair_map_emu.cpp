// TEST INFRASTRUCTURE ONLY -- the map paths of the chained replan's kernels (faster_b200/csrc/fq_decomp.cuh: fq_decomp_kernel
// and fq_decomp_csr_kernel with an indexed map; fq_pair.cuh: fq_pair_hr_kernel with an indexed map) compiled for the host and
// run under the block emulation of simt_emu/simt_emu.h, with the launch shapes of fq_kernels.cu.  The index comes from the
// numpy restatement of tests/test_pair_map_cpu.py, which compares the results with fq_ellipsoid_decomp and
// tests/pair_hr_oracle.py.  Not a CPU path of the product.
#define FQ_EMULATE_ON_HOST 1
#define __shared__ static
#include "simt_emu/cuda_runtime.h"

inline int __popc(unsigned v) { return __builtin_popcount(v); }
using std::isfinite;

#include "fq_kernels.cuh"
#include "fq_decomp.cuh"
#include "fq_pair.cuh"

#include <vector>

namespace
{
template <class F>
struct Thunk
{
  F f;
  static void call(void* p) { static_cast<Thunk*>(p)->f(); }
};
template <class F>
void launch(unsigned grid, unsigned block, F f)
{
  Thunk<F> t{ f };
  for (unsigned b = 0; b < grid; b++) simt::run_block(dim3(grid), dim3(block), uint3{ b, 0, 0 }, Thunk<F>::call, &t, 64 * 1024);
}

// grid: origin x, y, z, cell; dims: x, y, z.  unk / occ: the sorted points, their indices and the cell starts of each cloud
FqMapDev map_of(const double* grid, const int* dims, const double* unk_xyz, const int* unk_idx, const int* unk_start, int n_unk,
                const double* occ_xyz, const int* occ_idx, const int* occ_start, int n_occ)
{
  FqMapDev m;
  for (int k = 0; k < 3; k++) { m.grid.origin[k] = grid[k]; m.grid.dims[k] = dims[k]; }
  m.grid.cell = grid[3];
  m.grid.n_cells = dims[0] * dims[1] * dims[2];
  m.unk = { unk_xyz, unk_idx, unk_start, n_unk };
  m.occ = { occ_xyz, occ_idx, occ_start, n_occ };
  return m;
}
}  // namespace

extern "C" {
// fq_launch_decomp for one sweep against one map (map_unk 0: O, 1: U ++ O); max_local caps one segment's survivors.  The
// other arguments as pair_decomp_emu.cpp's emu_decomp.
void emu_decomp_map(int n_prob, int max_poly, const int* poly_ofs, const double* path, const double* first, const double* grid,
                    const int* dims, const double* unk_xyz, const int* unk_idx, const int* unk_start, int n_unk, const double* occ_xyz,
                    const int* occ_idx, const int* occ_start, int n_occ, int map_unk, int max_local, const double* bbox, double inflate,
                    double z_ground, int cap_pf, int max_faces, const double* goal, int* face_ofs, double* Ab, double* xf, double* pos_out,
                    int* status)
{
  const FqMapDev m = map_of(grid, dims, unk_xyz, unk_idx, unk_start, n_unk, occ_xyz, occ_idx, occ_start, n_occ);
  const FqMapDev* table[1] = { &m };
  FqDecompArgs a{};
  a.n_prob = n_prob; a.max_poly = max_poly; a.poly_ofs = poly_ofs; a.path = path; a.first = first;
  a.maps = table; a.map_index = nullptr; a.n_maps = 1; a.map_unk = map_unk; a.max_obs = max_local;
  a.bbox[0] = bbox[0]; a.bbox[1] = bbox[1]; a.bbox[2] = bbox[2]; a.inflate = inflate; a.z_ground = z_ground;
  a.cap_pf = cap_pf; a.max_faces = max_faces;
  const size_t slots = (size_t)n_prob * max_poly;
  std::vector<double> stage(slots * (size_t)cap_pf * 4 + 1);
  std::vector<int> stage_n(slots + 1, 0x7eadbeef);
  a.spill_n = max_local > fqd::kFitPts ? max_local - fqd::kFitPts : 0;
  std::vector<double> spill(slots * (size_t)a.spill_n * 4 + 1);
  std::vector<uint8_t> spill_flag(slots * (size_t)a.spill_n + 1);
  std::vector<int> spill_idx(slots * (size_t)a.spill_n + 1);
  a.stage = stage.data(); a.stage_n = stage_n.data(); a.spill = spill.data(); a.spill_flag = spill_flag.data(); a.spill_idx = spill_idx.data();
  a.goal = goal; a.face_cap = (int)slots; a.face_ofs = face_ofs; a.Ab = Ab; a.xf = xf; a.pos_out = pos_out; a.status = status;
  if (max_poly > 0) launch((unsigned)slots, fqd::kThreads, [&] { fqd::fq_decomp_kernel(a); });
  launch(1, 64, [&] { fqd::fq_decomp_csr_kernel(a); });
}

// fq_launch_pair_hr with `block` threads per corridor against one map's U; params: drone_radius, delta_a, delta_H
void emu_pair_hr_map(int block, int n_prob, int N, double DC, const double* params, const double* coeffs, const double* win_dt,
                     const int* win_idx, const double* lim, const double* grid, const int* dims, const double* unk_xyz, const int* unk_idx,
                     const int* unk_start, int n_unk, int* r_index, uint8_t* need, int* index_H)
{
  const FqMapDev m = map_of(grid, dims, unk_xyz, unk_idx, unk_start, n_unk, nullptr, nullptr, nullptr, 0);
  const FqMapDev* table[1] = { &m };
  FqPairHrArgs a;
  a.n_prob = n_prob; a.N = N; a.DC = DC; a.drone_radius = params[0]; a.delta_a = params[1]; a.delta_H = params[2];
  a.coeffs = coeffs; a.win_dt = win_dt; a.win_idx = win_idx; a.lim = lim; a.unk_ofs = nullptr; a.unk = nullptr;
  a.r_index = r_index; a.need = need; a.need_out = nullptr; a.index_H = index_H;
  a.maps = table; a.map_index = nullptr;
  launch((unsigned)n_prob, (unsigned)block, [&] { fqp::fq_pair_hr_kernel(a); });
}
}
