// TEST INFRASTRUCTURE ONLY -- the device decomposition of the chained replan (faster_b200/csrc/fq_decomp.cuh: fq_decomp_kernel
// and fq_decomp_csr_kernel) compiled for the host and run under the block emulation of simt_emu/simt_emu.h, block by block
// with the launch shapes of fq_launch_decomp.  tests/test_pair_decomp_cpu.py compares it with fq_ellipsoid_decomp bit for
// bit.  Not a CPU path of the product.
#define FQ_EMULATE_ON_HOST 1
#define __shared__ static
#include "simt_emu/cuda_runtime.h"

inline int __popc(unsigned v) { return __builtin_popcount(v); }
using std::isfinite;

#include "fq_kernels.cuh"
#include "fq_decomp.cuh"

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
}  // namespace

extern "C" {
int emu_fit_pts() { return fqd::kFitPts; }

// fq_launch_decomp for one sweep: the staging and spill arrays are allocated here.  first: NULL or n_prob x 9 (the safe
// sweep's R).  face_ofs: n_prob * max_poly + 1; Ab: n_prob * max_faces rows; xf: n_prob x 9; pos_out / status optional.
// csr_threads: the CSR kernel's block size (any up to 1024).
void emu_decomp(int n_prob, int max_poly, const int* poly_ofs, const double* path, const double* first, const int* obs_ofs,
                const double* obs, int max_obs, const double* bbox, double inflate, double z_ground, int cap_pf, int max_faces,
                const double* goal, int* face_ofs, double* Ab, double* xf, double* pos_out, int* status, int csr_threads)
{
  FqDecompArgs a{};
  a.n_prob = n_prob; a.max_poly = max_poly; a.poly_ofs = poly_ofs; a.path = path; a.first = first; a.obs_ofs = obs_ofs; a.obs = obs;
  a.max_obs = max_obs; a.bbox[0] = bbox[0]; a.bbox[1] = bbox[1]; a.bbox[2] = bbox[2]; a.inflate = inflate; a.z_ground = z_ground;
  a.cap_pf = cap_pf; a.max_faces = max_faces;
  const size_t slots = (size_t)n_prob * max_poly;
  std::vector<double> stage(slots * (size_t)cap_pf * 4 + 1);
  std::vector<int> stage_n(slots + 1, 0x7eadbeef);
  a.spill_n = max_obs > fqd::kFitPts ? max_obs - fqd::kFitPts : 0;
  std::vector<double> spill(slots * (size_t)a.spill_n * 4 + 1);
  std::vector<uint8_t> spill_flag(slots * (size_t)a.spill_n + 1);
  a.stage = stage.data(); a.stage_n = stage_n.data(); a.spill = spill.data(); a.spill_flag = spill_flag.data();
  a.goal = goal; a.face_cap = (int)slots; a.face_ofs = face_ofs; a.Ab = Ab; a.xf = xf; a.pos_out = pos_out; a.status = status;
  if (max_poly > 0) launch((unsigned)slots, fqd::kThreads, [&] { fqd::fq_decomp_kernel(a); });
  launch(1, (unsigned)csr_threads, [&] { fqd::fq_decomp_csr_kernel(a); });
}
}

extern "C" {
// The host's segment decomposition (fq_decomp.cpp's decompose_segment, on the same fq_decomp.h helpers in the same order)
// up to carving round k, for telling a tie from a difference: out[0] = the distance of the host's pick at round k (the first
// strict minimum over the remaining points), out[1] = the smallest host distance of the remaining points within 1e-9 of the
// plane `row` (a, b: a.x = b, either sign), out[2] = that point's |a.p - b| (1e300: none).  Returns 0, or -1 when round k
// does not exist.
int emu_host_round(const double* p1_, const double* p2_, const double* obs, int n_obs, const double* bbox, double inflate, int k,
                   const double* row, double* out)
{
  using namespace fqd;
  const V3 p1 = { p1_[0], p1_[1], p1_[2] }, p2 = { p2_[0], p2_[1], p2_[2] };
  Plane bb[6];
  local_bbox(p1, p2, bbox, bb);
  double lo[3], hi[3];
  bbox_aabb(p1, bb, lo, hi);
  Ellip E;
  M3 Ri;
  double f;
  ellipsoid_start(p1, p2, &E, &Ri, &f);
  std::vector<V3> O;
  for (int i = 0; i < n_obs; i++)
  {
    const V3 pt = { obs[3 * i], obs[3 * i + 1], obs[3 * i + 2] };
    if (!outside_aabb(lo, hi, pt.x, pt.y, pt.z) && inside_bbox(bb, pt)) O.push_back(inflate_point(Ri, E.d, pt, inflate));
  }
  auto closest = [&](const std::vector<int>& idx) {
    int best = -1;
    double bd = 1.7976931348623157e308;
    for (int i : idx)
      if (E.dist(O[i]) < bd) { bd = E.dist(O[i]); best = i; }
    return best;
  };
  std::vector<int> inside0, cur, nxt;
  for (int i = 0; i < (int)O.size(); i++)
    if (E.dist(O[i]) <= 1) inside0.push_back(i);
  cur = inside0;
  while (!cur.empty())
  {
    shrink_short_axes(&E, Ri, O[closest(cur)]);
    nxt.clear();
    for (int i : cur) if (still_inside(E, O[i])) nxt.push_back(i);
    cur.swap(nxt);
  }
  E.ax[2] = f;
  cur.clear();
  for (int i : inside0) if (E.dist(O[i]) <= 1) cur.push_back(i);
  while (!cur.empty())
  {
    shrink_third_axis(&E, O[closest(cur)]);
    nxt.clear();
    for (int i : cur) if (still_inside(E, O[i])) nxt.push_back(i);
    cur.swap(nxt);
  }
  std::vector<int> remain(O.size());
  for (int i = 0; i < (int)O.size(); i++) remain[i] = i;
  for (int round = 0; !remain.empty(); round++)
  {
    const int best = closest(remain);
    if (round == k)
    {
      // the plane is tangent to the ellipsoid's level set at its point, so that point is the nearest of those on the plane
      out[0] = E.dist(O[best]);
      out[1] = 1e300; out[2] = 1e300;
      for (int i : remain)
      {
        const double r = std::fabs(row[0] * O[i].x + row[1] * O[i].y + row[2] * O[i].z - row[3]);
        if (r <= 1e-9 && E.dist(O[i]) < out[1]) { out[1] = E.dist(O[i]); out[2] = r; }
      }
      return 0;
    }
    const V3 cp = O[best], n = tangent_normal(E, cp);
    nxt.clear();
    for (int i : remain) if (before_plane(n, cp, O[i])) nxt.push_back(i);
    remain.swap(nxt);
  }
  return -1;
}
}
