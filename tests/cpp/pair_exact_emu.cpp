// TEST INFRASTRUCTURE ONLY -- the exact stage of the chained replan (faster_b200/csrc/fq_bnb.cuh: roots, the generalised
// level kernel, certify, resolve) and the presolve of fq_presolve.h compiled for the host and run under the block emulation
// of simt_emu/simt_emu.h, block by block with the launch shapes of fq_kernels.cu / fq_pair_capi.cu.  tests/test_pair_exact_cpu.py
// feeds it list winners computed on the CPU and compares the winners with the CPU restatement.  emu_strict_tree drives the
// same level kernel as fq_gen_new_traj_exact does: one corridor, one warp per child, strict pruning, the host reading the
// counts between levels.  Not a CPU path of the product.
#define FQ_EMULATE_ON_HOST 1
#include "simt_emu/cuda_runtime.h"

#include "fq_kernels.cuh"
#include "fq_kernels_t.cuh"
#include "fq_bnb.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

namespace fqt
{
alignas(16) unsigned char smem_raw[232 * 1024];
}
namespace fqb
{ // the level kernel's dynamic shared array (one block runs at a time)
alignas(16) unsigned char smem_raw[232 * 1024];
}

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
  for (unsigned b = 0; b < grid; b++) simt::run_block(dim3(grid), dim3(block), uint3{ b, 0, 0 }, Thunk<F>::call, &t, 512 * 1024);
}

struct Plan
{
  int N, ff;
  const double *TZ, *T0, *FT;
};
void fill_plan(const Plan& p, FqKernelArgs* k)
{
  const int ne = p.ff ? 3 : 2;
  k->N = p.N; k->force_final = p.ff; k->ne = ne; k->nz = p.N - ne; k->nw = 3 * (p.N - ne); k->NY = 6 * p.N + 1;
  k->ld = (3 * (p.N - ne)) | 1; k->TZ = p.TZ; k->T0 = p.T0; k->FT = p.FT;
}

// one level launch of fq_launch_bnb_level for the instantiated shapes
int level(const fqb::BnbArgs& b)
{
  const int key = b.k.N * 2 + (b.k.force_final ? 1 : 0);
  const unsigned blocks = (unsigned)((long long)b.k.n_prob * b.cpc);
  auto go = [&](auto kern, size_t smem) {
    if (smem > sizeof(fqb::smem_raw)) return -2;
    launch(blocks, fqb::W * 32, [&] { kern(b); });
    return 0;
  };
  switch (key)
  {
    case 6 * 2 + 1: return go(fqb::fq_bnb_level_kernel<6, true>, fqb::level_smem<6, true>(b.k.max_faces, b.k.item_cap));
    case 6 * 2 + 0: return go(fqb::fq_bnb_level_kernel<6, false>, fqb::level_smem<6, false>(b.k.max_faces, b.k.item_cap));
    default: return -1;
  }
}
}  // namespace

extern "C" {
// fqs::root_possible on the host, for n_t time allocations
void emu_presolve_host(int P, const int* face_ofs, const double* Ab, const double* x0, const double* xf, int ff, int n_t, const double* t,
                       double tol, uint8_t* out)
{
  for (int i = 0; i < n_t; i++) out[i] = fqs::root_possible(P, face_ofs, Ab, x0, xf, ff, t[i], tol) ? 1 : 0;
}

// fqa::rank (fq_assign.h): the index of sigma in L(N, P, all_limit), or -1
long long emu_rank(int N, int P, long long all_limit, const uint8_t* sigma)
{
  return fqa::rank(N, P, fqa::use_all(N, P, all_limit), sigma);
}

// fq_bnb_roots_kernel alone, every corridor without a list winner (all its factors searched): roots (n_prob x n_fac),
// their counts and the corridors' status
void emu_roots(int N, int ff, int n_prob, const double* x0, const double* xf, const int* poly_ofs, const int* face_ofs, const double* Ab,
               int max_faces, double row_tol, const int* cand_ofs, const double* cand_dt, int n_fac, int* roots, int* n_roots, uint8_t* status)
{
  const size_t cells = (size_t)n_prob * n_fac;
  std::vector<double> dts(cells);
  std::vector<unsigned long long> inc(cells), lb(cells);
  std::vector<uint8_t> closed(cells);
  std::vector<int> n_par(2 * (size_t)n_prob), n_leaves(n_prob), flags(2 * (size_t)n_prob), win_idx(n_prob, -1);
  std::vector<long long> nodes(n_prob);
  std::vector<double> win_cost(n_prob, INFINITY);
  FqBnbChainArgs c{};
  c.n_prob = n_prob; c.N = N; c.force_final = ff; c.stride = n_fac; c.max_faces = max_faces; c.tree_ok = 1; c.all_limit = 0;
  c.poly_ofs = poly_ofs; c.face_ofs = face_ofs; c.Ab = Ab; c.x0 = x0; c.xf = xf; c.row_tol = row_tol; c.cand_ofs = cand_ofs;
  c.cand_dt = cand_dt; c.n_fac = n_fac; c.win_idx = win_idx.data(); c.win_cost = win_cost.data();
  c.dts = dts.data(); c.incumbent = inc.data(); c.lbound = lb.data(); c.closed = closed.data(); c.roots = roots; c.n_par = n_par.data();
  c.n_leaves = n_leaves.data(); c.flags = flags.data(); c.nodes = nodes.data(); c.status = status;
  launch((unsigned)(n_prob + 63) / 64, 64, [&] { fqb::fq_bnb_roots_kernel(c); });
  for (int j = 0; j < n_prob; j++) n_roots[j] = n_par[j];
}

// The exact stage of one sweep for n_prob corridors (exact_stage of fq_pair_capi.cu): the list winners (win_* of
// fq_select_multi_kernel) in, the exact winners out.  cand_ofs / cand_dt: the sweep's candidates (factor-major, |L_c| per
// factor).  keep_ties and the pools as the chain uses them.  Returns 0, or < 0 when the shape is not instantiated.
int emu_exact_stage(int N, int ff, const double* TZ, const double* T0, const double* FT, int n_prob, const double* x0, const double* xf,
                    const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab, int max_faces, int max_poly_faces,
                    double row_tol, long long all_limit, const int* cand_ofs, const double* cand_dt, int n_fac, int cap, int cpc,
                    int* win_idx, double* win_cost, double* win_dt, uint8_t* win_sig, uint8_t* changed, int* exact_out, long long* nodes_out)
{
  const int stride = std::max(n_fac, 1), leaf_cap = 4096, n = n_prob;
  const size_t cells = (size_t)n * stride;
  std::vector<double> dts(cells);
  std::vector<unsigned long long> inc(cells), lb(cells);
  std::vector<uint8_t> closed(cells), keep_sig((size_t)n * N);
  std::vector<int> keep_idx(n);
  std::vector<double> keep_cost(n), keep_dt(n);
  std::vector<int> roots(cells), n_par(2 * (size_t)n), n_leaves(n), flags(2 * (size_t)n);
  std::vector<long long> nodes(n);
  std::vector<uint8_t> status(n);
  std::vector<fqb::LeafRec> leaves((size_t)n * leaf_cap);
  const size_t nb = ff ? (N == 6 ? fqb::node_bytes<fqt::Dims<6, true>>() : 0) : (N == 6 ? fqb::node_bytes<fqt::Dims<6, false>>() : 0);
  if (!nb) return -1;
  std::vector<unsigned char> pool0((size_t)n * cap * nb), pool1((size_t)n * cap * nb);
  FqBnbChainArgs c{};
  c.n_prob = n; c.N = N; c.force_final = ff; c.stride = stride; c.max_faces = std::min(max_faces, 2047); c.tree_ok = 1;
  c.all_limit = all_limit; c.poly_ofs = poly_ofs; c.face_ofs = face_ofs; c.Ab = Ab; c.x0 = x0; c.xf = xf; c.row_tol = row_tol;
  c.cand_ofs = cand_ofs; c.cand_dt = cand_dt; c.n_fac = n_fac; c.n_fac_j = nullptr;
  c.win_idx = win_idx; c.win_cost = win_cost; c.win_dt = win_dt; c.win_sig = win_sig;
  c.dts = dts.data(); c.incumbent = inc.data(); c.lbound = lb.data(); c.closed = closed.data(); c.roots = roots.data();
  c.keep_idx = keep_idx.data(); c.keep_cost = keep_cost.data(); c.keep_dt = keep_dt.data(); c.keep_sig = keep_sig.data(); c.n_par = n_par.data();
  c.n_leaves = n_leaves.data(); c.flags = flags.data(); c.nodes = nodes.data(); c.leaves = leaves.data(); c.leaf_cap = leaf_cap;
  c.status = status.data(); c.changed = changed; c.exact_out = exact_out; c.nodes_out = nodes_out;
  launch((unsigned)(n + 63) / 64, 64, [&] { fqb::fq_bnb_roots_kernel(c); });
  fqb::BnbArgs b{};
  fill_plan(Plan{ N, ff, TZ, T0, FT }, &b.k);
  b.k.n_prob = n; b.k.x0 = x0; b.k.xf = xf; b.k.lim = lim; b.k.poly_ofs = poly_ofs; b.k.face_ofs = face_ofs; b.k.Ab = Ab;
  b.k.max_faces = c.max_faces; b.k.item_cap = N * std::min(max_poly_faces, c.max_faces); b.k.row_tol = row_tol;
  b.n_dt = stride; b.dts = dts.data(); b.roots = roots.data(); b.cap = cap; b.incumbent = inc.data(); b.leaves = leaves.data();
  b.n_leaves = n_leaves.data(); b.leaf_cap = leaf_cap; b.flags = flags.data(); b.nodes = nodes.data(); b.keep_ties = 1;
  b.lbound = lb.data(); b.closed = closed.data(); b.cpc = cpc;
  unsigned char* pools[2] = { pool0.data(), pool1.data() };
  for (int depth = 0; depth < N; depth++)
  {
    b.depth = depth;
    b.n_parents = n_par.data() + (size_t)n * (depth & 1);
    b.n_children = n_par.data() + (size_t)n * ((depth + 1) & 1);
    b.parents = pools[depth & 1]; b.children = pools[(depth + 1) & 1];
    std::fill(b.n_children, b.n_children + n, 0);
    if (int rc = level(b)) return rc;
    if (depth == 0) launch((unsigned)(n + 63) / 64, 64, [&] { fqb::fq_bnb_certify_kernel(c); });
  }
  launch((unsigned)(n + 63) / 64, 64, [&] { fqb::fq_bnb_resolve_kernel(c); });
  return 0;
}

// fq_bnb_fallback_kernel then fq_bnb_adopt_kernel on given arrays (win_* and changed / exact in place): `feasible` stands
// for the winners' coefficient solve, redo_coeffs for the second solve of the reverted corridors
void emu_fallback(int n_prob, int N, int* win_idx, double* win_cost, double* win_dt, uint8_t* win_sig, const int* keep_idx,
                  const double* keep_cost, const double* keep_dt, const uint8_t* keep_sig, uint8_t* changed, int* exact_out,
                  const uint8_t* feasible, double* redo_dt, const double* redo_coeffs, double* coeffs)
{
  FqBnbChainArgs c{};
  c.n_prob = n_prob; c.N = N; c.win_idx = win_idx; c.win_cost = win_cost; c.win_dt = win_dt; c.win_sig = win_sig;
  c.keep_idx = const_cast<int*>(keep_idx); c.keep_cost = const_cast<double*>(keep_cost); c.keep_dt = const_cast<double*>(keep_dt);
  c.keep_sig = const_cast<uint8_t*>(keep_sig); c.changed = changed; c.exact_out = exact_out;
  launch((unsigned)(n_prob + 63) / 64, 64, [&] { fqb::fq_bnb_fallback_kernel(c, feasible, redo_dt); });
  launch((unsigned)n_prob, 128, [&] { fqb::fq_bnb_adopt_kernel(n_prob, N, redo_dt, redo_coeffs, coeffs); });
}

// fq_gen_new_traj_exact's tree for one corridor, restated around the same kernel: roots by the presolve up to n_search
// time allocations, incumbents given (+inf, or the list winner's cost at its index), strict pruning, one warp per child,
// the counts read between levels.  -> the incumbents, the stored leaves (n_leaves), exact (0: cut) and the nodes.
int emu_strict_tree(int N, int ff, const double* TZ, const double* T0, const double* FT, const double* x0, const double* xf,
                    const double* lim, int P, const int* face_ofs, const double* Ab, int max_poly_faces, double row_tol, int n_dt,
                    const double* dts, int n_search, unsigned long long* incumbent, int leaf_cap, void* leaves_out, int* n_leaves_out,
                    int* exact_out, long long* nodes_out)
{
  const int cap = 65536;
  const size_t nb = ff ? (N == 6 ? fqb::node_bytes<fqt::Dims<6, true>>() : 0) : (N == 6 ? fqb::node_bytes<fqt::Dims<6, false>>() : 0);
  if (!nb) return -1;
  std::vector<int> roots(n_dt), cnt(5, 0);
  int n_roots = 0;
  for (int d = 0; d < n_search; d++)
    if (fqs::root_possible(P, face_ofs, Ab, x0, xf, ff, dts[d], row_tol)) roots[n_roots++] = d;
  cnt[0] = n_roots;
  const int po[2] = { 0, P };
  std::vector<unsigned char> pool0((size_t)cap * nb), pool1((size_t)cap * nb);
  fqb::BnbArgs b{};
  fill_plan(Plan{ N, ff, TZ, T0, FT }, &b.k);
  b.k.n_prob = 1; b.k.x0 = x0; b.k.xf = xf; b.k.lim = lim; b.k.poly_ofs = po; b.k.face_ofs = face_ofs; b.k.Ab = Ab;
  b.k.max_faces = face_ofs[P] - face_ofs[0]; b.k.item_cap = N * max_poly_faces; b.k.row_tol = row_tol;
  b.n_dt = n_dt; b.dts = dts; b.roots = roots.data(); b.cap = cap; b.incumbent = incumbent;
  b.leaves = static_cast<fqb::LeafRec*>(leaves_out); b.n_leaves = cnt.data() + 2; b.leaf_cap = leaf_cap; b.flags = cnt.data() + 3;
  b.nodes = nullptr; b.keep_ties = 0;
  unsigned char* pools[2] = { pool0.data(), pool1.data() };
  long long nodes = 0;
  int n_par = n_roots, exact = 1;
  for (int depth = 0; depth < N && n_par > 0; depth++)
  {
    b.depth = depth; b.cpc = (n_par * P + fqb::W - 1) / fqb::W;
    b.n_parents = cnt.data() + (depth & 1); b.n_children = cnt.data() + ((depth + 1) & 1);
    b.parents = pools[depth & 1]; b.children = pools[(depth + 1) & 1];
    *b.n_children = 0;
    if (int rc = level(b)) return rc;
    nodes += (long long)n_par * P;
    if (cnt[3] || cnt[4]) { exact = 0; break; }
    n_par = cnt[(depth + 1) & 1];
  }
  *exact_out = exact; *nodes_out = nodes; *n_leaves_out = std::min(cnt[2], leaf_cap);
  return 0;
}
}
