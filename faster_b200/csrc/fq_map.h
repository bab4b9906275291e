// The indexed map of the chained replan (fq_map_* and fq_replan_pairs_map*, include/faster_b200.h) as the kernels read it.
//
// A map holds the occupied cloud O and the unknown cloud U of one mapper message (Faster::updateMap, faster.cpp:99-137).
// Each cloud is bucketed into one uniform grid of cells shared by both: the cloud's points sorted by (cell, index), their
// original indices beside them, and the first sorted point of every cell (CSR over the cells, n_cells + 1 entries).  The
// cells of one (z, y) row are consecutive, so the points of a run of cells along x are one contiguous range.
//
// The cell of a point is floor((p - origin) / cell) per axis, clamped to the grid.  Rounding of (p - origin) / cell is
// monotone in p, so lo <= p <= hi puts p's cell between the cells of lo and hi: the cell ranges below are conservative.
#pragma once
#include "fq_dtinit.h"

struct FqMapGrid
{
  double origin[3];        // the smallest coordinates of the map's finite points (0 for an empty map)
  double cell;             // the cell edge
  int dims[3];             // cells along x, y, z
  int n_cells;             // dims[0] * dims[1] * dims[2]
};

struct FqMapCloud
{
  const double* xyz;       // n x 3, sorted by (cell, index)
  const int* idx;          // n: each sorted point's index in its cloud
  const int* start;        // n_cells + 1: cell c holds sorted points start[c] .. start[c+1]-1
  int n;                   // points (non-finite ones sort past start[n_cells] and are never read)
};

// one map as a submission reads it: its grid and its two clouds.  It lives in device memory at one address for the map's
// whole life, and every update rewrites all of it on the update's stream (counts and array addresses included), so a
// submission -- or a CUDA graph replayed later -- always reads the map's last update.
struct FqMapDev
{
  FqMapGrid grid;
  FqMapCloud unk, occ;
};

// the most cells a map of n points may have: a grid that would need more doubles the cell edge (FQ_MAP_CELL_EDGE) until it
// does not
inline long long fq_map_cell_limit(long long n)
{
  const long long c = n * 4 > (1LL << 16) ? n * 4 : (1LL << 16);
  return c < (1LL << 26) ? c : (1LL << 26);
}

// the cell of coordinate v along one axis
FQ_HD int fq_map_axis(double v, double origin, double cell, int dim)
{
  const double t = floor(FQ_DIV(FQ_SUB(v, origin), cell));
  return t < 0 ? 0 : (t > (double)(dim - 1) ? dim - 1 : (int)t);
}

// the cells [c0, c1] (per axis) that can hold a point p with lo <= p <= hi
FQ_HD void fq_map_range(const FqMapGrid& g, const double* lo, const double* hi, int* c0, int* c1)
{
  for (int k = 0; k < 3; k++)
  {
    c0[k] = fq_map_axis(lo[k], g.origin[k], g.cell, g.dims[k]);
    c1[k] = fq_map_axis(hi[k], g.origin[k], g.cell, g.dims[k]);
  }
}

// the sorted points of row r (0 .. rows-1) of the cell range [c0, c1]: one run of cells along x
FQ_HD void fq_map_row(const FqMapGrid& g, const FqMapCloud& c, const int* c0, const int* c1, int r, int* b, int* e)
{
  const int ny = c1[1] - c0[1] + 1;
  const int z = c0[2] + r / ny, y = c0[1] + r % ny;
  const int base = (z * g.dims[1] + y) * g.dims[0];
  *b = c.start[base + c0[0]];
  *e = c.start[base + c1[0] + 1];
}
