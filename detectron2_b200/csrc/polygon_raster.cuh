// Polygon rasterizer of pycocotools' rleFrPoly + merge + decode, bit for bit, one CTA per output tile (DESIGN.md f-4).
//
// rleFrPoly snaps every vertex to the 5x lattice, X = (int)(5 x + 0.5), walks each edge of the closed ring with a DDA and
// keeps the consecutive point pairs whose lower u is 5c + 2 for a column c in [0, w): each such pair toggles the pixel
// parity at row ceil(clamp((min v + 0.5) / 5 - 0.5, 0, h)) of column c.  Three facts make that walk unnecessary here:
//   * u is monotone along an edge and a kept pair steps from 5c + 2 to 5c + 3, so an edge toggles each column at most
//     once; that toggle is found in closed form, with the DDA's own expressions evaluated at the two points of the step;
//   * pairs that straddle two edges differ only at negative u and are never kept;
//   * every column receives an even number of toggles, so columns are independent: pixel (r, c) is the parity of the
//     column's toggles at rows <= r, and a toggle at row h never shows.
// An instance is the union of its polygons' masks.  Every double operation here must be rounded on its own (the files
// that include this header are compiled with -fmad=false).
#pragma once
#include <stdint.h>

#define D2B_POLY_TILE 256  // columns and rows of one CTA's tile
#define D2B_POLY_WORDS (D2B_POLY_TILE / 32)

// A batch's polygons, as polygon_masks.pack_polygons lays them out: vertices coords[V][2] (x, y), polygon p = vertices
// [poly_start[p], poly_start[p+1]), instance g = polygons [inst_start[g], inst_start[g+1]).
struct PolyBatch {
  const double* coords;
  int V;
  const int* poly_start;
  int P;
  const int* inst_start;
  int G;
};

// x' = (x - ox) * rx, y' = (y - oy) * ry: rasterize_polygons_within_box's shift and scale, or the identity (0, 1).
struct PolyTransform {
  double ox, oy, rx, ry;
};

struct PolyTileSmem {
  uint32_t tog[D2B_POLY_TILE * D2B_POLY_WORDS];   // the current polygon's toggles, column-major, D2B_POLY_WORDS per column
  uint32_t mask[D2B_POLY_TILE * D2B_POLY_WORDS];  // the union of the instance's polygons so far, same layout
  uint32_t carry[D2B_POLY_TILE];                  // parity of each column's toggles in the rows above the tile
};

// The lattice coordinate (int)(5 x' + 0.5); false when it is not finite or not inside (-2^30, 2^30) (the cast is undefined
// behaviour in the reference for the first, and the edge arithmetic below stays inside int for the second).
__device__ __forceinline__ bool poly_snap(double x, double o, double r, int& X) {
  const double v = 5.0 * ((x - o) * r) + 0.5;
  if (!(fabs(v) < 1073741824.0)) return false;
  X = (int)v;
  return true;
}

__device__ __forceinline__ long long poly_floor_div5(long long a) { return a >= 0 ? a / 5 : -((-a + 4) / 5); }

// rleFrPoly's row of a toggle whose pair has lower v = vm, on an h-row grid.
__device__ __forceinline__ int poly_toggle_row(int vm, int h) {
  double yd = ((double)vm + .5) / 5.0 - .5;
  yd = yd < 0 ? 0 : (yd > (double)h ? (double)h : yd);
  return (int)ceil(yd);
}

// Calls emit(c, vm) for the toggle the edge (xs, ys) -> (xe, ye) puts in each column c of [c_lo, c_hi] (vm: the pair's
// lower v).  The same points as the DDA: dx, dy, flip and the slope s exactly as rleFrPoly computes them.
template <class Emit>
__device__ __forceinline__ void poly_edge_toggles(int xs, int ys, int xe, int ye, long long c_lo, long long c_hi,
                                                  Emit&& emit) {
  const int dx = abs(xe - xs), dy = abs(ys - ye);
  const bool flip = (dx >= dy && xs > xe) || (dx < dy && ys > ye);
  if (flip) {
    int t = xs;
    xs = xe;
    xe = t;
    t = ys;
    ys = ye;
    ye = t;
  }
  if (dx >= dy) {
    if (dx == 0) return;  // a repeated vertex: one point, no pair (its 0/0 slope is never evaluated)
    // u = t + xs: the pair (t, t + 1) is kept for t = 5c + 2 - xs, 0 <= t < dx
    const double s = (double)(ye - ys) / dx;
    const long long c0 = max(c_lo, -poly_floor_div5(-(long long)xs + 2)), c1 = min(c_hi, poly_floor_div5((long long)xe - 3));
    for (long long c = c0; c <= c1; ++c) {
      const int t = (int)(5 * c + 2 - xs);
      const int v0 = (int)(ys + s * t + .5), v1 = (int)(ys + s * (t + 1) + .5);
      emit((int)c, min(v0, v1));
    }
  } else {
    // v = t + ys, u(t) = (int)(xs + s t + 0.5), |s| < 1: u is monotone in t and steps by at most 1
    const double s = (double)(xe - xs) / dy;
    auto u = [&](int t) { return (int)(xs + s * t + .5); };
    const int ua = u(0), ub = u(dy);
    const bool up = ub > ua;
    const long long lo = min(ua, ub), hi = max(ua, ub);
    const long long c0 = max(c_lo, -poly_floor_div5(-lo + 2)), c1 = min(c_hi, poly_floor_div5(hi - 3));
    for (long long c = c0; c <= c1; ++c) {
      // the step between t - 1 and t that crosses from 5c + 2 to 5c + 3 (up) or back (down): the first t in [1, dy] with
      // u(t) >= 5c + 3 (up) or u(t) <= 5c + 2 (down).  u(0) is on the other side, u(dy) on this one.  The estimate only
      // seeds the search; the exact, monotone u decides.
      const int m = (int)(5 * c + (up ? 3 : 2));
      auto past = [&](int t) { return up ? u(t) >= m : u(t) <= m; };
      double est = ceil(((double)m - (up ? 0.5 : -0.5) - xs) / s);
      est = fmin(fmax(est, 1.0), (double)dy);
      int t = (int)est;
      while (t > 1 && past(t - 1)) --t;
      while (t < dy && !past(t)) ++t;
      if (min(u(t - 1), u(t)) == 5 * c + 2) emit((int)c, ys + t - 1);
    }
  }
}

// Rasterizes instance g of `pb` into s.mask for the tile of columns [c0, c0 + tc) and rows [r0, r0 + tr) (tc, tr <=
// D2B_POLY_TILE) of an h x w grid, after `tf`.  Bit (r - r0) & 31 of s.mask[(c - c0) * D2B_POLY_WORDS + ((r - r0) >> 5)] is
// pixel (r, c); bits past row r0 + tr - 1 are unspecified.  Every thread of the CTA calls it with the same arguments; it
// ends with a barrier.
// Contracts beyond the reference: g outside [0, G), an instance range out of order or past P, gives all zeros; a polygon
// range out of order or past V is empty; a polygon with a non-finite or out-of-range lattice coordinate adds nothing.
__device__ inline void poly_raster_instance(const PolyBatch& pb, long long g, const PolyTransform& tf, int h, int w, int c0,
                                     int tc, int r0, int tr, PolyTileSmem& s) {
  const int tid = threadIdx.x, nt = blockDim.x, nw = (tr + 31) >> 5;
  for (int i = tid; i < tc * D2B_POLY_WORDS; i += nt) {
    s.mask[i] = 0u;
    s.tog[i] = 0u;
  }
  for (int i = tid; i < tc; i += nt) s.carry[i] = 0u;
  __syncthreads();
  if (g < 0 || g >= pb.G) return;
  const int pa = pb.inst_start[g], pe = pb.inst_start[g + 1];
  if (pa < 0 || pe > pb.P || pa > pe) return;
  const long long c_lo = c0, c_hi = (long long)min(c0 + tc, w) - 1;
  for (int p = pa; p < pe; ++p) {
    const int va = pb.poly_start[p], ve = pb.poly_start[p + 1];
    if (va < 0 || ve > pb.V || ve <= va) continue;
    const int n = ve - va;
    const double* __restrict__ xy = pb.coords + (size_t)va * 2;
    bool bad = false;
    for (int j = tid; j < n; j += nt) {
      int X, Y;
      bad |= !poly_snap(xy[2 * j], tf.ox, tf.rx, X) || !poly_snap(xy[2 * j + 1], tf.oy, tf.ry, Y);
    }
    if (__syncthreads_or(bad)) continue;
    for (int j = tid; j < n; j += nt) {
      const int j1 = j + 1 == n ? 0 : j + 1;
      int xs, ys, xe, ye;
      poly_snap(xy[2 * j], tf.ox, tf.rx, xs);
      poly_snap(xy[2 * j + 1], tf.oy, tf.ry, ys);
      poly_snap(xy[2 * j1], tf.ox, tf.rx, xe);
      poly_snap(xy[2 * j1 + 1], tf.oy, tf.ry, ye);
      poly_edge_toggles(xs, ys, xe, ye, c_lo, c_hi, [&](int c, int vm) {
        const int r = poly_toggle_row(vm, h) - r0, cc = c - c0;
        if (r < 0)
          atomicXor(&s.carry[cc], 1u);
        else if (r < tr)
          atomicXor(&s.tog[cc * D2B_POLY_WORDS + (r >> 5)], 1u << (r & 31));
      });
    }
    __syncthreads();
    for (int cc = tid; cc < tc; cc += nt) {  // prefix XOR down the column, OR into the instance
      uint32_t par = s.carry[cc] ? 0xffffffffu : 0u;
      for (int wd = 0; wd < nw; ++wd) {
        uint32_t x = s.tog[cc * D2B_POLY_WORDS + wd];
        x ^= x << 1;
        x ^= x << 2;
        x ^= x << 4;
        x ^= x << 8;
        x ^= x << 16;
        x ^= par;
        par = (x >> 31) ? 0xffffffffu : 0u;
        s.mask[cc * D2B_POLY_WORDS + wd] |= x;
        s.tog[cc * D2B_POLY_WORDS + wd] = 0u;
      }
      s.carry[cc] = 0u;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ bool poly_mask_bit(const PolyTileSmem& s, int r, int c) {
  return (s.mask[c * D2B_POLY_WORDS + (r >> 5)] >> (r & 31)) & 1u;
}

// rasterize_polygons_within_box's transform of a float32 proposal box for an S x S grid.  false for a non-finite box.
// w = x1 - x0 in fp32; ratio = S / w in fp32 when w >= 0.1 (max(w, 0.1) picks w: for a float32 w, w < 0.1 in float64 iff
// w < 0.1f), else S / 0.1 in float64; the polygons are float64, so the shift and the scale are float64 operations.
__device__ __forceinline__ bool poly_box_transform(const float* b, int S, PolyTransform& tf) {
  if (!(isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]) && isfinite(b[3]))) return false;
  const float w = b[2] - b[0], h = b[3] - b[1];
  tf.ox = (double)b[0];
  tf.oy = (double)b[1];
  tf.rx = w >= 0.1f ? (double)((float)S / w) : (double)S / 0.1;
  tf.ry = h >= 0.1f ? (double)((float)S / h) : (double)S / 0.1;
  return true;
}
