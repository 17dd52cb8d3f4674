// Polygon ground-truth masks on the GPU (SURVEY.md 3(A) step 4, DESIGN.md f-4): PolygonMasks.crop_and_resize
// (detectron2/structures/masks.py:396-420 -> rasterize_polygons_within_box, :39-85) and polygons_to_bitmask /
// BitMasks.from_polygon_masks (:22-36, :166-180), bit for bit.  The reference copies the boxes to the host and rasterizes
// every proposal's polygons with pycocotools in a Python loop; here one CTA rasterizes one tile of one instance from the
// packed batch (polygon_raster.cuh).  Compiled with -fmad=false: every double operation of the reference is rounded alone.
#include <climits>

#include "common.cuh"
#include "polygon_raster.cuh"

namespace {

constexpr int kPolyThreads = 256;
constexpr int kBitmaskTileCols = 128;  // full-image tiles: 128 columns x 256 rows

__global__ void __launch_bounds__(kPolyThreads) polygons_crop_kernel(PolyBatch pb, const float* __restrict__ boxes,
                                                                     const long long* __restrict__ mask_index, int S,
                                                                     unsigned char* __restrict__ out) {
  __shared__ PolyTileSmem sm;
  const long long k = blockIdx.x;
  PolyTransform tf;
  const bool box_ok = poly_box_transform(boxes + k * 4, S, tf);
  const long long g = !box_ok ? -1 : mask_index ? mask_index[k] : k;
  poly_raster_instance(pb, g, tf, S, S, 0, S, 0, S, sm);
  unsigned char* o = out + (size_t)k * S * S;
  for (int i = threadIdx.x; i < S * S; i += kPolyThreads) {
    const int r = i / S;
    o[i] = poly_mask_bit(sm, r, i - r * S);
  }
}

__global__ void __launch_bounds__(kPolyThreads) polygons_bitmask_kernel(PolyBatch pb, int H, int W, int tiles_x,
                                                                        int tiles_y, unsigned char* __restrict__ out) {
  __shared__ PolyTileSmem sm;
  const int tile = blockIdx.x % (tiles_x * tiles_y), g = blockIdx.x / (tiles_x * tiles_y);
  const int c0 = (tile % tiles_x) * kBitmaskTileCols, r0 = (tile / tiles_x) * D2B_POLY_TILE;
  const int tc = min(kBitmaskTileCols, W - c0), tr = min(D2B_POLY_TILE, H - r0);
  poly_raster_instance(pb, g, PolyTransform{0.0, 0.0, 1.0, 1.0}, H, W, c0, tc, r0, tr, sm);
  unsigned char* o = out + (size_t)g * H * W;
  for (int i = threadIdx.x; i < tc * tr; i += kPolyThreads) {
    const int r = i / tc, c = i - r * tc;
    o[(size_t)(r0 + r) * W + c0 + c] = poly_mask_bit(sm, r, c);
  }
}

}  // namespace

D2B_API int d2b_polygons_crop_and_resize(const double* coords, int V, const int* poly_start, int P, const int* inst_start,
                                         int G, const float* boxes, const int64_t* mask_index, int K, int S, uint8_t* out,
                                         void* stream) {
  if (K < 0 || S < 1 || S > D2B_POLYGON_MAX_S || V < 0 || P < 0 || G < 0) return D2B_EINVAL;
  if (K == 0) return D2B_OK;
  if (!boxes || !out || (G > 0 && !inst_start) || (P > 0 && !poly_start) || (V > 0 && !coords)) return D2B_EINVAL;
  polygons_crop_kernel<<<K, kPolyThreads, 0, (cudaStream_t)stream>>>(PolyBatch{coords, V, poly_start, P, inst_start, G},
                                                                      boxes, (const long long*)mask_index, S, out);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_polygons_to_bitmask(const double* coords, int V, const int* poly_start, int P, const int* inst_start,
                                    int G, int H, int W, uint8_t* out, void* stream) {
  if (V < 0 || P < 0 || G < 0 || H < 1 || W < 1 || (long long)H * W > INT_MAX) return D2B_EINVAL;
  const long long tiles = (long long)d2b_cdiv(W, kBitmaskTileCols) * d2b_cdiv(H, D2B_POLY_TILE);
  if ((long long)G * tiles > INT_MAX) return D2B_EINVAL;
  if (G == 0) return D2B_OK;
  if (!out || !inst_start || (P > 0 && !poly_start) || (V > 0 && !coords)) return D2B_EINVAL;
  polygons_bitmask_kernel<<<(unsigned)(G * tiles), kPolyThreads, 0, (cudaStream_t)stream>>>(
      PolyBatch{coords, V, poly_start, P, inst_start, G}, H, W, d2b_cdiv(W, kBitmaskTileCols), d2b_cdiv(H, D2B_POLY_TILE),
      out);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
