// Panoptic FPN inference: the semantic labels and the thing / stuff combine of PanopticFPN.inference
// (detectron2/modeling/meta_arch/panoptic_fpn.py:159-179), for all images of a batch without host reads.
//
// d2b_sem_seg_labels replaces sem_seg_postprocess (modeling/postprocessing.py:77-100) + argmax(dim=0): one thread per
// output pixel evaluates PyTorch's CUDA upsample_bilinear2d of the crop channel by channel and keeps the running argmax,
// so the C x H x W fp32 map of the reference (230 MB at 54 x 800 x 1333) is never written or read back.
//
// d2b_panoptic_combine replaces combine_semantic_and_instance_outputs (panoptic_fpn.py:184-269):
//   panoptic_pack_kernel    one CTA per instance (all images): the uint8 mask packed into bit rows [R, H, ceil(W/32)]
//                           with one warp ballot per 32 pixels; the instance's area and bounding rectangle (rows, words)
//   panoptic_walk_kernel    one CTA per image: the instances ranked by counting, then walked in that order against a
//                           painted bitmap (L2-resident: 134 KB at 800 x 1333) -- popc(mask & painted) over the instance's
//                           rectangle, one block reduction, the same decision in every thread, then the new bits painted
//                           and their ids written; also clears the image's histogram, presence and status
//   panoptic_hist_kernel    whole grid: label presence and the histogram of the unpainted pixels (shared-memory counts,
//                           then integer atomics: deterministic); labels outside [0, C) flag the image's status
//   panoptic_stuff_kernel   whole grid: every CTA derives the stuff id table from the histogram (a prefix over the labels),
//                           writes the stuff ids / zeros of the unpainted pixels; CTA 0 of an image writes the stuff
//                           records, zeroes the unused slots and the segment count
// Every decision is integer arithmetic or a double comparison, so the outputs are bitwise reproducible.
//
// This file is compiled with -fmad=false: the fused multiply-adds of the bilinear interpolation are written as __fmaf_rn
// exactly where PyTorch's sm_90 build of upsample_bilinear2d_out_frame<T, float> contracts (its SASS): the source index
// scale * (d + 0.5) - 0.5, and each two-term sum a * x + b * y as fma(a, x, b * y) with the right product rounded on its own.
#include <algorithm>
#include <climits>

#include "bilinear.cuh"
#include "common.cuh"

namespace {

constexpr int kLabelThreads = 256;
constexpr int kPackThreads = 512;
constexpr int kWalkThreads = 1024;
constexpr int kPixThreads = 256;
constexpr int kPixPerThread = 16;
constexpr int kPixChunk = kPixThreads * kPixPerThread;  // pixels per CTA of the histogram and stuff launches
constexpr int kInstInts = 5;                             // per instance: area, y0, y1, x0, x1 (x in words, ends exclusive)
constexpr size_t kAlign = 256;

__host__ __device__ inline size_t align_up(size_t v) { return (v + kAlign - 1) / kAlign * kAlign; }
__host__ __device__ inline int words_per_row(int W) { return (W + 31) >> 5; }

// ---- semantic labels (taps: bilinear.cuh) -----------------------------------------------------------------------------
// torch.argmax on CUDA: v replaces the running best when it is a NaN and the best is not, or when neither is a NaN and
// v is larger; ties keep the earlier channel (-0.0 == +0.0 compares equal).
__device__ __forceinline__ bool beats(float v, float best) {
  return (v != v) ? (best == best) : (best == best && v > best);
}

template <int DT>
__global__ void __launch_bounds__(kLabelThreads) sem_seg_labels_kernel(const typename Elem<DT>::T* __restrict__ logits,
                                                                       int C, int Hp, int Wp,
                                                                       const __grid_constant__ d2b_sem_seg_images img) {
  const int n = blockIdx.y;
  const int H = img.H[n], W = img.W[n];
  const long long p = (long long)blockIdx.x * kLabelThreads + threadIdx.x;
  if (p >= (long long)H * W) return;
  const int oy = (int)(p / W), ox = (int)(p - (long long)oy * W);
  const int h = img.h[n], w = img.w[n];
  const size_t plane = (size_t)Hp * Wp;
  const typename Elem<DT>::T* __restrict__ src = logits + (size_t)n * C * plane;
  float best = 0.f;
  int arg = 0;
  if (h == H && w == W) {  // PyTorch's special case: the crop is copied, no arithmetic
    const size_t off = (size_t)oy * Wp + ox;
    for (int c = 0; c < C; ++c) {
      const float v = Elem<DT>::ld(src + c * plane + off);
      if (c == 0 || beats(v, best)) best = v, arg = c;
    }
  } else {
    // area_pixel_compute_scale: (float)input_size / output_size, computed by torch on the host
    const Tap ty = make_tap(__fdiv_rn((float)h, (float)H), oy, h);
    const Tap tx = make_tap(__fdiv_rn((float)w, (float)W), ox, w);
    const size_t r0 = (size_t)ty.i0 * Wp, r1 = (size_t)ty.i1 * Wp;
    for (int c = 0; c < C; ++c) {
      const typename Elem<DT>::T* s = src + c * plane;
      const float a = Elem<DT>::ld(s + r0 + tx.i0), b = Elem<DT>::ld(s + r0 + tx.i1);
      const float d = Elem<DT>::ld(s + r1 + tx.i0), e = Elem<DT>::ld(s + r1 + tx.i1);
      const float top = __fmaf_rn(tx.l0, a, __fmul_rn(tx.l1, b));
      const float bot = __fmaf_rn(tx.l0, d, __fmul_rn(tx.l1, e));
      const float acc = __fmaf_rn(ty.l0, top, __fmul_rn(ty.l1, bot));
      const float v = Elem<DT>::ld(Elem<DT>::st(acc));  // odata[...] = static_cast<scalar_t>(val)
      if (c == 0 || beats(v, best)) best = v, arg = c;
    }
  }
  img.labels[n][p] = arg;
}

// ---- combine ----------------------------------------------------------------------------------------------------------
struct PanArgs {
  d2b_panoptic_images img;
  size_t off_bits[D2B_MAX_IMAGES];   // [R, H, Wb] uint32
  size_t off_paint[D2B_MAX_IMAGES];  // [H, Wb] uint32
  size_t off_inst[D2B_MAX_IMAGES];   // [R, kInstInts] int32
  size_t off_hist[D2B_MAX_IMAGES];   // [C] unpainted counts, [C] presence, [1] thing segments
  int inst_start[D2B_MAX_IMAGES + 1];  // prefix of R over the images (pack grid)
  int N, C, S;
  const int64_t* num_instances;
  double overlap, stuff_thresh, score_thresh;
  int64_t* num_segments;
  int64_t* seg_info;
  float* seg_score;
  int* status;
  unsigned char* ws;
};

template <class T>
__device__ __forceinline__ T* ws_at(const PanArgs& a, size_t off) {
  return reinterpret_cast<T*>(a.ws + off);
}

__device__ __forceinline__ int live_count(const PanArgs& a, int n) {
  const int R = a.img.R[n];
  if (!a.num_instances) return R;
  const long long c = a.num_instances[n];
  return c < 0 ? 0 : (c > R ? R : (int)c);
}

__global__ void __launch_bounds__(kPackThreads) panoptic_pack_kernel(const __grid_constant__ PanArgs a) {
  __shared__ int s_area, s_y0, s_y1, s_x0, s_x1;
  const int g = blockIdx.x;
  int n = 0;
  while (g >= a.inst_start[n + 1]) ++n;
  const int i = g - a.inst_start[n];
  if (i >= live_count(a, n)) return;  // a padding row: never read
  const int H = a.img.H[n], W = a.img.W[n], Wb = words_per_row(W);
  if (threadIdx.x == 0) s_area = 0, s_y0 = INT_MAX, s_y1 = -1, s_x0 = INT_MAX, s_x1 = -1;
  __syncthreads();
  const uint8_t* __restrict__ mask = a.img.masks[n] + (size_t)i * H * W;
  uint32_t* __restrict__ bits = ws_at<uint32_t>(a, a.off_bits[n]) + (size_t)i * H * Wb;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int area = 0, y0 = INT_MAX, y1 = -1, x0 = INT_MAX, x1 = -1;
  for (int y = warp; y < H; y += kPackThreads / 32) {
    const uint8_t* row = mask + (size_t)y * W;
    for (int w0 = 0; w0 < Wb; w0 += 32) {
      uint32_t mine = 0;
      const int nw = min(32, Wb - w0);
#pragma unroll 8
      for (int j = 0; j < nw; ++j) {  // word w0 + j: lane l holds pixel 32 (w0 + j) + l
        const int x = ((w0 + j) << 5) + lane;
        const uint32_t word = __ballot_sync(0xffffffffu, x < W && row[x] != 0);
        if (lane == j) mine = word;
      }
      if (lane < nw) {
        bits[(size_t)y * Wb + w0 + lane] = mine;
        if (mine) {
          area += __popc(mine);
          y0 = min(y0, y), y1 = max(y1, y);
          x0 = min(x0, w0 + lane), x1 = max(x1, w0 + lane);
        }
      }
    }
  }
  if (area) {
    atomicAdd(&s_area, area);
    atomicMin(&s_y0, y0), atomicMax(&s_y1, y1), atomicMin(&s_x0, x0), atomicMax(&s_x1, x1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int* inst = ws_at<int>(a, a.off_inst[n]) + (size_t)i * kInstInts;
    const bool any = s_area > 0;
    inst[0] = s_area;
    inst[1] = any ? s_y0 : 0, inst[2] = any ? s_y1 + 1 : 0;
    inst[3] = any ? s_x0 : 0, inst[4] = any ? s_x1 + 1 : 0;
  }
}

// j is walked before i: ascending -score, NaN (either sign) last, ties to the lower index
__device__ __forceinline__ bool walked_before(float sj, int j, float si, int i) {
  const bool nj = sj != sj, ni = si != si;
  if (nj || ni) return nj == ni ? j < i : ni;
  return sj > si || (sj == si && j < i);
}

__device__ __forceinline__ int block_sum(int v, int* s_red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();  // s_red may still be read by the previous reduction
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = 0;
#pragma unroll
  for (int k = 0; k < kWalkThreads / 32; ++k) t += s_red[k];
  return t;
}

__global__ void __launch_bounds__(kWalkThreads) panoptic_walk_kernel(const __grid_constant__ PanArgs a) {
  __shared__ float s_score[D2B_PANOPTIC_MAX_INSTANCES];
  __shared__ short s_order[D2B_PANOPTIC_MAX_INSTANCES];
  __shared__ int s_red[kWalkThreads / 32];
  const int n = blockIdx.x, tid = threadIdx.x;
  const int H = a.img.H[n], W = a.img.W[n], Wb = words_per_row(W), C = a.C;
  uint32_t* __restrict__ paint = ws_at<uint32_t>(a, a.off_paint[n]);
  unsigned* __restrict__ hist = ws_at<unsigned>(a, a.off_hist[n]);
  for (long long k = tid; k < (long long)H * Wb; k += kWalkThreads) paint[k] = 0u;
  for (int k = tid; k < 2 * C + 1; k += kWalkThreads) hist[k] = 0u;
  if (tid == 0) a.status[n] = 0;
  const int R = live_count(a, n);
  const float* __restrict__ scores = a.img.scores[n];
  for (int k = tid; k < R; k += kWalkThreads) s_score[k] = scores[k];
  __syncthreads();
  for (int k = tid; k < R; k += kWalkThreads) {  // rank by counting: R <= D2B_PANOPTIC_MAX_INSTANCES
    const float s = s_score[k];
    int rank = 0;
    for (int j = 0; j < R; ++j) rank += walked_before(s_score[j], j, s, k);
    s_order[rank] = (short)k;
  }
  __syncthreads();
  const uint32_t* __restrict__ bits = ws_at<uint32_t>(a, a.off_bits[n]);
  const int* __restrict__ inst = ws_at<int>(a, a.off_inst[n]);
  int32_t* __restrict__ pan = a.img.panoptic[n];
  int64_t* info = a.seg_info + (size_t)n * a.S * 5;
  float* sscore = a.seg_score + (size_t)n * a.S;
  int next_id = 0;
  for (int r = 0; r < R; ++r) {
    const int i = s_order[r];
    const float score = s_score[i];
    if ((double)score < a.score_thresh) break;  // every thread reads the same value: a uniform exit
    const int* q = inst + (size_t)i * kInstInts;
    const int area = q[0];
    if (area == 0) continue;
    const int y0 = q[1], bw = q[4] - q[3], x0 = q[3];
    const int nw = (q[2] - y0) * bw;
    const uint32_t* m = bits + (size_t)i * H * Wb;
    int inter = 0;
    for (int t = tid; t < nw; t += kWalkThreads) {
      const int dy = t / bw;
      const size_t o = (size_t)(y0 + dy) * Wb + x0 + (t - dy * bw);
      inter += __popc(m[o] & paint[o]);
    }
    inter = block_sum(inter, s_red);
    if ((double)inter / (double)area > a.overlap) continue;
    const int id = ++next_id;
    for (int t = tid; t < nw; t += kWalkThreads) {
      const int dy = t / bw, xw = x0 + (t - dy * bw), y = y0 + dy;
      const size_t o = (size_t)y * Wb + xw;
      uint32_t fresh = m[o] & ~paint[o];
      if (!fresh) continue;
      paint[o] |= fresh;
      int32_t* px = pan + (size_t)y * W + (xw << 5);
      while (fresh) {
        const int b = __ffs(fresh) - 1;
        px[b] = id;
        fresh &= fresh - 1;
      }
    }
    if (tid == 0) {
      int64_t* rec = info + (size_t)(id - 1) * 5;
      rec[0] = id, rec[1] = 1, rec[2] = a.img.classes[n][i], rec[3] = i, rec[4] = area - inter;
      sscore[id - 1] = score;
    }
    __syncthreads();  // the next instance's count reads the bits painted here
  }
  if (tid == 0) hist[2 * C] = (unsigned)next_id;
}

__global__ void __launch_bounds__(kPixThreads) panoptic_hist_kernel(const __grid_constant__ PanArgs a) {
  extern __shared__ unsigned s_hist[];  // [C] unpainted counts, [C] presence
  const int n = blockIdx.y, C = a.C;
  const int H = a.img.H[n], W = a.img.W[n], Wb = words_per_row(W);
  const long long p0 = (long long)blockIdx.x * kPixChunk;
  if (p0 >= (long long)H * W) return;
  for (int k = threadIdx.x; k < 2 * C; k += kPixThreads) s_hist[k] = 0u;
  __syncthreads();
  const int64_t* __restrict__ labels = a.img.labels[n];
  const uint32_t* __restrict__ paint = ws_at<uint32_t>(a, a.off_paint[n]);
  const int npix = H * W;
  bool bad = false;
  for (int j = 0; j < kPixPerThread; ++j) {
    const long long p = p0 + (long long)j * kPixThreads + threadIdx.x;
    if (p >= npix) break;
    const long long l = labels[p];
    if (l < 0 || l >= C) {
      bad = true;
      continue;
    }
    s_hist[C + l] = 1u;
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    if (!((paint[(size_t)y * Wb + (x >> 5)] >> (x & 31)) & 1u)) atomicAdd(&s_hist[l], 1u);
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(a.status + n, D2B_PANOPTIC_STATUS_BAD_LABEL);
  unsigned* __restrict__ hist = ws_at<unsigned>(a, a.off_hist[n]);
  for (int k = threadIdx.x; k < C; k += kPixThreads) {
    if (s_hist[k]) atomicAdd(hist + k, s_hist[k]);
    if (s_hist[C + k]) hist[C + k] = 1u;
  }
}

__global__ void __launch_bounds__(kPixThreads) panoptic_stuff_kernel(const __grid_constant__ PanArgs a) {
  extern __shared__ int s_id[];  // [C] the stuff id of every label, 0 = none
  __shared__ int s_tot[32];
  const int n = blockIdx.y, C = a.C;
  const int H = a.img.H[n], W = a.img.W[n], Wb = words_per_row(W);
  const int npix = H * W;
  const long long p0 = (long long)blockIdx.x * kPixChunk;
  if (p0 >= npix) return;
  const unsigned* __restrict__ hist = ws_at<unsigned>(a, a.off_hist[n]);
  const int things = (int)hist[2 * C];
  int base = things;
  for (int c0 = 0; c0 < C; c0 += kPixThreads) {  // stuff ids: a prefix over the labels, ascending
    const int l = c0 + threadIdx.x;
    const bool stuff = l > 0 && l < C && hist[C + l] && !((double)hist[l] < a.stuff_thresh);
    int total;
    const int before = block_exclusive_scan(stuff ? 1 : 0, s_tot, total);
    if (l < C) s_id[l] = stuff ? base + before + 1 : 0;
    base += total;
    __syncthreads();  // s_tot is written again by the next chunk's scan
  }
  const int64_t* __restrict__ labels = a.img.labels[n];
  const uint32_t* __restrict__ paint = ws_at<uint32_t>(a, a.off_paint[n]);
  int32_t* __restrict__ pan = a.img.panoptic[n];
  for (int j = 0; j < kPixPerThread; ++j) {
    const long long p = p0 + (long long)j * kPixThreads + threadIdx.x;
    if (p >= npix) break;
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    if ((paint[(size_t)y * Wb + (x >> 5)] >> (x & 31)) & 1u) continue;  // written by the walk
    const long long l = labels[p];
    pan[p] = (l >= 0 && l < C) ? s_id[l] : 0;
  }
  if (blockIdx.x != 0) return;
  int64_t* info = a.seg_info + (size_t)n * a.S * 5;
  float* sscore = a.seg_score + (size_t)n * a.S;
  for (int l = threadIdx.x; l < C; l += kPixThreads) {
    const int id = s_id[l];
    if (!id) continue;
    int64_t* rec = info + (size_t)(id - 1) * 5;
    rec[0] = id, rec[1] = 0, rec[2] = l, rec[3] = -1, rec[4] = hist[l];
    sscore[id - 1] = 0.f;
  }
  for (long long k = (long long)base * 5 + threadIdx.x; k < (long long)a.S * 5; k += kPixThreads) info[k] = 0;
  for (int k = base + threadIdx.x; k < a.S; k += kPixThreads) sscore[k] = 0.f;
  if (threadIdx.x == 0) a.num_segments[n] = base;
}

bool panoptic_images_ok(const d2b_panoptic_images* img, int N) {
  for (int n = 0; n < N; ++n) {
    const int R = img->R[n], H = img->H[n], W = img->W[n];
    if (H < 1 || W < 1 || (long long)H * W > INT_MAX || R < 0 || R > D2B_PANOPTIC_MAX_INSTANCES) return false;
    if (!img->labels[n] || !img->panoptic[n]) return false;
    if (R > 0 && (!img->scores[n] || !img->classes[n] || !img->masks[n])) return false;
  }
  return true;
}

// Workspace layout (offsets from the 256-byte aligned base); returns the total.  The description must be valid.
size_t panoptic_layout(const d2b_panoptic_images* img, int N, int C, PanArgs* a) {
  size_t off = 0;
  for (int n = 0; n < N; ++n) {
    const size_t H = img->H[n], Wb = words_per_row(img->W[n]), R = img->R[n];
    if (a) a->off_bits[n] = off;
    off = align_up(off + R * H * Wb * 4);
    if (a) a->off_paint[n] = off;
    off = align_up(off + H * Wb * 4);
    if (a) a->off_inst[n] = off;
    off = align_up(off + R * kInstInts * 4);
    if (a) a->off_hist[n] = off;
    off = align_up(off + ((size_t)2 * C + 1) * 4);
  }
  return off;
}

}  // namespace

D2B_API int d2b_sem_seg_labels(const void* logits, int dtype, int N, int C, int Hp, int Wp, const d2b_sem_seg_images* img,
                               void* stream) {
  if (!img || N < 0 || N > D2B_MAX_IMAGES) return D2B_EINVAL;
  if (dtype != D2B_F32 && dtype != D2B_F16 && dtype != D2B_BF16) return D2B_EINVAL;
  if (C < 1 || Hp < 1 || Wp < 1) return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  if (!logits) return D2B_EINVAL;
  long long max_pix = 0;
  for (int n = 0; n < N; ++n) {
    if (img->h[n] < 1 || img->h[n] > Hp || img->w[n] < 1 || img->w[n] > Wp) return D2B_EINVAL;
    if (img->H[n] < 1 || img->W[n] < 1 || (long long)img->H[n] * img->W[n] > INT_MAX || !img->labels[n]) return D2B_EINVAL;
    max_pix = std::max(max_pix, (long long)img->H[n] * img->W[n]);
  }
  const dim3 grid(d2b_cdiv(max_pix, kLabelThreads), N);
  const cudaStream_t st = (cudaStream_t)stream;
  if (dtype == D2B_F32)
    sem_seg_labels_kernel<D2B_F32><<<grid, kLabelThreads, 0, st>>>((const float*)logits, C, Hp, Wp, *img);
  else if (dtype == D2B_F16)
    sem_seg_labels_kernel<D2B_F16><<<grid, kLabelThreads, 0, st>>>((const __half*)logits, C, Hp, Wp, *img);
  else
    sem_seg_labels_kernel<D2B_BF16><<<grid, kLabelThreads, 0, st>>>((const __nv_bfloat16*)logits, C, Hp, Wp, *img);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API size_t d2b_panoptic_workspace_bytes(const d2b_panoptic_images* img, int N, int C) {
  if (!img || N < 0 || N > D2B_MAX_IMAGES || C < 1 || C > D2B_PANOPTIC_MAX_CLASSES) return 0;
  for (int n = 0; n < N; ++n) {
    const int R = img->R[n], H = img->H[n], W = img->W[n];
    if (H < 1 || W < 1 || (long long)H * W > INT_MAX || R < 0 || R > D2B_PANOPTIC_MAX_INSTANCES) return 0;
  }
  return panoptic_layout(img, N, C, nullptr);
}

D2B_API int d2b_panoptic_combine(const d2b_panoptic_images* img, int N, int C, const int64_t* num_instances,
                                 double overlap_threshold, double stuff_area_thresh, double instances_score_thresh,
                                 int64_t* num_segments, int64_t* seg_info, float* seg_score, int* status, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (!img || N < 0 || N > D2B_MAX_IMAGES || C < 1 || C > D2B_PANOPTIC_MAX_CLASSES) return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  if (!panoptic_images_ok(img, N)) return D2B_EINVAL;
  if (!num_segments || !seg_info || !seg_score || !status || !workspace) return D2B_EINVAL;
  if ((uintptr_t)workspace % kAlign) return D2B_EINVAL;
  PanArgs a;
  if (workspace_bytes < panoptic_layout(img, N, C, &a)) return D2B_EWORKSPACE;
  a.img = *img;
  a.inst_start[0] = 0;
  long long max_pix = 0;
  int rmax = 0;
  for (int n = 0; n < N; ++n) {
    a.inst_start[n + 1] = a.inst_start[n] + img->R[n];
    rmax = std::max(rmax, img->R[n]);
    max_pix = std::max(max_pix, (long long)img->H[n] * img->W[n]);
  }
  for (int n = N; n < D2B_MAX_IMAGES; ++n) a.inst_start[n + 1] = a.inst_start[N];
  a.N = N, a.C = C, a.S = rmax + C;
  a.num_instances = num_instances;
  a.overlap = overlap_threshold, a.stuff_thresh = stuff_area_thresh, a.score_thresh = instances_score_thresh;
  a.num_segments = num_segments, a.seg_info = seg_info, a.seg_score = seg_score, a.status = status;
  a.ws = (unsigned char*)workspace;
  const cudaStream_t st = (cudaStream_t)stream;
  if (a.inst_start[N] > 0) {
    panoptic_pack_kernel<<<a.inst_start[N], kPackThreads, 0, st>>>(a);
    D2B_CHECK_LAUNCH();
  }
  panoptic_walk_kernel<<<N, kWalkThreads, 0, st>>>(a);
  D2B_CHECK_LAUNCH();
  const dim3 grid(d2b_cdiv(max_pix, kPixChunk), N);
  panoptic_hist_kernel<<<grid, kPixThreads, 2 * C * sizeof(unsigned), st>>>(a);
  D2B_CHECK_LAUNCH();
  panoptic_stuff_kernel<<<grid, kPixThreads, C * sizeof(int), st>>>(a);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
