// Batched, fixed-capacity sampling of training labels: the law of subsample_labels (detectron2/modeling/sampling.py:9-54)
// for all images in one launch sequence, without the per-image nonzero() host syncs and torch.randperm calls of
//   RPN._subsample_labels                        (proposal_generator/rpn.py:286-303; RRPN, rrpn.py:184)
//   ROIHeads._sample_proposals                   (roi_heads/roi_heads.py:181-217; rotated_fast_rcnn.py:218-270)
//
// Every candidate i of image n gets a 64-bit key (SplitMix64, see d2b200.h); the sample is the k_pos smallest-key positives
// and the k_neg smallest-key negatives, each in ascending key order: a uniform random subset in uniform random order, the
// law of randperm(...)[:k].  Keys are injective in i for a fixed image, so "the k smallest" is always well defined.  The
// keys are recomputed wherever they are needed, never stored.
//
// Exact per-image k-smallest selection by a radix select on the key's top kDigit bits:
//   zero-fill        histograms and counters (one launch);
//   hist_kernel      grid (chunks, N): per-set histogram of the top digit, shared-memory counts then global atomics;
//   thresh_kernel    grid (2 sets, N): #pos / #neg -> k_pos, k_neg; the set's threshold bin b (keys in bins < b are taken
//                    outright, bin b holds the last ones) and its population;
//   select_kernel    grid (chunks, N): the RPN label map filled with -1; bins < b appended to `sel`, bin b to `cand` when it
//                    fits kCap slots;
//   finish_kernel    grid (2 sets, N): (bin b over kCap only: refine by the next key digits, rescanning the image) the
//                    selected and candidate indices sorted by key in shared memory, the first k emitted (and marked in
//                    the label map), -1 padding.
// The result is exact for every input: a threshold bin of more than kCap keys is refined digit by digit (the last digit
// leaves one key per bin), whatever the key distribution.
#include <climits>

#include "common.cuh"

namespace {

constexpr int kDigit = 10;  // bits per radix digit
constexpr int kBins = 1 << kDigit;
constexpr int kTopShift = 64 - kDigit;
constexpr int kCap = 2048;        // candidate slots per (image, set) for the threshold bin
constexpr int kThreads = 256;     // hist / select CTAs
constexpr int kChunk = 8192;      // elements per hist / select CTA
constexpr int kFinishThreads = 1024;

__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z ^= z >> 30;
  z *= 0xBF58476D1CE4E5B9ULL;
  z ^= z >> 27;
  z *= 0x94D049BB133111EBULL;
  z ^= z >> 31;
  return z;
}

__device__ __forceinline__ unsigned long long image_stream(unsigned long long seed, int n) {
  return mix64(seed + (unsigned long long)(n + 1) * 0xD1B54A32D192ED03ULL);
}

__device__ __forceinline__ unsigned long long key_of(unsigned long long s, int i) {
  return mix64(s + (unsigned long long)(i + 1) * 0x9E3779B97F4A7C15ULL);
}

struct Info {  // per (image, set), written by thresh_kernel
  int k;       // samples to take from the set
  int bin;     // threshold bin of the top digit: bins < bin are taken outright
  int count;   // keys of the set in that bin
  int pad;
};

struct SampleArgs {
  const void* labels;  // [N, P] int8 or int64
  int i64;
  int N, P, num_samples, max_pos;
  long long bg;
  const unsigned long long* seed;
  signed char* out_labels;  // [N, P] or NULL
  long long* sampled;       // [N, num_samples] or NULL
  long long* num_pos;       // [N]
  long long* num_neg;       // [N]
  unsigned* hist;           // [N, 2, kBins], zeroed
  unsigned* counters;       // [N, 2, 2] (selected, candidates), zeroed
  Info* info;               // [N, 2]
  int* sel;                 // [N, 2, num_samples]
  int* cand;                // [N, 2, kCap]
};

// 0 = positive, 1 = negative, -1 = neither (ignored or padding)
__device__ __forceinline__ int set_of(const SampleArgs& a, int n, int i) {
  const size_t o = (size_t)n * a.P + i;
  const long long l = a.i64 ? ((const long long*)a.labels)[o] : (long long)((const signed char*)a.labels)[o];
  return l == a.bg ? 1 : (l != -1 ? 0 : -1);
}

__global__ void __launch_bounds__(kThreads) hist_kernel(const SampleArgs a) {
  __shared__ unsigned h[2 * kBins];
  const int n = blockIdx.y;
  for (int t = threadIdx.x; t < 2 * kBins; t += kThreads) h[t] = 0u;
  __syncthreads();
  const unsigned long long s = image_stream(*a.seed, n);
  const int i0 = blockIdx.x * kChunk, i1 = min(a.P, i0 + kChunk);
  for (int i = i0 + threadIdx.x; i < i1; i += kThreads) {
    const int set = set_of(a, n, i);
    if (set >= 0) atomicAdd(&h[set * kBins + (int)(key_of(s, i) >> kTopShift)], 1u);
  }
  __syncthreads();
  unsigned* g = a.hist + (size_t)n * 2 * kBins;
  for (int t = threadIdx.x; t < 2 * kBins; t += kThreads)
    if (h[t]) atomicAdd(&g[t], h[t]);
}

// The bin whose [before, before + count) contains the need-th smallest key (need >= 1): one thread of the block finds it.
__device__ __forceinline__ void find_bin(unsigned before, unsigned count, unsigned need, int* s_bin, unsigned* s_below,
                                         unsigned* s_count) {
  if (count && before < need && need <= before + count) {
    *s_bin = threadIdx.x;
    *s_below = before;
    *s_count = count;
  }
}

__global__ void __launch_bounds__(kBins) thresh_kernel(const SampleArgs a) {
  __shared__ unsigned s_warp[32];
  __shared__ int s_bin;
  __shared__ unsigned s_below, s_count;
  const int set = blockIdx.x, n = blockIdx.y, t = threadIdx.x;
  const unsigned* g = a.hist + (size_t)n * 2 * kBins;
  const unsigned hp = g[t], hn = g[kBins + t];
  unsigned npos, nneg;
  const unsigned before_p = block_exclusive_scan(hp, s_warp, npos);
  __syncthreads();  // s_warp reuse
  const unsigned before_n = block_exclusive_scan(hn, s_warp, nneg);
  __syncthreads();
  // sampling.py:41-47: k_pos = min(#pos, int(num_samples * positive_fraction)), k_neg = min(#neg, num_samples - k_pos)
  const int k_pos = (int)min((unsigned)a.max_pos, npos);
  const int k_neg = (int)min((unsigned)(a.num_samples - k_pos), nneg);
  const int k = set ? k_neg : k_pos;
  if (t == 0) {
    s_bin = 0;
    s_below = 0u;
    s_count = 0u;
  }
  __syncthreads();
  if (k > 0) find_bin(set ? before_n : before_p, set ? hn : hp, (unsigned)k, &s_bin, &s_below, &s_count);
  __syncthreads();
  if (t == 0) {
    Info in;
    in.k = k;
    in.bin = k > 0 ? s_bin : 0;  // k == 0: no bin is below 0 and no candidate is collected
    in.count = k > 0 ? (int)s_count : 0;
    in.pad = 0;
    a.info[2 * n + set] = in;
    (set ? a.num_neg : a.num_pos)[n] = k;
  }
}

__global__ void __launch_bounds__(kThreads) select_kernel(const SampleArgs a) {
  const int n = blockIdx.y;
  const Info in0 = a.info[2 * n], in1 = a.info[2 * n + 1];
  const unsigned long long s = image_stream(*a.seed, n);
  const int i0 = blockIdx.x * kChunk, i1 = min(a.P, i0 + kChunk);
  unsigned* cnt = a.counters + (size_t)n * 4;
  for (int i = i0 + threadIdx.x; i < i1; i += kThreads) {
    if (a.out_labels) a.out_labels[(size_t)n * a.P + i] = -1;
    const int set = set_of(a, n, i);
    if (set < 0) continue;
    const Info& in = set ? in1 : in0;
    if (in.k == 0) continue;
    const int d = (int)(key_of(s, i) >> kTopShift);
    if (d < in.bin) {
      const unsigned j = atomicAdd(&cnt[2 * set], 1u);  // < k <= num_samples
      a.sel[((size_t)n * 2 + set) * a.num_samples + j] = i;
    } else if (d == in.bin && in.count <= kCap) {
      const unsigned j = atomicAdd(&cnt[2 * set + 1], 1u);  // < count <= kCap
      a.cand[((size_t)n * 2 + set) * kCap + j] = i;
    }
  }
}

__device__ __forceinline__ bool key_less(unsigned long long ka, int ia, unsigned long long kb, int ib) {
  return ka < kb || (ka == kb && ia < ib);
}

__global__ void __launch_bounds__(kFinishThreads) finish_kernel(const SampleArgs a) {
  extern __shared__ unsigned long long s_key[];  // [M] keys, then [M] indices (M = pow2 >= num_samples + kCap)
  __shared__ unsigned s_warp[32];
  __shared__ int s_bin;
  __shared__ unsigned s_below, s_count, s_nsel, s_ncand;
  const int set = blockIdx.x, n = blockIdx.y, t = threadIdx.x;
  const Info in = a.info[2 * n + set];
  const int k = in.k;
  const int k_pos = a.info[2 * n].k;
  const int off = set ? k_pos : 0;
  if (a.sampled && set == 1)  // padding after the negatives: sampled[n, k_pos + k_neg :] = -1
    for (int j = k_pos + k + t; j < a.num_samples; j += kFinishThreads) a.sampled[(size_t)n * a.num_samples + j] = -1;
  if (k == 0) return;
  const unsigned long long s = image_stream(*a.seed, n);
  int* sel = a.sel + ((size_t)n * 2 + set) * a.num_samples;
  int* cand = a.cand + ((size_t)n * 2 + set) * kCap;
  if (t == 0) {
    s_nsel = a.counters[(size_t)n * 4 + 2 * set];
    s_ncand = a.counters[(size_t)n * 4 + 2 * set + 1];
  }
  __syncthreads();
  if (in.count > kCap) {
    // The threshold bin overflowed the candidate slots: refine it by the next digits, one CTA rescanning the image.
    unsigned* h = reinterpret_cast<unsigned*>(s_key);  // kBins counters, before the sort uses the buffer
    unsigned long long prefix = (unsigned long long)in.bin;
    int shift = kTopShift;
    unsigned need = (unsigned)k - s_nsel;
    for (;;) {
      const int nshift = max(shift - kDigit, 0);
      const unsigned long long mask = (1ull << (shift - nshift)) - 1ull;
      h[t] = 0u;
      __syncthreads();
      for (int i = t; i < a.P; i += kFinishThreads) {
        if (set_of(a, n, i) != set) continue;
        const unsigned long long key = key_of(s, i);
        if ((key >> shift) == prefix) atomicAdd(&h[(int)((key >> nshift) & mask)], 1u);
      }
      __syncthreads();
      if (t == 0) s_count = 0u;
      unsigned total;
      const unsigned v = h[t];
      const unsigned before = block_exclusive_scan(v, s_warp, total);
      __syncthreads();
      find_bin(before, v, need, &s_bin, &s_below, &s_count);
      __syncthreads();
      const unsigned long long b = (unsigned long long)s_bin;
      const bool collect = s_count <= (unsigned)kCap;
      for (int i = t; i < a.P; i += kFinishThreads) {
        if (set_of(a, n, i) != set) continue;
        const unsigned long long key = key_of(s, i);
        if ((key >> shift) != prefix) continue;
        const unsigned long long d = (key >> nshift) & mask;
        if (d < b) {
          sel[atomicAdd(&s_nsel, 1u)] = i;
        } else if (d == b && collect) {
          cand[atomicAdd(&s_ncand, 1u)] = i;
        }
      }
      need -= s_below;
      prefix = (prefix << (shift - nshift)) | b;
      shift = nshift;
      __syncthreads();
      if (collect) break;  // shift 0 leaves one key per bin: the loop always ends
    }
  }
  // sort the selected keys and the threshold-bin candidates together; the first k are the sample
  const int nsel = (int)s_nsel, items = nsel + (int)s_ncand;
  int m = 1;
  while (m < items) m <<= 1;
  const int cap = 1 << (32 - __clz(a.num_samples + kCap - 1));
  int* s_idx = reinterpret_cast<int*>(s_key + cap);
  for (int j = t; j < m; j += kFinishThreads) {
    if (j < items) {
      const int i = j < nsel ? sel[j] : cand[j - nsel];
      s_key[j] = key_of(s, i);
      s_idx[j] = i;
    } else {
      s_key[j] = ~0ull;
      s_idx[j] = INT_MAX;  // after every real (key, index)
    }
  }
  __syncthreads();
  for (int size = 2; size <= m; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = t; i < m; i += kFinishThreads) {
        const int l = i ^ stride;
        if (l > i) {
          const bool up = (i & size) == 0;
          if (key_less(s_key[l], s_idx[l], s_key[i], s_idx[i]) == up) {
            const unsigned long long tk = s_key[i];
            s_key[i] = s_key[l];
            s_key[l] = tk;
            const int ti = s_idx[i];
            s_idx[i] = s_idx[l];
            s_idx[l] = ti;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int j = t; j < k; j += kFinishThreads) {
    const int i = s_idx[j];
    if (a.sampled) a.sampled[(size_t)n * a.num_samples + off + j] = i;
    if (a.out_labels) a.out_labels[(size_t)n * a.P + i] = set ? 0 : 1;  // rpn.py:301-303
  }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t finish_smem_bytes(int num_samples) {
  size_t m = 1;
  while (m < (size_t)num_samples + kCap) m <<= 1;
  return m * (sizeof(unsigned long long) + sizeof(int));
}

struct Layout {
  size_t hist, counters, info, sel, cand, total;
};

Layout layout(int N, int num_samples) {
  Layout l;
  l.hist = 0;
  l.counters = l.hist + align256(sizeof(unsigned) * (size_t)N * 2 * kBins);
  l.info = l.counters + align256(sizeof(unsigned) * (size_t)N * 4);
  l.sel = l.info + align256(sizeof(Info) * (size_t)N * 2);
  l.cand = l.sel + align256(sizeof(int) * (size_t)N * 2 * num_samples);
  l.total = l.cand + align256(sizeof(int) * (size_t)N * 2 * kCap);
  return l;
}

}  // namespace

D2B_API size_t d2b_sample_labels_workspace_bytes(int N, int P, int num_samples) {
  if (N <= 0 || P < 0 || num_samples < 0) return 0;
  return layout(N, num_samples).total;
}

D2B_API int d2b_sample_labels(const void* labels, int label_kind, int N, int P, int64_t bg_label, int num_samples,
                              int max_pos, const uint64_t* seed, int8_t* out_labels, int64_t* sampled, int64_t* num_pos,
                              int64_t* num_neg, void* workspace, size_t workspace_bytes, void* stream) {
  if (label_kind != D2B_LABELS_I8 && label_kind != D2B_LABELS_I64) return D2B_EINVAL;
  if (N < 0 || P < 0 || num_samples < 0) return D2B_EINVAL;
  if (max_pos < 0 || max_pos > num_samples) return D2B_EINVAL;
  if (!out_labels && !sampled) return D2B_EINVAL;
  if (out_labels && (const void*)out_labels == labels) return D2B_EINVAL;
  if (N > 65535 || num_samples > D2B_SAMPLE_MAX_SAMPLES || P > INT_MAX - kChunk) return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  if ((P > 0 && !labels) || !seed || !num_pos || !num_neg || !workspace) return D2B_EINVAL;
  const Layout l = layout(N, num_samples);
  if (workspace_bytes < l.total) return D2B_EINVAL;

  SampleArgs a = {};
  a.labels = labels;
  a.i64 = label_kind == D2B_LABELS_I64;
  a.N = N;
  a.P = P;
  a.num_samples = num_samples;
  a.max_pos = max_pos;
  a.bg = bg_label;
  a.seed = (const unsigned long long*)seed;
  a.out_labels = (signed char*)out_labels;
  a.sampled = (long long*)sampled;
  a.num_pos = (long long*)num_pos;
  a.num_neg = (long long*)num_neg;
  char* ws = (char*)workspace;
  a.hist = (unsigned*)(ws + l.hist);
  a.counters = (unsigned*)(ws + l.counters);
  a.info = (Info*)(ws + l.info);
  a.sel = (int*)(ws + l.sel);
  a.cand = (int*)(ws + l.cand);

  const cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = finish_smem_bytes(num_samples);
  D2B_ALLOW_BIG_SMEM(finish_kernel);
  void* ptrs[1] = {ws};  // hist and counters are adjacent
  size_t bytes[1] = {l.info};
  const int rc = d2b_zero_buffers(ptrs, bytes, 1, st);
  if (rc) return rc;
  const dim3 grid((unsigned)max(1, d2b_cdiv(P, kChunk)), (unsigned)N);
  hist_kernel<<<grid, kThreads, 0, st>>>(a);
  D2B_CHECK_LAUNCH();
  thresh_kernel<<<dim3(2, N), kBins, 0, st>>>(a);
  D2B_CHECK_LAUNCH();
  select_kernel<<<grid, kThreads, 0, st>>>(a);
  D2B_CHECK_LAUNCH();
  finish_kernel<<<dim3(2, N), kFinishThreads, smem, st>>>(a);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
