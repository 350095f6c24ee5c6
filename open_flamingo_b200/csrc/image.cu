// CLIP eval transform (open_clip image_transform(is_train=False): Resize(S, BICUBIC) + CenterCrop(S) + ToTensor +
// Normalize) on decoded uint8 RGB or L pixels, bit for bit what the PIL / torchvision pipeline computes.
//
// Resize is Pillow's two-pass fixed-point bicubic.  Per axis the host computes, in double without FMA contraction
// (the library is built with -ffp-contract=off), each output index's source span and int32 taps at 22 fractional bits;
// each pass sums 2^21 + pixel * tap in int32 and clamps `acc >> 22` to [0, 255].  Only the crop window is resampled:
// the first pass writes the source rows (or columns) the second pass's taps read, for the cropped columns (or rows)
// only, into a uint8 intermediate; the second pass writes the S x S window fused with channel replication of L
// images, /255 and (x - mean) / std in IEEE fp32.
//
// Pillow resizes horizontally first, except that Image.resize runs the vertical pass first when the image is more
// than 100 times taller than wide and its height shrinks; the plan records the order per image.  Pillow skips an axis
// whose size does not change; here that axis runs with its identity taps (0, 2^22, 0, ...), which copy each pixel
// exactly (2^21 + p 2^22 >> 22 = p), so every image takes the same two kernels.
//
// ofk_image_plan lays out, in one caller-owned host buffer, a header, one descriptor per image and the tap tables;
// ofk_clip_preprocess checks it, copies it into the device workspace and makes two launches for the whole batch.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <climits>

#include "ofk_internal.h"

namespace ofk {

constexpr int IMG_THREADS = 256;
constexpr int IMG_PREC = 22;
constexpr uint32_t PLAN_MAGIC = 0x4b464f49u;  // "IOFK"
constexpr int IMG_MAX_S = 4096;
constexpr int IMG_MAX_N = 65535;  // second-pass grid.y

struct PlanHeader {
  uint32_t magic;
  int n, S, blocks1;   // images, output side, blocks of the first pass
  long long bytes;     // plan size
  long long tmp;       // byte offset of the first intermediate in the workspace (= plan size rounded up to 16)
  long long ws_bytes;  // workspace size: plan + intermediates
  float mean[3], std_[3];
};

struct ImageDesc {
  const uint8_t* src;          // device address of pixel (0, 0)
  long long ld;                // source row stride, bytes
  int h, w, c, vfirst;         // vfirst: the vertical pass runs first
  int th, tw;                  // intermediate [th, tw, c] uint8
  int origin;                  // first source row (horizontal first) or column (vertical first) the first pass reads
  int blk0;                    // first block of this image in the first pass
  long long tmp;               // byte offset of the intermediate in the workspace
  long long ts1, os1;          // first pass: source bytes between taps and between positions on the other axis
  long long ts2, os2;          // second pass: intermediate bytes between taps and between positions on the other axis
  int tab1, k1, tab2, k2;      // int32 offsets of the tap tables in the plan and their tap counts; entry q of a table
                               // is (pos0, n, tap[0..k-1]) at tab + q (k + 2)
  int oh, ow, top, left;       // resized size and crop offsets
  int pad[2];
};

static_assert(sizeof(PlanHeader) % 16 == 0 && sizeof(ImageDesc) % 16 == 0, "plan records keep 16-byte alignment");

__device__ __forceinline__ int clip8(int acc) {
  return acc >= (1 << (IMG_PREC + 8)) ? 255 : acc <= 0 ? 0 : acc >> IMG_PREC;
}

// 2^21 + sum_t p[pos0 + t] k[t] per channel, p at base + pos * ts, c = 1 or 3 channels at consecutive bytes.
__device__ __forceinline__ void resample(const uint8_t* __restrict__ base, long long ts, const int* __restrict__ e,
                                         int c, int& a0, int& a1, int& a2) {
  const int pos0 = e[0], n = e[1];
  a0 = a1 = a2 = 1 << (IMG_PREC - 1);
  const uint8_t* p = base + pos0 * ts;
  if (c == 3) {
    for (int t = 0; t < n; ++t, p += ts) {
      const int k = e[2 + t];
      a0 += __ldg(p) * k;
      a1 += __ldg(p + 1) * k;
      a2 += __ldg(p + 2) * k;
    }
  } else {
    for (int t = 0; t < n; ++t, p += ts) a0 += __ldg(p) * e[2 + t];
  }
}

// First pass: one thread per intermediate pixel (i, j) of [th, tw], blocks flattened over the batch.
__global__ void __launch_bounds__(IMG_THREADS) image_resample_first_kernel(uint8_t* ws) {
  const PlanHeader* hd = reinterpret_cast<const PlanHeader*>(ws);
  const ImageDesc* ds = reinterpret_cast<const ImageDesc*>(ws + sizeof(PlanHeader));
  const int* tab = reinterpret_cast<const int*>(ws);
  int lo = 0, hi = hd->n - 1;  // last image whose blk0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (ds[mid].blk0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const ImageDesc& d = ds[lo];
  const long long idx = (long long)(blockIdx.x - d.blk0) * IMG_THREADS + threadIdx.x;
  if (idx >= (long long)d.th * d.tw) return;
  const int i = (int)(idx / d.tw), j = (int)(idx % d.tw);
  const int q = d.vfirst ? i : j, other = d.origin + (d.vfirst ? j : i);
  int a0, a1, a2;
  resample(d.src + other * d.os1, d.ts1, tab + d.tab1 + (long long)q * (d.k1 + 2), d.c, a0, a1, a2);
  uint8_t* o = ws + d.tmp + idx * d.c;
  o[0] = (uint8_t)clip8(a0);
  if (d.c == 3) {
    o[1] = (uint8_t)clip8(a1);
    o[2] = (uint8_t)clip8(a2);
  }
}

__device__ __forceinline__ float normalize(int v, float m, float s) {
  return __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), m), s);
}

// Second pass + ToTensor + Normalize: one thread per output pixel (y, x); grid (ceil(S^2 / 256), n).
__global__ void __launch_bounds__(IMG_THREADS) image_resample_second_kernel(const uint8_t* __restrict__ ws,
                                                                           float* __restrict__ out,
                                                                           long long out_stride) {
  const PlanHeader* hd = reinterpret_cast<const PlanHeader*>(ws);
  const ImageDesc& d = reinterpret_cast<const ImageDesc*>(ws + sizeof(PlanHeader))[blockIdx.y];
  const int S = hd->S;
  const int idx = blockIdx.x * IMG_THREADS + threadIdx.x;
  if (idx >= S * S) return;
  const int y = idx / S, x = idx % S;
  const int q = d.vfirst ? x : y, other = d.vfirst ? y : x;
  int a0, a1, a2;
  resample(ws + d.tmp + other * d.os2, d.ts2, reinterpret_cast<const int*>(ws) + d.tab2 + (long long)q * (d.k2 + 2),
           d.c, a0, a1, a2);
  const int r = clip8(a0), g = d.c == 3 ? clip8(a1) : r, b = d.c == 3 ? clip8(a2) : r;
  float* o = out + blockIdx.y * out_stride + idx;
  const long long plane = (long long)S * S;
  o[0] = normalize(r, hd->mean[0], hd->std_[0]);
  o[plane] = normalize(g, hd->mean[1], hd->std_[1]);
  o[2 * plane] = normalize(b, hd->mean[2], hd->std_[2]);
}

// ------------------------------------------------------------------------------------------------ host plan

static long long align16(long long x) { return (x + 15) & ~15LL; }

static double bicubic(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

static int axis_ksize(int in, int out) {
  const double scale = (double)in / out;
  return 2 * (int)ceil(2.0 * (scale < 1.0 ? 1.0 : scale)) + 1;
}

// Entries (pos0 - shift, n, taps[ksize]) for output indices first .. first + count - 1 of an in -> out axis.
static void axis_taps(int in, int out, int first, int count, int shift, int* dst) {
  const double scale = (double)in / out;
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * fs;
  const int ks = 2 * (int)ceil(support) + 1;
  for (int e = 0; e < count; ++e) {
    const int i = first + e;
    const double center = (i + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in) xmax = in;
    const int n = xmax - xmin;
    double ww = 0.0;  // summed left to right; each weight is recomputed below with the same bits
    for (int t = 0; t < n; ++t) ww += bicubic((t + xmin - center + 0.5) / fs);
    int* row = dst + (long long)e * (ks + 2);
    row[0] = xmin - shift;
    row[1] = n;
    for (int t = 0; t < ks; ++t) {
      double v = t < n ? bicubic((t + xmin - center + 0.5) / fs) : 0.0;
      if (ww != 0.0) v /= ww;
      row[2 + t] = v < 0 ? (int)(v * (1 << IMG_PREC) - 0.5) : (int)(v * (1 << IMG_PREC) + 0.5);
    }
  }
}

// Source span [first, last) that output indices first_out .. first_out + count - 1 read (spans grow monotonically).
static void axis_span(int in, int out, int first_out, int count, int* first, int* last) {
  const double scale = (double)in / out;
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * fs;
  const double c0 = (first_out + 0.5) * scale, c1 = (first_out + count - 1 + 0.5) * scale;
  int lo = (int)(c0 - support + 0.5);
  *first = lo < 0 ? 0 : lo;
  int hi = (int)(c1 + support + 0.5);
  *last = hi > in ? in : hi;
}

struct Geometry {
  int oh, ow, top, left, vfirst, th, tw, origin, k1, k2;
};

// torchvision Resize(S) + CenterCrop(S) on an h x w image, Pillow's pass order, and the intermediate's extent.
static Geometry geometry(int h, int w, int S) {
  Geometry g;
  if (w <= h) {
    g.ow = S;
    g.oh = (int)((double)((long long)S * h) / w);
  } else {
    g.oh = S;
    g.ow = (int)((double)((long long)S * w) / h);
  }
  g.top = (int)nearbyint((g.oh - S) / 2.0);  // half to even, as Python's round (default rounding mode)
  g.left = (int)nearbyint((g.ow - S) / 2.0);
  g.vfirst = h > 100LL * w && g.oh < h;
  const int kx = axis_ksize(w, g.ow), ky = axis_ksize(h, g.oh);
  int first, last;
  if (g.vfirst) {
    axis_span(w, g.ow, g.left, S, &first, &last);
    g.th = S;
    g.tw = last - first;
    g.k1 = ky;
    g.k2 = kx;
  } else {
    axis_span(h, g.oh, g.top, S, &first, &last);
    g.th = last - first;
    g.tw = S;
    g.k1 = kx;
    g.k2 = ky;
  }
  g.origin = first;
  return g;
}

static int check_image(long long h, long long w, long long c, long long ld, int S) {
  if (h < 1 || w < 1) return ofk_set_error(OFK_ERR_ARG, "image plan: image sides must be >= 1");
  if ((long long)S * (h > w ? h : w) > INT_MAX)
    return ofk_set_error(OFK_ERR_ARG, "image plan: S * longer side must fit in int32");
  if (c != 1 && c != 3) return ofk_set_error(OFK_ERR_ARG, "image plan: channels must be 1 (L) or 3 (RGB)");
  if (ld < w * c) return ofk_set_error(OFK_ERR_ARG, "image plan: row stride must be >= w * channels bytes");
  return 0;
}

static int check_common(int n, const long long* shape, int S) {
  if (!shape) return ofk_set_error(OFK_ERR_ARG, "image plan: null pointer");
  if (n < 1 || n > IMG_MAX_N) return ofk_set_error(OFK_ERR_ARG, "image plan: n must be in [1, 65535]");
  if (S < 1 || S > IMG_MAX_S) return ofk_set_error(OFK_ERR_ARG, "image plan: S must be in [1, 4096]");
  for (int i = 0; i < n; ++i) {
    const long long* s = shape + 4LL * i;
    if (int rc = check_image(s[0], s[1], s[2], s[3], S)) return rc;
  }
  return 0;
}

// Plan size, workspace size and first-pass blocks; the caller has checked the shapes.
static int sizes(int n, const long long* shape, int S, long long* plan, long long* ws, long long* blocks) {
  long long p = sizeof(PlanHeader) + (long long)n * sizeof(ImageDesc), t = 0, b = 0;
  for (int i = 0; i < n; ++i) {
    const Geometry g = geometry((int)shape[4 * i], (int)shape[4 * i + 1], S);
    p += 4LL * S * (g.k1 + 2 + g.k2 + 2);
    t += align16((long long)g.th * g.tw * shape[4 * i + 2]);
    b += ((long long)g.th * g.tw + IMG_THREADS - 1) / IMG_THREADS;
  }
  if (b > INT_MAX || p > INT_MAX) return ofk_set_error(OFK_ERR_ARG, "image plan: batch too large for one plan");
  *plan = p;
  *ws = align16(p) + t;
  *blocks = b;
  return 0;
}

static bool bad_float(float v) { return !isfinite(v); }

}  // namespace ofk

extern "C" int ofk_image_plan_size(int n, const long long* shape, int S, long long* plan_bytes,
                                   long long* workspace_bytes) {
  using namespace ofk;
  if (!plan_bytes || !workspace_bytes) return ofk_set_error(OFK_ERR_ARG, "image plan size: null pointer");
  if (int rc = check_common(n, shape, S)) return rc;
  long long blocks;
  return sizes(n, shape, S, plan_bytes, workspace_bytes, &blocks);
}

extern "C" int ofk_image_plan(int n, const void* const* src, const long long* shape, int S, const float* mean,
                              const float* std_, void* plan, long long plan_bytes) {
  using namespace ofk;
  if (!src || !mean || !std_ || !plan) return ofk_set_error(OFK_ERR_ARG, "image plan: null pointer");
  if (int rc = check_common(n, shape, S)) return rc;
  for (int i = 0; i < n; ++i)
    if (!src[i]) return ofk_set_error(OFK_ERR_ARG, "image plan: null image pointer");
  for (int ch = 0; ch < 3; ++ch)
    if (bad_float(mean[ch]) || bad_float(std_[ch]) || std_[ch] == 0.f)
      return ofk_set_error(OFK_ERR_ARG, "image plan: mean and std must be finite and std nonzero");
  if (reinterpret_cast<uintptr_t>(plan) & 15) return ofk_set_error(OFK_ERR_ALIGN, "image plan: plan must be 16-byte aligned");
  long long need, ws, blocks;
  if (int rc = sizes(n, shape, S, &need, &ws, &blocks)) return rc;
  if (plan_bytes != need) return ofk_set_error(OFK_ERR_ARG, "image plan: plan_bytes must equal ofk_image_plan_size's");

  uint8_t* base = static_cast<uint8_t*>(plan);
  PlanHeader* hd = reinterpret_cast<PlanHeader*>(base);
  memset(hd, 0, sizeof(PlanHeader));
  hd->magic = PLAN_MAGIC;
  hd->n = n;
  hd->S = S;
  hd->blocks1 = (int)blocks;
  hd->bytes = need;
  hd->tmp = align16(need);
  hd->ws_bytes = ws;
  for (int ch = 0; ch < 3; ++ch) {
    hd->mean[ch] = mean[ch];
    hd->std_[ch] = std_[ch];
  }
  ImageDesc* ds = reinterpret_cast<ImageDesc*>(base + sizeof(PlanHeader));
  int* tab = reinterpret_cast<int*>(base);
  long long off = (sizeof(PlanHeader) + (long long)n * sizeof(ImageDesc)) / 4, tmp = hd->tmp;
  int blk = 0;
  for (int i = 0; i < n; ++i) {
    const long long* s = shape + 4LL * i;
    const int h = (int)s[0], w = (int)s[1], c = (int)s[2];
    const Geometry g = geometry(h, w, S);
    ImageDesc& d = ds[i];
    memset(&d, 0, sizeof(ImageDesc));
    d.src = static_cast<const uint8_t*>(src[i]);
    d.ld = s[3];
    d.h = h; d.w = w; d.c = c; d.vfirst = g.vfirst;
    d.th = g.th; d.tw = g.tw; d.origin = g.origin;
    d.oh = g.oh; d.ow = g.ow; d.top = g.top; d.left = g.left;
    d.blk0 = blk;
    d.tmp = tmp;
    d.k1 = g.k1;
    d.k2 = g.k2;
    d.tab1 = (int)off;
    d.tab2 = (int)(off + (long long)S * (g.k1 + 2));
    if (g.vfirst) {      // rows first: taps between source rows, positions on the other axis are columns
      d.ts1 = d.ld; d.os1 = c;
      d.ts2 = c; d.os2 = (long long)g.tw * c;
      axis_taps(h, g.oh, g.top, S, 0, tab + d.tab1);
      axis_taps(w, g.ow, g.left, S, g.origin, tab + d.tab2);
    } else {
      d.ts1 = c; d.os1 = d.ld;
      d.ts2 = (long long)g.tw * c; d.os2 = c;
      axis_taps(w, g.ow, g.left, S, 0, tab + d.tab1);
      axis_taps(h, g.oh, g.top, S, g.origin, tab + d.tab2);
    }
    off = d.tab2 + (long long)S * (g.k2 + 2);
    tmp += align16((long long)g.th * g.tw * c);
    blk += (int)(((long long)g.th * g.tw + IMG_THREADS - 1) / IMG_THREADS);
  }
  return 0;
}

namespace ofk {

// Every table entry reads inside its axis: 0 <= pos0, 0 <= n <= k, pos0 + n <= extent.
static bool bad_table(const int* tab, long long words, long long at, int k, int S, long long extent) {
  if (k < 1 || at < 0 || at + (long long)S * (k + 2) > words) return true;
  for (int q = 0; q < S; ++q) {
    const int* e = tab + at + (long long)q * (k + 2);
    if (e[0] < 0 || e[1] < 0 || e[1] > k || (long long)e[0] + e[1] > extent) return true;
  }
  return false;
}

// A plan whose every read and write stays inside the images, the workspace and `out`.
static int check_plan(const uint8_t* plan, long long plan_bytes, long long ws_bytes) {
  if (plan_bytes < (long long)sizeof(PlanHeader)) return ofk_set_error(OFK_ERR_ARG, "clip preprocess: plan too small");
  const PlanHeader* hd = reinterpret_cast<const PlanHeader*>(plan);
  if (hd->magic != PLAN_MAGIC || hd->bytes != plan_bytes || hd->n < 1 || hd->n > IMG_MAX_N || hd->S < 1 ||
      hd->S > IMG_MAX_S || plan_bytes < (long long)sizeof(PlanHeader) + (long long)hd->n * sizeof(ImageDesc) ||
      hd->tmp != align16(plan_bytes) || hd->blocks1 < 1)
    return ofk_set_error(OFK_ERR_ARG, "clip preprocess: not a plan made by ofk_image_plan");
  if (ws_bytes < hd->ws_bytes) return ofk_set_error(OFK_ERR_ARG, "clip preprocess: workspace smaller than the plan's");
  const ImageDesc* ds = reinterpret_cast<const ImageDesc*>(plan + sizeof(PlanHeader));
  const int* tab = reinterpret_cast<const int*>(plan);
  const long long words = plan_bytes / 4;
  const int S = hd->S;
  long long blk = 0;
  for (int i = 0; i < hd->n; ++i) {
    const ImageDesc& d = ds[i];
    const bool v = d.vfirst != 0;
    if (!d.src || check_image(d.h, d.w, d.c, d.ld, S) || d.th < 1 || d.tw < 1 || d.blk0 != blk ||
        d.ts1 != (v ? d.ld : d.c) || d.os1 != (v ? d.c : d.ld) || d.ts2 != (v ? d.c : (long long)d.tw * d.c) ||
        d.os2 != (v ? (long long)d.tw * d.c : d.c) || (v ? d.th : d.tw) != S || d.origin < 0 ||
        d.origin + (long long)(v ? d.tw : d.th) > (v ? d.w : d.h) || d.tmp < hd->tmp ||
        d.tmp + (long long)d.th * d.tw * d.c > hd->ws_bytes ||
        bad_table(tab, words, d.tab1, d.k1, S, v ? d.h : d.w) ||
        bad_table(tab, words, d.tab2, d.k2, S, v ? d.tw : d.th))
      return ofk_set_error(OFK_ERR_ARG, "clip preprocess: plan descriptor out of range");
    blk += ((long long)d.th * d.tw + IMG_THREADS - 1) / IMG_THREADS;
  }
  if (blk != hd->blocks1) return ofk_set_error(OFK_ERR_ARG, "clip preprocess: plan block count mismatch");
  return 0;
}

}  // namespace ofk

extern "C" int ofk_clip_preprocess(const void* plan, long long plan_bytes, void* workspace, long long workspace_bytes,
                                   float* out, long long out_image_stride, void* stream_) {
  using namespace ofk;
  if (!plan || !workspace || !out) return ofk_set_error(OFK_ERR_ARG, "clip preprocess: null pointer");
  if (reinterpret_cast<uintptr_t>(plan) & 15) return ofk_set_error(OFK_ERR_ALIGN, "clip preprocess: plan must be 16-byte aligned");
  if (int rc = check_plan(static_cast<const uint8_t*>(plan), plan_bytes, workspace_bytes)) return rc;
  const PlanHeader* hd = static_cast<const PlanHeader*>(plan);
  if (out_image_stride < 3LL * hd->S * hd->S)
    return ofk_set_error(OFK_ERR_ARG, "clip preprocess: out image stride must be >= 3 * S * S");
  if (reinterpret_cast<uintptr_t>(workspace) & 15)
    return ofk_set_error(OFK_ERR_ALIGN, "clip preprocess: workspace must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(out) & 3) return ofk_set_error(OFK_ERR_ALIGN, "clip preprocess: out must be 4-byte aligned");
  cudaStream_t s = (cudaStream_t)stream_;
  cudaError_t e = cudaMemcpyAsync(workspace, plan, plan_bytes, cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e));
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  image_resample_first_kernel<<<hd->blocks1, IMG_THREADS, 0, s>>>(ws);
  OFK_CHECK_LAUNCH();
  const dim3 grid2((unsigned)((hd->S * hd->S + IMG_THREADS - 1) / IMG_THREADS), (unsigned)hd->n);
  image_resample_second_kernel<<<grid2, IMG_THREADS, 0, s>>>(ws, out, out_image_stride);
  OFK_CHECK_LAUNCH();
  return 0;
}
