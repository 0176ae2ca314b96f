// Byte/integer image kernels of the parse path (HBM-bound, bit-exact targets):
//   * letterbox: Pillow-exact LANCZOS resize (two-pass integer FIR, u8 intermediate) + paste on a 114 canvas,
//     replacing PIL Image.resize + Image.paste at ref:util/yolov9.py:82-84.
//   * im2col_u8: tiny-Cin conv stems (YOLOv9-E 3x3/s2, DaViT 7x7/s4) as a dense [pixels][Kpad] fp16 matrix with
//     the per-channel u8 -> float map (the /255, ref:util/yolov9.py:85; CLIP rescale+normalize, ref:util/utils.py:121)
//     folded into a 256-entry table.
//   * crop_resize: batched ROI crop + OpenCV-exact INTER_LINEAR u8 resize to 64x64, replacing the Python loop at
//     ref:util/utils.py:97-103.
#include "b2p_internal.h"
#include <cuda_fp16.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <list>
#include <vector>
#include <map>
#include <mutex>

namespace b2p {

// ----------------------------------------------------------------------------------------- LANCZOS
// Pillow src/libImaging/Resample.c: precompute_coeffs() + normalize_coeffs_8bpc(), PRECISION_BITS = 22.
static double sinc_filter(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return sin(x) / x;
}
static double lanczos_filter(double x) {
  if (-3.0 <= x && x < 3.0) return sinc_filter(x) * sinc_filter(x / 3);
  return 0.0;
}
// Pillow bicubic_filter (a = -0.5, support 2): the CLIP image processor's resample=3 of the reference's CPU caption
// branch (ref:util/utils.py:123 -> HF processor default do_resize=True, 768x768)
static double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

struct Coeffs {
  int ksize = 0, out = 0;
  int* d_bounds = nullptr;   // [out][2] xmin, count
  int* d_kk = nullptr;       // [out][ksize] 22-bit fixed point
};

void host_lanczos_coeffs(int inSize, int outSize, int* ksize_out, std::vector<int>& bounds, std::vector<int>& kk, int filter = 0) {
  const double fsupport = filter == 1 ? 2.0 : 3.0;
  const float in0 = 0.f, in1 = float(inSize);
  double filterscale, scale;
  filterscale = scale = double(in1 - in0) / outSize;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = fsupport * filterscale;
  const int ksize = int(ceil(support)) * 2 + 1;
  bounds.assign(size_t(outSize) * 2, 0);
  kk.assign(size_t(outSize) * ksize, 0);
  std::vector<double> k(ksize);
  for (int xx = 0; xx < outSize; ++xx) {
    const double center = in0 + (xx + 0.5) * scale;
    double ww = 0.0;
    const double ss = 1.0 / filterscale;
    int xmin = int(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = int(center + support + 0.5);
    if (xmax > inSize) xmax = inSize;
    xmax -= xmin;
    int x;
    for (x = 0; x < xmax; ++x) {
      const double arg = (x + xmin - center + 0.5) * ss;
      const double w = filter == 1 ? bicubic_filter(arg) : lanczos_filter(arg);
      k[x] = w;
      ww += w;
    }
    for (x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    for (; x < ksize; ++x) k[x] = 0;
    bounds[xx * 2] = xmin;
    bounds[xx * 2 + 1] = xmax;
    for (x = 0; x < ksize; ++x) {
      const double v = k[x];
      kk[size_t(xx) * ksize + x] = (v < 0) ? int(-0.5 + v * (1 << 22)) : int(0.5 + v * (1 << 22));
    }
  }
  *ksize_out = ksize;
}

static std::mutex g_coeff_mu;
static std::map<std::pair<std::pair<int, int>, int>, Coeffs> g_coeffs;   // (in, out, filter); one process per GPU

static int get_coeffs(int inSize, int outSize, Coeffs* out, int filter = 0) {
  std::lock_guard<std::mutex> lk(g_coeff_mu);
  auto key = std::make_pair(std::make_pair(inSize, outSize), filter);
  auto it = g_coeffs.find(key);
  if (it != g_coeffs.end()) { *out = it->second; return 0; }
  std::vector<int> bounds, kk;
  Coeffs c;
  host_lanczos_coeffs(inSize, outSize, &c.ksize, bounds, kk, filter);
  c.out = outSize;
  if (cudaMalloc(&c.d_bounds, bounds.size() * 4) != cudaSuccess || cudaMalloc(&c.d_kk, kk.size() * 4) != cudaSuccess)
    return set_error("letterbox: cudaMalloc for coefficient tables failed");
  cudaMemcpy(c.d_bounds, bounds.data(), bounds.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(c.d_kk, kk.data(), kk.size() * 4, cudaMemcpyHostToDevice);
  g_coeffs[key] = c;
  *out = c;
  return 0;
}

__device__ __forceinline__ unsigned char clip8(int v) {
  v >>= 22;
  return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// One output pixel of a Pillow 8-bit pass: cnt taps of 22-bit weights k over the RGB pixels s, s + step, ...; the
// accumulators start at the rounding half (1 << 21) and the result is clipped to u8.  Every LANCZOS / BICUBIC pass below
// (one-size and batched, horizontal and vertical) goes through this, so their arithmetic cannot drift apart.
template <typename Step>
__device__ __forceinline__ void fir_px(const unsigned char* __restrict__ s, Step step, const int* __restrict__ k, int cnt,
                                       unsigned char* __restrict__ d) {
  int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
  for (int t = 0; t < cnt; ++t) {
    const int w = k[t];
    const unsigned char* p = s + t * step;
    a0 += p[0] * w; a1 += p[1] * w; a2 += p[2] * w;
  }
  d[0] = clip8(a0); d[1] = clip8(a1); d[2] = clip8(a2);
}

// horizontal pass: src [B][H][W][3] -> tmp [B][H][Wo][3]
__global__ void lanczos_h_kernel(const unsigned char* __restrict__ src, int B, int H, int W, int Wo,
                                 const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                 unsigned char* __restrict__ tmp) {
  const long long n = (long long)B * H * Wo;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int xo = int(i % Wo);
    const long long row = i / Wo;
    const int xmin = bounds[2 * xo], cnt = bounds[2 * xo + 1];
    fir_px(src + (row * W + xmin) * 3, 3, kk + (long long)xo * ksize, cnt, tmp + i * 3);
  }
}

// vertical pass + paste: tmp [B][H][Wo][3] -> canvas [B][Th][Tw][3] at (pad_l, pad_t), 114 elsewhere
__global__ void lanczos_v_paste_kernel(const unsigned char* __restrict__ tmp, int B, int H, int Wo, int Ho,
                                       const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                       int Tw, int Th, int pad_l, int pad_t, unsigned char* __restrict__ canvas) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const long long n = (long long)B * Th * Tw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = int(i % Tw);
    const int y = int((i / Tw) % Th);
    const int b = int(i / ((long long)Tw * Th));
    unsigned char* d = canvas + i * 3;
    const int xo = x - pad_l, yo = y - pad_t;
    if (xo < 0 || xo >= Wo || yo < 0 || yo >= Ho) { d[0] = d[1] = d[2] = 114; continue; }
    if (!bounds) {   // no vertical resample needed (Ho == H)
      const unsigned char* s = tmp + (((long long)b * H + yo) * Wo + xo) * 3;
      d[0] = s[0]; d[1] = s[1]; d[2] = s[2];
      continue;
    }
    const int ymin = bounds[2 * yo], cnt = bounds[2 * yo + 1];
    fir_px(tmp + (((long long)b * H + ymin) * Wo + xo) * 3, (long long)Wo * 3, kk + (long long)yo * ksize, cnt, d);
  }
}

// ----------------------------------------------------------------------------------------- ragged letterbox
// A batch of screenshots of different sizes onto one canvas size.  desc [B][kLbDesc] (int64, include/b200parse.h):
// byte offsets of image b in the flat src / tmp buffers, its geometry, and the element offsets of its horizontal /
// vertical tables in the packed int32 table buffer ([out][2] bounds, then [out][ksize] weights), -1 for a skipped pass.
enum { kLbSrc, kLbTmp, kLbH, kLbW, kLbWr, kLbHr, kLbPadL, kLbPadT, kLbHTab, kLbHK, kLbVTab, kLbVK, kLbDesc };

// horizontal pass of every image that needs one: grid (chunks, image); image b: src [H][W][3] -> tmp [H][Wr][3]
__global__ void lanczos_h_batch_kernel(const unsigned char* __restrict__ src, const long long* __restrict__ desc,
                                       const int* __restrict__ tables, unsigned char* __restrict__ tmp) {
  const long long* d = desc + (long long)blockIdx.y * kLbDesc;
  const long long htab = d[kLbHTab];
  if (htab < 0) return;
  const int W = int(d[kLbW]), Wo = int(d[kLbWr]), ksize = int(d[kLbHK]);
  const long long n = d[kLbH] * Wo;
  const unsigned char* s = src + d[kLbSrc];
  unsigned char* t = tmp + d[kLbTmp];
  const int* bounds = tables + htab;
  const int* kk = bounds + 2LL * Wo;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int xo = int(i % Wo);
    const long long row = i / Wo;
    const int xmin = bounds[2 * xo], cnt = bounds[2 * xo + 1];
    fir_px(s + (row * W + xmin) * 3, 3, kk + (long long)xo * ksize, cnt, t + i * 3);
  }
}

// vertical pass + paste: grid (chunks, image); image b's rows of width Wr come from tmp when it had a horizontal pass,
// else straight from src (Wr == W) -> canvas [b][Th][Tw][3] at (pad_l, pad_t), 114 elsewhere
__global__ void lanczos_v_paste_batch_kernel(const unsigned char* __restrict__ src, const long long* __restrict__ desc,
                                             const int* __restrict__ tables, const unsigned char* __restrict__ tmp, int Tw,
                                             int Th, unsigned char* __restrict__ canvas) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const long long* d = desc + (long long)blockIdx.y * kLbDesc;
  const int Wo = int(d[kLbWr]), Ho = int(d[kLbHr]), pad_l = int(d[kLbPadL]), pad_t = int(d[kLbPadT]);
  const long long vtab = d[kLbVTab];
  const int ksize = int(d[kLbVK]);
  const unsigned char* rows = d[kLbHTab] >= 0 ? tmp + d[kLbTmp] : src + d[kLbSrc];
  const int* bounds = vtab >= 0 ? tables + vtab : nullptr;
  const int* kk = vtab >= 0 ? bounds + 2LL * Ho : nullptr;
  const long long n = (long long)Th * Tw;
  unsigned char* out = canvas + (long long)blockIdx.y * n * 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int x = int(i % Tw);
    const int y = int(i / Tw);
    unsigned char* o = out + i * 3;
    const int xo = x - pad_l, yo = y - pad_t;
    if (xo < 0 || xo >= Wo || yo < 0 || yo >= Ho) { o[0] = o[1] = o[2] = 114; continue; }
    if (!bounds) {   // no vertical resample needed (Ho == H)
      const unsigned char* s = rows + ((long long)yo * Wo + xo) * 3;
      o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
      continue;
    }
    const int ymin = bounds[2 * yo], cnt = bounds[2 * yo + 1];
    fir_px(rows + ((long long)ymin * Wo + xo) * 3, (long long)Wo * 3, kk + (long long)yo * ksize, cnt, o);
  }
}

// Host-side cache of packed tables ([out][2] bounds | [out][ksize] weights) per (in, out) LANCZOS pair, least recently
// used first out, so a server that sees recurring screenshot sizes computes each table once.
struct PackedTable { int ksize; std::vector<int> data; };
static std::mutex g_lb_mu;
static std::list<std::pair<std::pair<int, int>, PackedTable>> g_lb_lru;   // most recently used first
static constexpr size_t kLbCacheEntries = 256;

static PackedTable lb_table(int in, int out) {
  std::lock_guard<std::mutex> lk(g_lb_mu);
  const auto key = std::make_pair(in, out);
  for (auto it = g_lb_lru.begin(); it != g_lb_lru.end(); ++it)
    if (it->first == key) {
      g_lb_lru.splice(g_lb_lru.begin(), g_lb_lru, it);
      return it->second;
    }
  std::vector<int> bounds, kk;
  PackedTable t;
  host_lanczos_coeffs(in, out, &t.ksize, bounds, kk);
  t.data = std::move(bounds);
  t.data.insert(t.data.end(), kk.begin(), kk.end());
  g_lb_lru.emplace_front(key, t);
  if (g_lb_lru.size() > kLbCacheEntries) g_lb_lru.pop_back();
  return t;
}

static int lb_check_geometry(long long H, long long W, long long Wr, long long Hr, long long pad_l, long long pad_t, int Tw,
                             int Th, const char* who) {
  char msg[160];
  if (W < 1 || H < 1 || Wr < 1 || Hr < 1) {
    snprintf(msg, sizeof msg, "%s: source and resized sizes must be >= 1", who);
    return set_error(msg);
  }
  if (pad_l < 0 || pad_t < 0 || pad_l + Wr > Tw || pad_t + Hr > Th) {
    snprintf(msg, sizeof msg, "%s: the resized image must lie inside the canvas", who);
    return set_error(msg);
  }
  return 0;
}

// ----------------------------------------------------------------------------------------- im2col
// One thread per output pixel writes the whole row.  (One thread per 8-element chunk -- coalesced 16-byte stores across the
// warp -- is slower on the detector stem, 8x640x640, Kpad 32: the per-element index arithmetic is the
// bound, not the store pattern.)
__global__ void im2col_u8_kernel(const unsigned char* __restrict__ img, int B, int H, int W, int k, int s, int p,
                                 int Ho, int Wo, int Kpad, const float* __restrict__ lut /*[3][256]*/,
                                 __half* __restrict__ out, int split) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const long long n = (long long)B * Ho * Wo;
  const int K = k * k * 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int ox = int(i % Wo);
    const int oy = int((i / Wo) % Ho);
    const int b = int(i / ((long long)Wo * Ho));
    __half* o = out + i * (split ? 2 * Kpad : Kpad);
    for (int k0 = 0; k0 < Kpad; k0 += 8) {
      __align__(16) __half v[8];
      __align__(16) __half lo[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int kk = k0 + j;
        float f = 0.f;
        if (kk < K) {
          const int c = kk % 3;
          const int tap = kk / 3;
          const int ky = tap / k, kx = tap - ky * k;
          const int y = oy * s - p + ky, x = ox * s - p + kx;
          if (y >= 0 && y < H && x >= 0 && x < W) f = lut[c * 256 + img[(((long long)b * H + y) * W + x) * 3 + c]];
        }
        v[j] = __float2half_rn(f);
        lo[j] = __float2half_rn(f - __half2float(v[j]));
      }
      *reinterpret_cast<uint4*>(o + k0) = *reinterpret_cast<const uint4*>(v);
      if (split)   // fp16x3 operand layout [hi | lo], see florence_ops.cu::store_act
        *reinterpret_cast<uint4*>(o + Kpad + k0) = *reinterpret_cast<const uint4*>(lo);
    }
  }
}

// ----------------------------------------------------------------------------------------- crop + resize
// One CTA per crop.  OpenCV resize (INTER_LINEAR, 8UC3): 11-bit coefficients, rows first horizontally into
// int32, then vertically: ((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2; exact 2x2 mean when the crop is 2x the
// output in both dimensions (OpenCV switches to INTER_AREA).
__global__ void crop_resize_kernel(const unsigned char* __restrict__ imgs, const int* __restrict__ img_hw /*[nimg][2]*/,
                                   const long long* __restrict__ img_off, const float* __restrict__ boxes /*[n][4] ratios*/,
                                   const int* __restrict__ box_img, int out_hw, unsigned char* __restrict__ out,
                                   int* __restrict__ status) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const int n = blockIdx.x;
  const int im = box_img[n];
  const int H = img_hw[2 * im], W = img_hw[2 * im + 1];
  const unsigned char* img = imgs + img_off[im];
  // ref:util/utils.py:99-100: int(coord * shape) on float32 tensors, truncation toward zero
  int xmin = __float2int_rz(__fmul_rn(boxes[4 * n + 0], float(W)));
  int ymin = __float2int_rz(__fmul_rn(boxes[4 * n + 1], float(H)));
  int xmax = __float2int_rz(__fmul_rn(boxes[4 * n + 2], float(W)));
  int ymax = __float2int_rz(__fmul_rn(boxes[4 * n + 3], float(H)));
  // numpy slicing clamps to the array bounds
  xmin = max(0, min(xmin, W)); xmax = max(0, min(xmax, W));
  ymin = max(0, min(ymin, H)); ymax = max(0, min(ymax, H));
  const int sw = xmax - xmin, sh = ymax - ymin;
  unsigned char* o = out + (long long)n * out_hw * out_hw * 3;
  if (sw <= 0 || sh <= 0) {   // cv2.resize raises -> the reference skips the crop (ref:util/utils.py:104-105)
    for (int i = threadIdx.x; i < out_hw * out_hw * 3; i += blockDim.x) o[i] = 0;
    if (threadIdx.x == 0) status[n] = 1;
    return;
  }
  if (threadIdx.x == 0) status[n] = 0;
  const unsigned char* src = img + ((long long)ymin * W + xmin) * 3;
  const long long rs = (long long)W * 3;
  if (sw == 2 * out_hw && sh == 2 * out_hw) {
    for (int i = threadIdx.x; i < out_hw * out_hw * 3; i += blockDim.x) {
      const int c = i % 3, dx = (i / 3) % out_hw, dy = i / (3 * out_hw);
      const unsigned char* p = src + (2 * dy) * rs + (2 * dx) * 3 + c;
      o[i] = (unsigned char)((p[0] + p[3] + p[rs] + p[rs + 3] + 2) >> 2);
    }
    return;
  }
  const double scale_x = 1.0 / (double(out_hw) / double(sw));
  const double scale_y = 1.0 / (double(out_hw) / double(sh));
  for (int i = threadIdx.x; i < out_hw * out_hw; i += blockDim.x) {
    const int dx = i % out_hw, dy = i / out_hw;
    float fx = float((dx + 0.5) * scale_x - 0.5);
    int sx = int(floorf(fx));
    fx -= float(sx);
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= sw - 1) { fx = 0.f; sx = sw - 1; }
    float fy = float((dy + 0.5) * scale_y - 0.5);
    const int sy = int(floorf(fy));
    fy -= float(sy);
    const int a0 = int(rintf((1.f - fx) * 2048.f)), a1 = int(rintf(fx * 2048.f));
    const int b0 = int(rintf((1.f - fy) * 2048.f)), b1 = int(rintf(fy * 2048.f));
    const int y0 = min(max(sy, 0), sh - 1), y1 = min(max(sy + 1, 0), sh - 1);
    const int x1 = min(sx + 1, sw - 1);
    const unsigned char* r0 = src + y0 * rs;
    const unsigned char* r1 = src + y1 * rs;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int S0 = r0[sx * 3 + c] * a0 + r0[x1 * 3 + c] * a1;
      const int S1 = r1[sx * 3 + c] * a0 + r1[x1 * 3 + c] * a1;
      const int v = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2;
      o[i * 3 + c] = (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
  }
}

static inline int grid_for(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  const long long cap = 132LL * 16;
  return int(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace b2p

using namespace b2p;

extern "C" {

// Host-side coefficient table exactly as Pillow computes it (exposed so CPU tests can pin it without a GPU).
int b2p_lanczos_coeffs_host(int in_size, int out_size, int* ksize, int* bounds /*[out][2]*/, int* kk /*[out][ksize_max]*/,
                            int kk_capacity) {
  std::vector<int> b, k;
  int ks = 0;
  host_lanczos_coeffs(in_size, out_size, &ks, b, k);
  *ksize = ks;
  if ((long long)k.size() > kk_capacity) return set_error("lanczos_coeffs_host: kk buffer too small");
  for (size_t i = 0; i < b.size(); ++i) bounds[i] = b[i];
  for (size_t i = 0; i < k.size(); ++i) kk[i] = k[i];
  return 0;
}

// src: device u8 [B][H][W][3]; tmp: device scratch [B][H][Wr][3]; canvas: device u8 [B][Th][Tw][3].
// (Wr, Hr) = resized size, pasted at (pad_l, pad_t); ref:util/yolov9.py:73-84.
int b2p_letterbox(const unsigned char* src, int B, int H, int W, int Wr, int Hr, int Tw, int Th, int pad_l, int pad_t,
                  unsigned char* tmp, unsigned char* canvas, cudaStream_t st) {
  // Pillow raises on an empty resize; an empty coefficient table would otherwise leave an all-114 canvas
  if (W < 1 || H < 1 || Wr < 1 || Hr < 1) return set_error("letterbox: source and resized sizes must be >= 1");
  if (pad_l < 0 || pad_t < 0 || pad_l + Wr > Tw || pad_t + Hr > Th)
    return set_error("letterbox: the resized image must lie inside the canvas");
  const unsigned char* hsrc = src;
  int hW = W;
  if (Wr != W) {   // Pillow skips a pass whose size does not change
    Coeffs ch;
    if (int e = get_coeffs(W, Wr, &ch)) return e;
    lanczos_h_kernel<<<grid_for((long long)B * H * Wr, 256), 256, 0, st>>>(src, B, H, W, Wr, ch.d_bounds, ch.d_kk, ch.ksize, tmp);
    B2P_CHECK_LAUNCH();
    hsrc = tmp;
    hW = Wr;
  }
  Coeffs cv{};
  if (Hr != H)
    if (int e = get_coeffs(H, Hr, &cv)) return e;
  launch_pdl(lanczos_v_paste_kernel, dim3(grid_for((long long)B * Th * Tw, 256)), dim3(256), 0, st, hsrc, B, H, hW, Hr, cv.d_bounds, cv.d_kk, cv.ksize,
                                                                              Tw, Th, pad_l, pad_t, canvas);
  B2P_CHECK_LAUNCH();
  return 0;
}

// Host only: the descriptors, packed tables and buffer sizes of one ragged letterbox batch (include/b200parse.h).
int b2p_letterbox_batch_plan_host(int B, const int* geom_host, int Tw, int Th, long long* desc_host, int* tables_host,
                                  long long tables_capacity, long long* sizes_host) {
  if (B < 1 || B > 65535) return set_error("letterbox_batch_plan: B must be in [1, 65535]");
  for (int b = 0; b < B; ++b) {
    const int* g = geom_host + 6LL * b;
    if (int e = lb_check_geometry(g[0], g[1], g[2], g[3], g[4], g[5], Tw, Th, "letterbox_batch_plan")) return e;
  }
  // tables: one copy per distinct (in, out) pair of the batch
  std::vector<long long> desc(size_t(B) * kLbDesc);
  std::vector<std::pair<std::pair<int, int>, long long>> placed;   // (in, out) -> element offset
  std::vector<PackedTable> order;
  long long n_tab = 0, tmp_bytes = 0, src_bytes = 0;
  auto place = [&](int in, int out, long long* off, long long* ks) {
    for (size_t j = 0; j < placed.size(); ++j)
      if (placed[j].first == std::make_pair(in, out)) { *off = placed[j].second; *ks = order[j].ksize; return; }
    PackedTable t = lb_table(in, out);
    placed.emplace_back(std::make_pair(in, out), n_tab);
    *off = n_tab;
    *ks = t.ksize;
    n_tab += (long long)t.data.size();
    order.push_back(std::move(t));
  };
  for (int b = 0; b < B; ++b) {
    const int* g = geom_host + 6LL * b;
    const int H = g[0], W = g[1], Wr = g[2], Hr = g[3];
    long long* d = desc.data() + size_t(b) * kLbDesc;
    d[kLbSrc] = src_bytes;
    src_bytes += 3LL * H * W;
    d[kLbH] = H; d[kLbW] = W; d[kLbWr] = Wr; d[kLbHr] = Hr; d[kLbPadL] = g[4]; d[kLbPadT] = g[5];
    d[kLbTmp] = d[kLbHTab] = d[kLbHK] = d[kLbVTab] = d[kLbVK] = -1;
    if (Wr != W) {   // Pillow skips a pass whose size does not change
      d[kLbTmp] = tmp_bytes;
      tmp_bytes += 3LL * H * Wr;
      place(W, Wr, &d[kLbHTab], &d[kLbHK]);
    }
    if (Hr != H) place(H, Hr, &d[kLbVTab], &d[kLbVK]);
  }
  if (tables_host && tables_capacity < n_tab) return set_error("letterbox_batch_plan: the table buffer is too small");
  sizes_host[0] = n_tab; sizes_host[1] = tmp_bytes; sizes_host[2] = src_bytes;
  if (!tables_host) return 0;
  memcpy(desc_host, desc.data(), desc.size() * sizeof(long long));
  for (size_t j = 0; j < order.size(); ++j)
    memcpy(tables_host + placed[j].second, order[j].data.data(), order[j].data.size() * sizeof(int));
  return 0;
}

// src / tmp: flat device buffers addressed by the descriptors' byte offsets; canvas: device u8 [B][Th][Tw][3].
int b2p_letterbox_batch(const unsigned char* src, int B, const long long* desc_host, const long long* desc, const int* tables,
                        int Tw, int Th, unsigned char* tmp, unsigned char* canvas, cudaStream_t st) {
  if (B < 1 || B > 65535) return set_error("letterbox_batch: B must be in [1, 65535]");
  if (Tw < 1 || Th < 1) return set_error("letterbox_batch: the canvas must be at least 1 x 1");
  long long h_max = 0;
  for (int b = 0; b < B; ++b) {
    const long long* d = desc_host + (long long)b * kLbDesc;
    if (int e = lb_check_geometry(d[kLbH], d[kLbW], d[kLbWr], d[kLbHr], d[kLbPadL], d[kLbPadT], Tw, Th, "letterbox_batch"))
      return e;
    const bool h = d[kLbWr] != d[kLbW], v = d[kLbHr] != d[kLbH];
    if (d[kLbSrc] < 0 || h != (d[kLbHTab] >= 0) || v != (d[kLbVTab] >= 0) || (h && (d[kLbHK] < 1 || d[kLbTmp] < 0)) ||
        (v && d[kLbVK] < 1))
      return set_error("letterbox_batch: a descriptor's offsets or tables disagree with its geometry");
    if (h) h_max = std::max(h_max, d[kLbH] * d[kLbWr]);
  }
  const long long cap = std::max(1LL, (132LL * 16 + B - 1) / B);   // grid_for's cap, shared by the images
  if (h_max) {
    lanczos_h_batch_kernel<<<dim3(unsigned(std::min(cap, (h_max + 255) / 256)), B), 256, 0, st>>>(src, desc, tables, tmp);
    B2P_CHECK_LAUNCH();
  }
  const long long v_chunks = std::min(cap, ((long long)Tw * Th + 255) / 256);
  launch_pdl(lanczos_v_paste_batch_kernel, dim3(unsigned(v_chunks), B), dim3(256), 0, st, src, desc, tables,
             (const unsigned char*)tmp, Tw, Th, canvas);
  B2P_CHECK_LAUNCH();
  return 0;
}

// Pillow-exact resize of u8 HWC images (filter 0 = LANCZOS, 1 = BICUBIC), no padding: [B][H][W][3] -> [B][Hr][Wr][3].
int b2p_resize_u8(const unsigned char* src, int B, int H, int W, int Wr, int Hr, int filter, unsigned char* tmp,
                  unsigned char* out, cudaStream_t st) {
  if (filter != 0 && filter != 1) return set_error("resize_u8: filter must be 0 (LANCZOS) or 1 (BICUBIC)");
  if (W < 1 || H < 1 || Wr < 1 || Hr < 1) return set_error("resize_u8: source and resized sizes must be >= 1");
  const unsigned char* hsrc = src;
  int hW = W;
  if (Wr != W) {
    Coeffs ch;
    if (int e = get_coeffs(W, Wr, &ch, filter)) return e;
    lanczos_h_kernel<<<grid_for((long long)B * H * Wr, 256), 256, 0, st>>>(src, B, H, W, Wr, ch.d_bounds, ch.d_kk, ch.ksize, tmp);
    B2P_CHECK_LAUNCH();
    hsrc = tmp;
    hW = Wr;
  }
  Coeffs cv{};
  if (Hr != H)
    if (int e = get_coeffs(H, Hr, &cv, filter)) return e;
  launch_pdl(lanczos_v_paste_kernel, dim3(grid_for((long long)B * Hr * Wr, 256)), dim3(256), 0, st, hsrc, B, H, hW, Hr, cv.d_bounds,
             cv.d_kk, cv.ksize, Wr, Hr, 0, 0, out);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_im2col_u8(const unsigned char* img, int B, int H, int W, int k, int s, int p, int Kpad, const float* lut,
                  void* out, int split, cudaStream_t st) {
  if (Kpad % 8 || Kpad < k * k * 3) return set_error("im2col_u8: Kpad must be a multiple of 8 and >= 3*k*k");
  const int Ho = (H + 2 * p - k) / s + 1, Wo = (W + 2 * p - k) / s + 1;
  launch_pdl(im2col_u8_kernel, dim3(grid_for((long long)B * Ho * Wo, 128)), dim3(128), 0, st, img, B, H, W, k, s, p, Ho, Wo, Kpad, lut, (__half*)out, split);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_crop_resize(const unsigned char* imgs, const int* img_hw, const long long* img_off, const float* boxes,
                    const int* box_img, int n_box, int out_hw, unsigned char* out, int* status, cudaStream_t st) {
  if (n_box <= 0) return 0;
  launch_pdl(crop_resize_kernel, dim3(n_box), dim3(256), 0, st, imgs, img_hw, img_off, boxes, box_img, out_hw, out, status);
  B2P_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
