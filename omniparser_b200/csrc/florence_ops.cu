// Non-GEMM kernels of the Florence-2 caption path (ref:util/utils.py:125 -> HF generate): LayerNorm, DaViT
// depthwise conv / window attention / channel attention, BART multi-head attention with KV cache, embedding +
// position + LayerNorm, image-token projector prep, and the greedy token pick with HF logits processors.
// All are HBM/latency-bound SIMT kernels in fp32; the dense contractions run in gemm_wgmma.cu.
// Residual streams are fp32, GEMM operands fp16.
#include "b2p_internal.h"
#include <atomic>
#include <cuda_fp16.h>
#include <math.h>

namespace b2p {

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// fp16 activation store.  split == 0: plain.  split == K > 0: "fp16x3" operand layout [hi(K) | lo(K)] (row stride 2K):
// the GEMM loads both halves of A and of W = [W_hi | W_lo] once per k-block and accumulates hi*hi + hi*lo + lo*hi in
// fp32 (2^-22-class products instead of 2^-11): the parity-grade precision mode of the caption path.
__device__ __forceinline__ void store_act(__half* row, int c, int split, float v) {
  const __half h = __float2half_rn(v);
  row[c] = h;
  if (split) row[split + c] = __float2half_rn(v - __half2float(h));
}

// 4 consecutive channels (c % 4 == 0) as one 8-byte store per copy
__device__ __forceinline__ void store_act4(__half* row, int c, int split, const float4& v) {
  __align__(8) __half2 h[2] = {__floats2half2_rn(v.x, v.y), __floats2half2_rn(v.z, v.w)};
  *reinterpret_cast<uint2*>(row + c) = *reinterpret_cast<const uint2*>(h);
  if (split) {
    const float2 a = __half22float2(h[0]), b = __half22float2(h[1]);
    __align__(8) __half2 l[2] = {__floats2half2_rn(v.x - a.x, v.y - a.y), __floats2half2_rn(v.z - b.x, v.w - b.y)};
    *reinterpret_cast<uint2*>(row + split + c) = *reinterpret_cast<const uint2*>(l);
  }
}

// ---------------------------------------------------------------------------------------- LayerNorm
// one warp per row; x fp32 [T][ldx]; writes fp16 and/or fp32 (nn.LayerNorm, biased variance, eps inside sqrt)
__global__ void layernorm_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ g,
                                 const float* __restrict__ b, float eps, int T, int C, __half* __restrict__ o16,
                                 long long ld16, float* __restrict__ o32, long long ld32, int split) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= T) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)row * ldx);
  const int C4 = C >> 2;
  float4 v[8];   // C <= 1024
  float s = 0.f;
  int n = 0;
  for (int c = lane; c < C4; c += 32, ++n) { v[n] = xr[c]; s += (v[n].x + v[n].y) + (v[n].z + v[n].w); }
  const float mean = warp_sum(s) / float(C);
  float q = 0.f;
  for (int i = 0; i < n; ++i) {
    const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
  const float rstd = rsqrtf(warp_sum(q) / float(C) + eps);
  n = 0;
  for (int c = lane; c < C4; c += 32, ++n) {
    const float4 gg = reinterpret_cast<const float4*>(g)[c], bb = reinterpret_cast<const float4*>(b)[c];
    float4 y;
    y.x = (v[n].x - mean) * rstd * gg.x + bb.x; y.y = (v[n].y - mean) * rstd * gg.y + bb.y;
    y.z = (v[n].z - mean) * rstd * gg.z + bb.z; y.w = (v[n].w - mean) * rstd * gg.w + bb.w;
    if (o16) store_act4(o16 + (long long)row * ld16, 4 * c, split, y);
    if (o32) reinterpret_cast<float4*>(o32 + (long long)row * ld32)[c] = y;
  }
}

// Split-K reduction + bias + residual + LayerNorm in one pass over the partial tiles a park-only GEMM left in the split-K
// workspace (gemm_wgmma.cu, GemmArgs::park): the decoder's out-proj / cross out-proj / fc2 GEMMs (N = 768, M = crops) are
// split-K launches followed by a LayerNorm; inside the GEMM the slices had to wait for each other and re-read the partials,
// and the LayerNorm was one more launch.  One warp per row.  Same arithmetic in the same order as
// the GEMM epilogue (slices in order, + bias, + residual) and layernorm_kernel => bit-identical results.
__global__ void splitk_ln_kernel(ParkInfo pk, int M, int N, const float* __restrict__ bias, const float* __restrict__ res, long long ldr,
                                 const float* __restrict__ g, const float* __restrict__ b, float eps, __half* __restrict__ o16,
                                 long long ld16, float* __restrict__ o32, long long ld32, int split) {
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const int mt = row >> 7, r = row & 127;
  const int C4 = N >> 2;
  const size_t sl_stride = size_t(128) * pk.bn;     // floats between consecutive k slices of a tile
  float4 v[8];   // N <= 1024
  float s = 0.f;
  int n = 0;
  for (int c = lane; c < C4; c += 32, ++n) {
    const int col = 4 * c;
    const int nt = col / pk.bn, cc = col - nt * pk.bn;
    const int tile = pk.mt_fast ? nt * pk.m_tiles + mt : mt * pk.n_tiles + nt;
    const float* p = pk.ws + (size_t(tile) * pk.ksplit * 128 + r) * pk.bn + cc;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    int sidx = 0;
    for (; sidx + 2 <= pk.ksplit; sidx += 2) {       // two slices in flight; adds in slice order
      const float4 t0 = __ldcg(reinterpret_cast<const float4*>(p + size_t(sidx) * sl_stride));
      const float4 t1 = __ldcg(reinterpret_cast<const float4*>(p + size_t(sidx + 1) * sl_stride));
      a.x += t0.x; a.y += t0.y; a.z += t0.z; a.w += t0.w;
      a.x += t1.x; a.y += t1.y; a.z += t1.z; a.w += t1.w;
    }
    if (sidx < pk.ksplit) {
      const float4 t0 = __ldcg(reinterpret_cast<const float4*>(p + size_t(sidx) * sl_stride));
      a.x += t0.x; a.y += t0.y; a.z += t0.z; a.w += t0.w;
    }
    if (bias) {
      const float4 bb = reinterpret_cast<const float4*>(bias)[c];
      a.x += bb.x; a.y += bb.y; a.z += bb.z; a.w += bb.w;
    }
    if (res) {
      const float4 rr = reinterpret_cast<const float4*>(res + (long long)row * ldr)[c];
      a.x += rr.x; a.y += rr.y; a.z += rr.z; a.w += rr.w;
    }
    v[n] = a;
    s += (a.x + a.y) + (a.z + a.w);
  }
  const float mean = warp_sum(s) / float(N);
  float q = 0.f;
  for (int i = 0; i < n; ++i) {
    const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
  const float rstd = rsqrtf(warp_sum(q) / float(N) + eps);
  n = 0;
  for (int c = lane; c < C4; c += 32, ++n) {
    const float4 gg = reinterpret_cast<const float4*>(g)[c], bb = reinterpret_cast<const float4*>(b)[c];
    float4 y;
    y.x = (v[n].x - mean) * rstd * gg.x + bb.x; y.y = (v[n].y - mean) * rstd * gg.y + bb.y;
    y.z = (v[n].z - mean) * rstd * gg.z + bb.z; y.w = (v[n].w - mean) * rstd * gg.w + bb.w;
    if (o16) store_act4(o16 + (long long)row * ld16, 4 * c, split, y);
    if (o32) reinterpret_cast<float4*>(o32 + (long long)row * ld32)[c] = y;
  }
}

// Fused DaViT pre-block: y = dwconv3x3(x) + bias + x (fp32, the new residual stream) and h = LayerNorm(y) as the next
// GEMM operand.  One warp per token; channels in float4 lanes (C <= 1024).
__global__ void dwconv_ln_kernel(const float* __restrict__ x, int B, int H, int W, int C, const float* __restrict__ w9c,
                                 const float* __restrict__ bias, float* __restrict__ y, const float* __restrict__ g,
                                 const float* __restrict__ bt, float eps, __half* __restrict__ o16, int split) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const long long tok = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (tok >= (long long)B * H * W) return;
  const int xx = int(tok % W), yy = int((tok / W) % H);
  const int C4 = C >> 2;
  float4 v[8];
  float s = 0.f;
  int n = 0;
  for (int c = lane; c < C4; c += 32, ++n) {
    float4 acc = reinterpret_cast<const float4*>(bias)[c];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int sy = yy + ky - 1;
      if (sy < 0 || sy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int sx = xx + kx - 1;
        if (sx < 0 || sx >= W) continue;
        const float4 xv = reinterpret_cast<const float4*>(x + (tok + (long long)(ky - 1) * W + (kx - 1)) * C)[c];
        const float4 wv = reinterpret_cast<const float4*>(w9c + (ky * 3 + kx) * C)[c];
        acc.x += xv.x * wv.x; acc.y += xv.y * wv.y; acc.z += xv.z * wv.z; acc.w += xv.w * wv.w;
      }
    }
    const float4 xc = reinterpret_cast<const float4*>(x + tok * C)[c];
    acc.x += xc.x; acc.y += xc.y; acc.z += xc.z; acc.w += xc.w;
    reinterpret_cast<float4*>(y + tok * C)[c] = acc;
    v[n] = acc;
    s += (acc.x + acc.y) + (acc.z + acc.w);
  }
  const float mean = warp_sum(s) / float(C);
  float q = 0.f;
  for (int i = 0; i < n; ++i) {
    const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
  const float rstd = rsqrtf(warp_sum(q) / float(C) + eps);
  n = 0;
  __half* orow = o16 + tok * (split ? 2 * C : C);
  for (int c = lane; c < C4; c += 32, ++n) {
    const float4 gg = reinterpret_cast<const float4*>(g)[c], bb = reinterpret_cast<const float4*>(bt)[c];
    float4 o;
    o.x = (v[n].x - mean) * rstd * gg.x + bb.x; o.y = (v[n].y - mean) * rstd * gg.y + bb.y;
    o.z = (v[n].z - mean) * rstd * gg.z + bb.z; o.w = (v[n].w - mean) * rstd * gg.w + bb.w;
    store_act4(orow, 4 * c, split, o);
  }
}

// Tiled variant (split bit 1; the default, B2P_NO_DWCONV_TILE=1 disables it): one CTA
// per image stages the whole H x W x C map in shared memory once, so the nine taps read smem instead of re-reading L2 nine
// times (the per-token kernel above moves ~36 B per element through L2).  Same
// arithmetic in the same order as dwconv_ln_kernel => bit-identical outputs (tests/test_ops_gpu.py, gated).
__global__ void dwconv_ln_tile_kernel(const float* __restrict__ x, int H, int W, int C, const float* __restrict__ w9c,
                                      const float* __restrict__ bias, float* __restrict__ y, const float* __restrict__ g,
                                      const float* __restrict__ bt, float eps, __half* __restrict__ o16, int split) {
  pdl_wait();
  extern __shared__ float4 xs4[];   // [H*W][C/4]
  const int HW = H * W, C4 = C >> 2;
  const long long tok0 = (long long)blockIdx.x * HW;
  const float4* xin = reinterpret_cast<const float4*>(x + tok0 * C);
  for (int i = threadIdx.x; i < HW * C4; i += blockDim.x) xs4[i] = xin[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int t = warp; t < HW; t += nw) {
    const int xx = t % W, yy = t / W;
    const long long tok = tok0 + t;
    float4 v[8];
    float s = 0.f;
    int n = 0;
    for (int c = lane; c < C4; c += 32, ++n) {
      float4 acc = reinterpret_cast<const float4*>(bias)[c];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int sy = yy + ky - 1;
        if (sy < 0 || sy >= H) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int sx = xx + kx - 1;
          if (sx < 0 || sx >= W) continue;
          const float4 xv = xs4[(t + (ky - 1) * W + (kx - 1)) * C4 + c];
          const float4 wv = reinterpret_cast<const float4*>(w9c + (ky * 3 + kx) * C)[c];
          acc.x += xv.x * wv.x; acc.y += xv.y * wv.y; acc.z += xv.z * wv.z; acc.w += xv.w * wv.w;
        }
      }
      const float4 xc = xs4[t * C4 + c];
      acc.x += xc.x; acc.y += xc.y; acc.z += xc.z; acc.w += xc.w;
      reinterpret_cast<float4*>(y + tok * C)[c] = acc;
      v[n] = acc;
      s += (acc.x + acc.y) + (acc.z + acc.w);
    }
    const float mean = warp_sum(s) / float(C);
    float q = 0.f;
    for (int i = 0; i < n; ++i) {
      const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    const float rstd = rsqrtf(warp_sum(q) / float(C) + eps);
    n = 0;
    __half* orow = o16 + tok * (split ? 2 * C : C);
    for (int c = lane; c < C4; c += 32, ++n) {
      const float4 gg = reinterpret_cast<const float4*>(g)[c], bb = reinterpret_cast<const float4*>(bt)[c];
      float4 o;
      o.x = (v[n].x - mean) * rstd * gg.x + bb.x; o.y = (v[n].y - mean) * rstd * gg.y + bb.y;
      o.z = (v[n].z - mean) * rstd * gg.z + bb.z; o.w = (v[n].w - mean) * rstd * gg.w + bb.w;
      store_act4(orow, 4 * c, split, o);
    }
  }
}

// ---------------------------------------------------------------------------------------- depthwise 3x3 + residual
// y = dwconv3x3(x) + bias + x   (hf:models/florence2/modeling_florence2.py:281,293 and :431,443)
__global__ void dwconv3x3_res_kernel(const float* __restrict__ x, int B, int H, int W, int C,
                                     const float* __restrict__ w /*[9][C]*/, const float* __restrict__ bias,
                                     float* __restrict__ y) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const long long n = (long long)B * H * W * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % C);
    long long p = i / C;
    const int xx = int(p % W); p /= W;
    const int yy = int(p % H);
    const int b = int(p / H);
    float acc = bias[c];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int sy = yy + ky - 1;
      if (sy < 0 || sy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int sx = xx + kx - 1;
        if (sx < 0 || sx >= W) continue;
        acc += x[(((long long)b * H + sy) * W + sx) * C + c] * w[(ky * 3 + kx) * C + c];
      }
    }
    y[i] = acc + x[i];
  }
}

// ---------------------------------------------------------------------------------------- window attention
// qkv fp16 [B*H*W][3C] for REAL tokens only.  The reference zero-pads the normed map to a multiple of the 12x12
// window; padded tokens have qkv = bias and take part as keys/values unmasked
// (hf:models/florence2/modeling_florence2.py:346-350,377-383).  Exact shortcut: one "pad key" (k = bias_k,
// v = bias_v) with multiplicity n_pad = 144 - n_real.  One CTA per (batch, window, head); one thread per query.
// QB queries per thread (t, t + ceil(nreal / QB), ...): every K / V row read from shared memory feeds QB independent
// online-softmax chains.  Only QB = 1 is instantiated (see b2p_window_attn).
template <int D, int QB>
__global__ void window_attn_kernel(const float* __restrict__ qkv, const float* __restrict__ qkv_bias, int B, int H,
                                   int W, int C, int heads, int win, __half* __restrict__ out, int split, int kv_cap) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  extern __shared__ float4 sm4[];
  constexpr int D4 = D / 4;
  const int nwx = (W + win - 1) / win, nwy = (H + win - 1) / win;
  int bid = blockIdx.x;
  const int head = bid % heads; bid /= heads;
  const int wx = bid % nwx; bid /= nwx;
  const int wy = bid % nwy;
  const int b = bid / nwy;
  const int y0 = wy * win, x0 = wx * win;
  const int ny = min(win, H - y0), nx = min(win, W - x0);
  const int nreal = ny * nx, npad = win * win - nreal;
  float4* Ks = sm4;                       // [nreal][D4]
  float4* Vs = sm4 + kv_cap * D4;         // [nreal][D4]; kv_cap = most real tokens any window of this map holds
  for (int i = threadIdx.x; i < nreal * D4; i += blockDim.x) {
    const int t = i / D4, d = i - t * D4;
    const long long tok = ((long long)b * H + y0 + t / nx) * W + x0 + t % nx;
    Ks[i] = reinterpret_cast<const float4*>(qkv + tok * 3 * C + C + head * D)[d];
    Vs[i] = reinterpret_cast<const float4*>(qkv + tok * 3 * C + 2 * C + head * D)[d];
  }
  __syncthreads();
  const float scale = rsqrtf(float(D));
  const int nq = (nreal + QB - 1) / QB;
  for (int t0 = threadIdx.x; t0 < nq; t0 += blockDim.x) {
    long long tok[QB];
    bool live[QB];
    float4 q[QB][D4], acc[QB][D4];
    float m[QB], l[QB];
#pragma unroll
    for (int u = 0; u < QB; ++u) {
      const int t = t0 + u * nq;
      live[u] = t < nreal;
      const int tc = live[u] ? t : t0;      // a dead slot recomputes query t0 and stores nothing
      tok[u] = ((long long)b * H + y0 + tc / nx) * W + x0 + tc % nx;
#pragma unroll
      for (int d = 0; d < D4; ++d) {
        q[u][d] = reinterpret_cast<const float4*>(qkv + tok[u] * 3 * C + head * D)[d];
        q[u][d].x *= scale; q[u][d].y *= scale; q[u][d].z *= scale; q[u][d].w *= scale;
        acc[u][d] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      m[u] = -INFINITY; l[u] = 0.f;
    }
    if (npad > 0) {
#pragma unroll
      for (int u = 0; u < QB; ++u) {
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < D4; ++d) {
          const float4 kb = reinterpret_cast<const float4*>(qkv_bias + C + head * D)[d];
          s += (q[u][d].x * kb.x + q[u][d].y * kb.y) + (q[u][d].z * kb.z + q[u][d].w * kb.w);
        }
        m[u] = s;
        l[u] = float(npad);
#pragma unroll
        for (int d = 0; d < D4; ++d) {
          const float4 vb = reinterpret_cast<const float4*>(qkv_bias + 2 * C + head * D)[d];
          acc[u][d] = make_float4(l[u] * vb.x, l[u] * vb.y, l[u] * vb.z, l[u] * vb.w);
        }
      }
    }
    for (int j = 0; j < nreal; ++j) {
      float s[QB], p[QB];
#pragma unroll
      for (int u = 0; u < QB; ++u) s[u] = 0.f;
#pragma unroll
      for (int d = 0; d < D4; ++d) {
        const float4 kk = Ks[j * D4 + d];
#pragma unroll
        for (int u = 0; u < QB; ++u) s[u] += (q[u][d].x * kk.x + q[u][d].y * kk.y) + (q[u][d].z * kk.z + q[u][d].w * kk.w);
      }
#pragma unroll
      for (int u = 0; u < QB; ++u) {
        if (s[u] > m[u]) {
          const float r = __expf(m[u] - s[u]);
          l[u] *= r;
#pragma unroll
          for (int d = 0; d < D4; ++d) { acc[u][d].x *= r; acc[u][d].y *= r; acc[u][d].z *= r; acc[u][d].w *= r; }
          m[u] = s[u];
        }
        p[u] = __expf(s[u] - m[u]);
        l[u] += p[u];
      }
#pragma unroll
      for (int d = 0; d < D4; ++d) {
        const float4 vv = Vs[j * D4 + d];
#pragma unroll
        for (int u = 0; u < QB; ++u) {
          acc[u][d].x += p[u] * vv.x; acc[u][d].y += p[u] * vv.y; acc[u][d].z += p[u] * vv.z; acc[u][d].w += p[u] * vv.w;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < QB; ++u) {
      if (!live[u]) continue;
      const float inv = 1.f / l[u];
      __half* orow = out + tok[u] * (split ? 2 * C : C);
#pragma unroll
      for (int d = 0; d < D4; ++d)
        store_act4(orow, head * D + 4 * d, split, make_float4(acc[u][d].x * inv, acc[u][d].y * inv, acc[u][d].z * inv, acc[u][d].w * inv));
    }
  }
}

// ---------------------------------------------------------------------------------------- channel attention
// hf:models/florence2/modeling_florence2.py:228-264: per (batch, group) a d x d (d = 32) attention over channels:
// S[i][j] = N^-0.5 * sum_n q[n][i] k[n][j]; P = softmax_j(S); out[n][i] = sum_j P[i][j] v[n][j].
// One CTA (256 threads = 8 warps x 32 columns) per (batch, group); tokens streamed through shared memory in chunks.
// Each chunk's 64 products are summed in fp32 into a fresh register and the chunk sums are added in fp64, in chunk order.
// One fp32 running sum over all N tokens lost ~eps * N^1.5 when the inputs have a non-zero mean (they are a biased linear
// layer's output): at the 768 mode's 36 864 tokens the [hi | lo] outputs were 21x over their 2e-5 bound
// (tests/test_davit_kernels_gpu.py).  N <= 64 is one chunk: the same sums as before, so channel_attn_small_kernel stays
// bit-identical with this kernel (float(double(s) * sc) is the fp32 product s * sc).
__global__ void __launch_bounds__(256) channel_attn_kernel(const float* __restrict__ qkv, int N, int C, int groups,
                                                           __half* __restrict__ out, int split) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  constexpr int D = 32, CH = 64;
  __shared__ float qs[CH][D + 1], ks[CH][D + 1];
  __shared__ float P[D][D + 1];
  const int g = blockIdx.x % groups, b = blockIdx.x / groups;
  const int w = threadIdx.x >> 5, j = threadIdx.x & 31;   // warp w owns rows i = 4w .. 4w+3, lane = column j
  const float* base = qkv + (long long)b * N * 3 * C;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int n0 = 0; n0 < N; n0 += CH) {
    const int cn = min(CH, N - n0);
    for (int t = threadIdx.x; t < cn * D; t += blockDim.x) {
      const int n = t / D, d = t - n * D;
      qs[n][d] = base[(long long)(n0 + n) * 3 * C + g * D + d];
      ks[n][d] = base[(long long)(n0 + n) * 3 * C + C + g * D + d];
    }
    __syncthreads();
    float cs[4] = {0.f, 0.f, 0.f, 0.f};
    for (int n = 0; n < cn; ++n) {
      const float kv = ks[n][j];
#pragma unroll
      for (int r = 0; r < 4; ++r) cs[r] += qs[n][4 * w + r] * kv;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) s[r] += double(cs[r]);
    __syncthreads();
  }
  const float sc = rsqrtf(float(N));
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const float v = float(s[r] * double(sc));
    const float m = warp_max(v);
    const float e = __expf(v - m);
    P[4 * w + r][j] = e / warp_sum(e);
  }
  __syncthreads();
  // out[n][g*32 + j] = sum_jj P[j][jj] v[n][jj]: 8 tokens per pass (one per warp), lane = output channel j
  float pr[D];
#pragma unroll
  for (int jj = 0; jj < D; ++jj) pr[jj] = P[j][jj];
  for (int n = w; n < N; n += 8) {
    const float* vr = base + (long long)n * 3 * C + 2 * C + g * D;
    const float vj = vr[j];
    float acc = 0.f;
#pragma unroll
    for (int jj = 0; jj < D; ++jj) acc += pr[jj] * __shfl_sync(0xffffffffu, vj, jj);
    store_act(out + ((long long)b * N + n) * (split ? 2 * C : C), g * D + j, split, acc);
  }
}

// Small-N variant (split bit 1; the default, B2P_NO_CHATTN_SMALL=1 disables it): for
// the 4x4 / 2x2 maps of the 64x64-crop mode (N <= 16 tokens) the 256-thread CTA above is almost all synchronisation; here
// ONE WARP owns a (batch, group) pair, 4 pairs per CTA.  Same sums in the same order => bit-identical outputs.
__global__ void __launch_bounds__(128) channel_attn_small_kernel(const float* __restrict__ qkv, int B, int N, int C, int groups,
                                                                 __half* __restrict__ out, int split) {
  pdl_wait();
  constexpr int D = 32, NMAX = 16;
  __shared__ float sm[4][2 * NMAX + D][D + 1];   // per warp: q rows [0,N), k rows [NMAX, NMAX+N), P rows [2*NMAX, 2*NMAX+32)
  const int w = threadIdx.x >> 5, j = threadIdx.x & 31;
  const int pair = blockIdx.x * 4 + w;
  if (pair >= B * groups) return;
  const int g = pair % groups, b = pair / groups;
  float (*qs)[D + 1] = sm[w];
  float (*ks)[D + 1] = sm[w] + NMAX;
  float (*P)[D + 1] = sm[w] + 2 * NMAX;
  const float* base = qkv + (long long)b * N * 3 * C;
  for (int n = 0; n < N; ++n) {
    qs[n][j] = base[(long long)n * 3 * C + g * D + j];
    ks[n][j] = base[(long long)n * 3 * C + C + g * D + j];
  }
  __syncwarp();
  const float sc = rsqrtf(float(N));
  for (int i = 0; i < D; ++i) {
    float s = 0.f;
    for (int n = 0; n < N; ++n) s += qs[n][i] * ks[n][j];
    const float v = s * sc;
    const float m = warp_max(v);
    const float e = __expf(v - m);
    P[i][j] = e / warp_sum(e);
  }
  __syncwarp();
  float pr[D];
#pragma unroll
  for (int jj = 0; jj < D; ++jj) pr[jj] = P[j][jj];
  for (int n = 0; n < N; ++n) {
    const float vj = base[(long long)n * 3 * C + 2 * C + g * D + j];
    float acc = 0.f;
#pragma unroll
    for (int jj = 0; jj < D; ++jj) acc += pr[jj] * __shfl_sync(0xffffffffu, vj, jj);
    store_act(out + ((long long)b * N + n) * (split ? 2 * C : C), g * D + j, split, acc);
  }
}

// ---------------------------------------------------------------------------------------- BART attention
// One warp per (batch, head, query).  d_head = 64 (2 values per lane), scale applied to q (hf:models/bart/
// modeling_bart.py:143-258).  K/V row b*Lk + j at k + (b*Lk + j)*ldk + h*64.  Decoder self-attention: the current
// step's k, v (columns of the fused qkv GEMM output) are appended to the cache at position *step, and the
// attention covers cache[0..*step].
struct MhaArgs {
  const float* q; long long ldq;
  const float* k; const float* v; long long ldk;     // encoder / cross: [B*Lk][ldk]
  float* kcache; float* vcache; int tmax;             // decoder self: cache [B][tmax][heads*64]
  const float* knew; const float* vnew; long long ldnew;
  const int* step;
  int B, Lq, Lk, heads;
  __half* out; long long ldo; int split;
  const int* src; int rows_per_kv;                    // beam layout only (kBeam), see below
};

// kBeam = false: the greedy decoder / encoder layout above.  kBeam = true, beam search (R = crops * num_beams rows):
//  - cached: row b's cache entry for position j < *step lives in physical row src[b][j] (src [B][tmax], kept by
//    b2p_beam_update), the current position in row b itself, so a beam reorder never moves the caches;
//  - explicit K / V: row b reads batch b / rows_per_kv (the cross-attention K / V of its crop, shared by its beams).
template <bool kBeam>
__global__ void mha_kernel(MhaArgs a) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int total = a.B * a.heads * a.Lq;
  if (wid >= total) return;
  const int qi = wid % a.Lq;
  const int h = (wid / a.Lq) % a.heads;
  const int b = wid / (a.Lq * a.heads);
  const int HD = a.heads * 64;
  float2 q = *reinterpret_cast<const float2*>(a.q + ((long long)b * a.Lq + qi) * a.ldq + h * 64 + 2 * lane);
  q.x *= 0.125f; q.y *= 0.125f;
  int Lk = a.Lk;
  const float *kb, *vb;
  long long ldk;
  const int* srow = nullptr;   // kBeam, cached: physical cache row of every position < t
  int t = 0;
  if (a.kcache) {
    t = *a.step;
    // append this step's k, v
    const float2 kn = *reinterpret_cast<const float2*>(a.knew + (long long)b * a.ldnew + h * 64 + 2 * lane);
    const float2 vn = *reinterpret_cast<const float2*>(a.vnew + (long long)b * a.ldnew + h * 64 + 2 * lane);
    *reinterpret_cast<float2*>(a.kcache + ((long long)b * a.tmax + t) * HD + h * 64 + 2 * lane) = kn;
    *reinterpret_cast<float2*>(a.vcache + ((long long)b * a.tmax + t) * HD + h * 64 + 2 * lane) = vn;
    __syncwarp();
    Lk = t + 1;
    kb = a.kcache + (long long)b * a.tmax * HD + h * 64;
    vb = a.vcache + (long long)b * a.tmax * HD + h * 64;
    ldk = HD;
    if (kBeam) {
      srow = a.src + (long long)b * a.tmax;
      kb = a.kcache + h * 64;
      vb = a.vcache + h * 64;
    }
  } else {
    const int bk = kBeam ? b / a.rows_per_kv : b;
    kb = a.k + (long long)bk * a.Lk * a.ldk + h * 64;
    vb = a.v + (long long)bk * a.Lk * a.ldk + h * 64;
    ldk = a.ldk;
  }
  // offset of key / value row j from kb / vb
  auto koff = [&](int jj) -> long long {
    if (kBeam && srow) return ((long long)(jj < t ? srow[jj] : b) * a.tmax + jj) * HD;
    return (long long)jj * ldk;
  };
  float m = -INFINITY, l = 0.f;
  float2 acc = make_float2(0.f, 0.f);
  int j = 0;
  // four keys per iteration: 8 independent row loads in flight and four interleaved butterfly reductions (the one-key loop
  // below is a ~700-cycle dependent chain per key: at L = 13 the whole kernel was load-latency bound)
  for (; j + 4 <= Lk; j += 4) {
    float2 kf[4], vf[4];
    float s[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long o = koff(j + u);
      kf[u] = *reinterpret_cast<const float2*>(kb + o + 2 * lane);
      vf[u] = *reinterpret_cast<const float2*>(vb + o + 2 * lane);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) s[u] = q.x * kf[u].x + q.y * kf[u].y;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < 4; ++u) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
    }
    const float mn = fmaxf(fmaxf(m, fmaxf(s[0], s[1])), fmaxf(s[2], s[3]));
    const float r = __expf(m - mn);
    l *= r; acc.x *= r; acc.y *= r;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float p = __expf(s[u] - mn);
      l += p;
      acc.x += p * vf[u].x;
      acc.y += p * vf[u].y;
    }
    m = mn;
  }
  for (; j < Lk; ++j) {
    const long long o = koff(j);
    const float2 kf = *reinterpret_cast<const float2*>(kb + o + 2 * lane);
    const float s = warp_sum(q.x * kf.x + q.y * kf.y);
    const float mn = fmaxf(m, s);
    const float r = __expf(m - mn), p = __expf(s - mn);
    const float2 vf = *reinterpret_cast<const float2*>(vb + o + 2 * lane);
    l = l * r + p;
    acc.x = acc.x * r + p * vf.x;
    acc.y = acc.y * r + p * vf.y;
    m = mn;
  }
  const float inv = 1.f / l;
  __half* orow = a.out + ((long long)b * a.Lq + qi) * a.ldo;
  store_act(orow, h * 64 + 2 * lane, a.split, acc.x * inv);
  store_act(orow, h * 64 + 2 * lane + 1, a.split, acc.y * inv);
}

// ---------------------------------------------------------------------------------------- embeddings
// Encoder input: row (b, i) = (i < n_img ? image_feat[b][i] : E[prompt[i - n_img]]) + P[i + 2]
// (hf:models/florence2/modeling_florence2.py:742-761; learned positions with offset 2, hf:models/bart/
// modeling_bart.py:74-98).  Decoder input: row b = E[token[b]] + P[*step + 2].  Output fp32 (LayerNorm follows).
__global__ void encoder_embed_kernel(const float* __restrict__ img, int n_img, const float* __restrict__ E,
                                     const int* __restrict__ prompt, int n_prompt, const float* __restrict__ P, int B,
                                     int C, float* __restrict__ out) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const int L = n_img + n_prompt;
  const long long n = (long long)B * L * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % C);
    const int t = int((i / C) % L);
    const int b = int(i / ((long long)C * L));
    const float e = (t < n_img) ? img[((long long)b * n_img + t) * C + c] : E[(long long)prompt[t - n_img] * C + c];
    out[i] = e + P[(long long)(t + 2) * C + c];
  }
}

__global__ void decoder_embed_kernel(const float* __restrict__ E, const int* __restrict__ seq, int seq_ld,
                                     const int* __restrict__ step, const float* __restrict__ P, int B, int C,
                                     float* __restrict__ out) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const int t = *step;
  const long long n = (long long)B * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % C);
    const int b = int(i / C);
    out[i] = E[(long long)seq[b * seq_ld + t] * C + c] + P[(long long)(t + 2) * C + c];
  }
}

// Projector prep (hf:models/florence2/modeling_florence2.py:573-595): tokens = x + pos2d + temporal(0);
// rows: [mean over HW] ++ [HW tokens]; fp16 out [B][1+HW][C] feeding the 1024->768 projection GEMM.
__global__ void projector_prep_kernel(const float* __restrict__ x /*[B][HW][C]*/, const float* __restrict__ pos /*[HW][C]*/,
                                      int B, int HW, int C, __half* __restrict__ out, int split) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const long long n = (long long)B * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = int(i % C);
    const int b = int(i / C);
    float s = 0.f;
    for (int t = 0; t < HW; ++t) {
      const float v = x[((long long)b * HW + t) * C + c] + pos[(long long)t * C + c];
      s += v;
      store_act(out + ((long long)b * (HW + 1) + 1 + t) * (split ? 2 * C : C), c, split, v);
    }
    store_act(out + (long long)b * (HW + 1) * (split ? 2 * C : C), c, split, s / float(HW));
  }
}

// ---------------------------------------------------------------------------------------- greedy pick
// HF greedy step (hf:generation/utils.py:2727-2805) with the processors Florence-2 configures, in HF order:
// no_repeat_ngram (hf:generation/logits_process.py:1012-1079), forced BOS (:1552), forced EOS (:1597); then
// argmax (first maximum), pad for finished rows, EOS bookkeeping.  seq[b][0] = decoder_start; this kernel writes
// seq[b][*step + 1], *step + 1 <= max_len - 1.  One CTA per row.
struct PickArgs {
  const float* logits; long long ld; int V;
  int* seq; int seq_ld;
  int* finished;        // [B]
  const int* step;      // current decoder length - 1
  int ngram, forced_bos, forced_eos, eos, pad, max_len;   // max_len = total sequence length incl. start token
  float* dump;          // optional [B][V] processed scores of this step (parity checks)
  int* n_unfinished;    // device counter, decremented when a row finishes
};

// The ban list lives in dynamic shared memory, max_len ints: a pick at length cur_len <= max_len - 1 bans at most
// cur_len - ngram + 1 < max_len tokens (greedy decoding never repeats an n-gram, so a recurring (n-1)-gram prefix bans
// one more distinct token every time it recurs: long generations do reach hundreds of bans).
constexpr int kPickMaxLen = 8192;   // 32 KiB of bans

// No-repeat-n-gram ban scan (hf:generation/logits_process.py:1012-1079) of one row, shared by the greedy pick and the beam
// top-k: appends to banned[] every token that would complete an n-gram already present in seq[0..cur_len), one start
// position per thread (the list order does not matter: it is only tested for membership).  *nbanned_s must be 0 and
// visible to the whole CTA on entry; the caller synchronises before reading the list.
__device__ __forceinline__ void ngram_bans(const int* seq, int cur_len, int ngram, int max_len, int* banned, int* nbanned_s) {
  if (ngram > 0 && cur_len + 1 >= ngram) {
    const int pre = ngram - 1;
    for (int s = threadIdx.x; s + ngram <= cur_len; s += blockDim.x) {
      bool eq = true;
      for (int k = 0; k < pre; ++k) eq = eq && (seq[s + k] == seq[cur_len - pre + k]);
      if (eq) {
        const int i = atomicAdd(nbanned_s, 1);
        if (i < max_len) banned[i] = seq[s + pre];   // always true for cur_len <= max_len - 1
      }
    }
  }
}

__global__ void __launch_bounds__(1024) greedy_pick_kernel(PickArgs a) {
  pdl_wait();   // PDL: inputs come from the previous kernel in the stream
  const int b = blockIdx.x;
  const int t = *a.step;            // tokens so far = t + 1
  const int cur_len = t + 1;
  const float* lg = a.logits + (long long)b * a.ld;
  int* seq = a.seq + (long long)b * a.seq_ld;
  __shared__ float bv[32];
  __shared__ int bi[32];
  extern __shared__ int banned[];   // [max_len]
  __shared__ int nbanned_s;
  if (threadIdx.x == 0) nbanned_s = 0;
  __syncthreads();
  ngram_bans(seq, cur_len, a.ngram, a.max_len, banned, &nbanned_s);
  __syncthreads();
  const int nbanned = min(nbanned_s, a.max_len);
  int force = -1;
  if (cur_len == 1 && a.forced_bos >= 0) force = a.forced_bos;
  if (cur_len == a.max_len - 1 && a.forced_eos >= 0) force = a.forced_eos;
  float best = -INFINITY;
  int besti = 0x7fffffff;
  if (a.dump || force < 0) {
    const bool vec = !a.dump && force < 0 && (a.ld % 2 == 0) && ((reinterpret_cast<uintptr_t>(lg) & 7) == 0);
    if (vec) {
      // plain scan; the ban list is only consulted when a value would become the running maximum
      const float2* lp = reinterpret_cast<const float2*>(lg);
      const int V2 = a.V >> 1;
      // four strided loads in flight per thread before the compares (one load per iteration left every thread waiting on an
      // L2 round trip 25 times per row); the compares stay in ascending index order
      for (int v0 = threadIdx.x; v0 < V2; v0 += 4 * blockDim.x) {
        float2 t4[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int v2 = v0 + u * blockDim.x;
          t4[u] = (v2 < V2) ? lp[v2] : make_float2(-INFINITY, -INFINITY);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int v2 = v0 + u * blockDim.x;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float sv = e ? t4[u].y : t4[u].x;
            const int v = 2 * v2 + e;
            if (sv > best) {   // ascending v within a thread: ties keep the earlier index
              bool ban = false;
              for (int k = 0; k < nbanned; ++k) ban = ban || (banned[k] == v);
              if (!ban) { best = sv; besti = v; }
            }
          }
        }
      }
      if ((a.V & 1) && threadIdx.x == 0) {
        const int v = a.V - 1;
        const float sv = lg[v];
        bool ban = false;
        for (int k = 0; k < nbanned; ++k) ban = ban || (banned[k] == v);
        if (!ban && sv > best) { best = sv; besti = v; }
      }
    } else {
      for (int v = threadIdx.x; v < a.V; v += blockDim.x) {
        float sv = lg[v];
        for (int k = 0; k < nbanned; ++k) if (banned[k] == v) sv = -INFINITY;
        if (force >= 0) sv = (v == force) ? 0.f : -INFINITY;
        if (a.dump) a.dump[(long long)b * a.V + v] = sv;
        if (sv > best || (sv == best && v < besti)) { best = sv; besti = v; }
      }
    }
  } else if (threadIdx.x == 0) {
    best = 0.f;          // forced token: every other score is -inf (hf:generation/logits_process.py:1552,1597)
    besti = force;
  }
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ov > best || (ov == best && oi < besti)) { best = ov; besti = oi; }
  }
  if ((threadIdx.x & 31) == 0) { bv[threadIdx.x >> 5] = best; bi[threadIdx.x >> 5] = besti; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (bv[w] > best || (bv[w] == best && bi[w] < besti)) { best = bv[w]; besti = bi[w]; }
    int tok = besti;
    if (a.finished[b]) tok = a.pad;
    seq[cur_len] = tok;
    if (!a.finished[b] && tok == a.eos) {
      a.finished[b] = 1;
      if (a.n_unfinished) atomicSub(a.n_unfinished, 1);
    }
  }
}

__global__ void step_advance_kernel(int* step) {
  pdl_wait();
  *step += 1;
}

// ---------------------------------------------------------------------------------------- beam search
// HF beam search (hf:generation/utils.py:3076-3386, helpers :2876-3072) for decoder rows r = crop * nb + beam.  Tie rule
// of every selection: higher score first, on equal scores the lower index (flat index beam * V + token in the top-k, position
// in the list for the later selections).  See include/b200parse.h for why the ties torch.topk may order differently never
// reach the output.
constexpr int kBeamMax = 16;
constexpr int kBeamSeqInts = 16384;   // staged seq + src rows of one crop: nb * max_len ints each (64 KiB)

__device__ __forceinline__ bool beam_before(float v, int i, float w, int j) { return v > w || (v == w && i < j); }

struct BeamTopkArgs {
  const float* logits; long long ld; int V; int nb;
  const int* seq; int seq_ld; const int* step;
  int ngram, forced_bos, forced_eos, max_len;
  const float* bscore;      // [B] running beam scores
  const int* done;          // [B / nb] crops whose hypotheses are final (skipped); may be null
  float* cand_score;        // [B][2 nb] best continuations of the row, best first
  int* cand_idx;            // [B][2 nb] flat index beam * V + token
};

// One CTA per row: log_softmax in fp32, the processors on the log-probs (n-gram bans -> -inf; a forced step is -inf except the
// forced token's 0, without reading the logits), + the row's running score, best 2 nb.  Each thread keeps its best M in
// registers (M >= 2 nb, a power of two); the CTA then pops the best head 2 nb times.
template <int M>
__global__ void __launch_bounds__(256) beam_topk_kernel(BeamTopkArgs a) {
  pdl_wait();
  const int r = blockIdx.x, beam = r % a.nb, need = 2 * a.nb;
  if (a.done && a.done[r / a.nb]) return;
  const int t = *a.step, cur_len = t + 1;
  const float* lg = a.logits + (long long)r * a.ld;
  const int* seq = a.seq + (long long)r * a.seq_ld;
  const float bs = a.bscore[r];
  const int fbase = beam * a.V;
  float* co = a.cand_score + (long long)r * need;
  int* ci = a.cand_idx + (long long)r * need;
  int force = -1;
  if (cur_len == 1 && a.forced_bos >= 0) force = a.forced_bos;
  if (cur_len == a.max_len - 1 && a.forced_eos >= 0) force = a.forced_eos;
  if (force >= 0) {
    // forced token first (0 + beam score), then -inf for the lowest other token ids (hf:generation/logits_process.py:1552,1597)
    for (int j = threadIdx.x; j < need; j += blockDim.x) {
      const int tok = j == 0 ? force : j - 1 + (j - 1 >= force ? 1 : 0);
      co[j] = j == 0 ? 0.f + bs : -INFINITY;
      ci[j] = fbase + tok;
    }
    return;
  }
  extern __shared__ int banned[];   // [max_len]
  __shared__ int nbanned_s;
  __shared__ float red_m[8], red_s[8];
  __shared__ float win_v[2][8];
  __shared__ int win_i[2][8];
  if (threadIdx.x == 0) nbanned_s = 0;
  __syncthreads();
  ngram_bans(seq, cur_len, a.ngram, a.max_len, banned, &nbanned_s);
  // log-sum-exp of the raw logits (online max / sum per thread, then across the CTA)
  float m = -INFINITY, s = 0.f;
  for (int v = threadIdx.x; v < a.V; v += blockDim.x) {
    const float x = lg[v];
    if (x > m) { s = s * expf(m - x) + 1.f; m = x; }
    else if (x > -INFINITY) s += expf(x - m);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int o = 16; o; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    const float mn = fmaxf(m, om);
    s = (m > -INFINITY ? s * expf(m - mn) : 0.f) + (om > -INFINITY ? os * expf(om - mn) : 0.f);
    m = mn;
  }
  if (lane == 0) { red_m[warp] = m; red_s[warp] = s; }
  __syncthreads();   // also publishes the ban list
  float mx = -INFINITY;
  for (int w = 0; w < nwarp; ++w) mx = fmaxf(mx, red_m[w]);
  float sum = 0.f;
  for (int w = 0; w < nwarp; ++w) if (red_m[w] > -INFINITY) sum += red_s[w] * expf(red_m[w] - mx);
  const float lse = logf(sum);
  const int nbanned = min(nbanned_s, a.max_len);
  // per-thread best M of (log_softmax + bans) + beam score, ascending token order within the thread
  float tv[M];
  int ti[M];
#pragma unroll
  for (int k = 0; k < M; ++k) { tv[k] = -INFINITY; ti[k] = 0x7fffffff; }
  for (int v = threadIdx.x; v < a.V; v += blockDim.x) {
    float sv = ((lg[v] - mx) - lse) + bs;
    const int f = fbase + v;
    if (!beam_before(sv, f, tv[M - 1], ti[M - 1])) continue;
    bool ban = false;
    for (int k = 0; k < nbanned; ++k) ban = ban || (banned[k] == v);
    if (ban) {
      sv = -INFINITY;
      if (!beam_before(sv, f, tv[M - 1], ti[M - 1])) continue;
    }
    bool placed = false;
#pragma unroll
    for (int k = M - 1; k > 0; --k) {
      if (!placed) {
        if (beam_before(sv, f, tv[k - 1], ti[k - 1])) { tv[k] = tv[k - 1]; ti[k] = ti[k - 1]; }
        else { tv[k] = sv; ti[k] = f; placed = true; }
      }
    }
    if (!placed) { tv[0] = sv; ti[0] = f; }
  }
  // pop the CTA's best head `need` times (flat indices are unique, so exactly one thread owns the winner)
  for (int j = 0; j < need; ++j) {
    float bv = tv[0];
    int bi = ti[0];
    for (int o = 16; o; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (beam_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { win_v[j & 1][warp] = bv; win_i[j & 1][warp] = bi; }
    __syncthreads();
    bv = win_v[j & 1][0]; bi = win_i[j & 1][0];
    for (int w = 1; w < nwarp; ++w)
      if (beam_before(win_v[j & 1][w], win_i[j & 1][w], bv, bi)) { bv = win_v[j & 1][w]; bi = win_i[j & 1][w]; }
    if (ti[0] == bi) {
#pragma unroll
      for (int k = 0; k < M - 1; ++k) { tv[k] = tv[k + 1]; ti[k] = ti[k + 1]; }
      tv[M - 1] = -INFINITY; ti[M - 1] = 0x7fffffff;
    }
    if (threadIdx.x == 0) { co[j] = bv; ci[j] = bi; }
  }
}

struct BeamUpdateArgs {
  const float* cand_score; const int* cand_idx;   // [K * nb][2 nb], b2p_beam_topk
  int V, nb;
  int* seq; int seq_ld;                           // running sequences [K * nb][seq_ld]
  int* src; int tmax;                             // cache ancestor table [K * nb][tmax]
  const int* step;
  int eos, pad, max_len, early_stopping, lp_positive;
  const float* lp_pow;                            // [max_len + 1]: float(L ** length_penalty)
  float* bscore; int* parent;                     // [K * nb]; parent: beam index of each new running row (may be null)
  int* hyp_seq; float* hyp_score; int* hyp_len; int* hyp_fin;   // finished hypotheses [K * nb] (hyp_seq pitch seq_ld)
  int* heur; int* done; int* n_open;              // [K], [K], counter of crops not done
};

// One CTA per crop: HF steps c-g.  Thread 0 makes the (small, serial) selections; the CTA stages the crop's seq / src rows in
// shared memory and writes the parent-gathered rows back in place.
__global__ void __launch_bounds__(256) beam_update_kernel(BeamUpdateArgs a) {
  pdl_wait();
  const int k = blockIdx.x, nb = a.nb, need = 2 * nb, r0 = k * nb;
  if (a.done[k]) return;   // hypotheses are final (see include/b200parse.h): nothing of this crop changes any more
  const int t = *a.step, cur_len = t + 1;   // the new token goes to position cur_len
  extern __shared__ int bsm[];
  int* sseq = bsm;                          // [nb][cur_len]
  int* ssrc = bsm + nb * a.max_len;         // [nb][t]
  __shared__ float top_s[2 * kBeamMax];
  __shared__ int top_f[2 * kBeamMax];
  __shared__ int run_from[kBeamMax];        // new running beam j <- top position
  __shared__ float run_s[kBeamMax];
  __shared__ int hyp_from[kBeamMax];        // new hypothesis slot j <- merged index (< nb: old slot, else nb + top position)
  for (int i = threadIdx.x; i < nb * cur_len; i += blockDim.x) {
    const int b = i / cur_len, j = i - b * cur_len;
    sseq[i] = a.seq[(long long)(r0 + b) * a.seq_ld + j];
  }
  for (int i = threadIdx.x; i < nb * t; i += blockDim.x) {
    const int b = i / t, j = i - b * t;
    ssrc[i] = a.src[(long long)(r0 + b) * a.tmax + j];
  }
  if (threadIdx.x == 0) {
    const float NEG = -1.0e9f;
    // c. the crop's best 2 nb: merge of the rows' sorted lists
    int head[kBeamMax];
    for (int b = 0; b < nb; ++b) head[b] = 0;
    for (int j = 0; j < need; ++j) {
      int bb = -1, bi = 0;
      float bv = 0.f;
      for (int b = 0; b < nb; ++b) {
        if (head[b] >= need) continue;
        const float v = a.cand_score[(long long)(r0 + b) * need + head[b]];
        const int f = a.cand_idx[(long long)(r0 + b) * need + head[b]];
        if (bb < 0 || beam_before(v, f, bv, bi)) { bb = b; bv = v; bi = f; }
      }
      top_s[j] = bv; top_f[j] = bi; ++head[bb];
    }
    // d. stopping criteria per candidate: EOS, or the sequence reaches max_len
    bool hit[2 * kBeamMax], all_hit = true;
    for (int j = 0; j < need; ++j) {
      hit[j] = (top_f[j] % a.V) == a.eos || cur_len + 1 >= a.max_len;
      all_hit = all_hit && hit[j];
    }
    // e. running beams: best nb of score + hit * -1e9 (_get_running_beams_for_next_iteration)
    float rs[2 * kBeamMax];
    for (int j = 0; j < need; ++j) rs[j] = __fadd_rn(top_s[j], hit[j] ? NEG : -0.f);
    unsigned used = 0;
    for (int j = 0; j < nb; ++j) {
      int bj = -1;
      for (int i = 0; i < need; ++i)
        if (!((used >> i) & 1u) && (bj < 0 || rs[i] > rs[bj])) bj = i;
      used |= 1u << bj;
      run_from[j] = bj; run_s[j] = rs[bj];
    }
    // f. finished hypotheses (_update_finished_beams), the same fp32 operations in the same order
    const int h0 = r0;
    bool all_fin = true;
    for (int s = 0; s < nb; ++s) all_fin = all_fin && a.hyp_fin[h0 + s];
    const bool heur = a.heur[k] != 0;
    const float lpow = a.lp_pow[cur_len];
    float c[2 * kBeamMax];
    bool did[2 * kBeamMax];
    for (int j = 0; j < need; ++j) {
      float v = __fdiv_rn(top_s[j], lpow);
      v = __fadd_rn(v, (all_fin && a.early_stopping == 1) ? NEG : -0.f);
      v = __fadd_rn(v, heur ? -0.f : NEG);
      did[j] = hit[j] && j < nb;
      v = __fadd_rn(v, did[j] ? -0.f : NEG);
      c[j] = v;
    }
    float old_s[kBeamMax], new_s[kBeamMax];
    int old_f[kBeamMax], old_l[kBeamMax], new_f[kBeamMax];
    for (int s = 0; s < nb; ++s) { old_s[s] = a.hyp_score[h0 + s]; old_f[s] = a.hyp_fin[h0 + s]; old_l[s] = a.hyp_len[h0 + s]; }
    unsigned long long used2 = 0;
    for (int j = 0; j < nb; ++j) {
      int bj = -1;
      float bv = 0.f;
      for (int i = 0; i < nb + need; ++i) {
        const float v = i < nb ? old_s[i] : c[i - nb];
        if (!((used2 >> i) & 1ull) && (bj < 0 || v > bv)) { bj = i; bv = v; }
      }
      used2 |= 1ull << bj;
      hyp_from[j] = bj;
      new_s[j] = bv;
      new_f[j] = bj < nb ? old_f[bj] : (int)did[bj - nb];
      a.hyp_score[h0 + j] = bv;
      a.hyp_fin[h0 + j] = new_f[j];
      a.hyp_len[h0 + j] = bj < nb ? old_l[bj] : cur_len;
    }
    // g. early-stop heuristic at the next length (_check_early_stop_heuristic) and the crop's stopping condition
    //    (_beam_search_has_unfinished_sequences restricted to this crop)
    const int best_len = (a.early_stopping == 2 && a.lp_positive) ? a.max_len - 1 : cur_len;
    const float best = __fdiv_rn(run_s[0], a.lp_pow[best_len]);
    float mn = new_s[0];
    for (int s = 1; s < nb; ++s) mn = fminf(mn, new_s[s]);
    bool improvable = false, all_fin_new = true;
    for (int s = 0; s < nb; ++s) {
      improvable = improvable || best > (new_f[s] ? mn : NEG);
      all_fin_new = all_fin_new && new_f[s];
    }
    const bool heur_new = heur && improvable;
    a.heur[k] = heur_new;
    const bool open = heur_new && !(all_fin_new && a.early_stopping == 1) && !all_hit;
    if (!open) {
      a.done[k] = 1;
      if (a.n_open) atomicSub(a.n_open, 1);
    }
  }
  __syncthreads();
  // running rows: parent-gathered prefix + the new token; cache ancestors; scores
  for (int i = threadIdx.x; i < nb * (cur_len + 1); i += blockDim.x) {
    const int b = i / (cur_len + 1), j = i - b * (cur_len + 1);
    const int f = top_f[run_from[b]], p = f / a.V;
    a.seq[(long long)(r0 + b) * a.seq_ld + j] = j < cur_len ? sseq[p * cur_len + j] : f - p * a.V;
  }
  for (int i = threadIdx.x; i < nb * (t + 1); i += blockDim.x) {
    const int b = i / (t + 1), j = i - b * (t + 1);
    const int p = top_f[run_from[b]] / a.V;
    a.src[(long long)(r0 + b) * a.tmax + j] = j < t ? ssrc[p * t + j] : r0 + p;
  }
  for (int b = threadIdx.x; b < nb; b += blockDim.x) {
    a.bscore[r0 + b] = run_s[b];
    if (a.parent) a.parent[r0 + b] = top_f[run_from[b]] / a.V;
  }
  // hypothesis rows, in place: the kept old slots are a prefix 0..m-1 of the old list and move to slots j >= their old
  // index, so filling the slots from the last to the first never overwrites a row that is still to be read
  for (int j = nb - 1; j >= 0; --j) {
    const int from = hyp_from[j];
    int* dst = a.hyp_seq + (long long)(r0 + j) * a.seq_ld;
    if (from < nb) {
      if (from != j) {
        const int* srow = a.hyp_seq + (long long)(r0 + from) * a.seq_ld;
        for (int i = threadIdx.x; i < a.seq_ld; i += blockDim.x) dst[i] = srow[i];
      }
    } else {
      const int f = top_f[from - nb], p = f / a.V;
      for (int i = threadIdx.x; i < a.seq_ld; i += blockDim.x)
        dst[i] = i < cur_len ? sseq[p * cur_len + i] : (i == cur_len ? f - p * a.V : a.pad);
    }
    __syncthreads();
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

int b2p_layernorm(const float* x, long long ldx, const float* gamma, const float* beta, float eps, int T, int C,
                  void* out16, long long ld16, float* out32, long long ld32, int split, cudaStream_t st) {
  if (T <= 0) return 0;
  if (C % 4 || C > 1024 || (ldx % 4) || (ld32 % 4) || (ld16 % 4)) return set_error("layernorm: C, ld must be multiples of 4, C <= 1024");
  const int wpb = 8;
  launch_pdl(layernorm_kernel, dim3((T + wpb - 1) / wpb), dim3(wpb * 32), 0, st, x, ldx, gamma, beta, eps, T, C, (__half*)out16, ld16, out32, ld32, split ? C : 0);
  B2P_CHECK_LAUNCH();
  return 0;
}

// out = LayerNorm(A * B^T + bias + residual): a park-only GEMM (raw partial accumulators of every (tile, k slice) in the
// split-K workspace) followed by splitk_ln_kernel.  A, B as b2p_gemm (flags & 8: fp16x3 operands); residual fp32 [M][ldr];
// out16: fp16 (flags & 4: [hi | lo], ld16 >= 2N) and / or out32: fp32.  Replaces b2p_gemm(+residual) + b2p_layernorm.
int b2p_gemm_ln(const void* A, long long lda, const void* B, int M, int N, int K, const float* bias, const float* residual,
                long long ldr, const float* gamma, const float* beta, float eps, void* out16, long long ld16, float* out32,
                long long ld32, int flags, cudaStream_t st) {
  if (M <= 0) return 0;
  if (N % 16 || N > 1024 || (ldr % 4) || (ld32 % 4) || (ld16 % 4)) return set_error("gemm_ln: N must be a multiple of 16 and <= 1024, ld multiples of 4");
  ParkInfo pk{};
  ConvGemm d{};
  d.mode = 0; d.bf16 = 0; d.A = A; d.lda = lda; d.B = B; d.M = M; d.N = N; d.K = K;
  d.out = nullptr; d.ldc = N; d.out_f32 = 1; d.bias = nullptr; d.res = nullptr; d.ldr = 0; d.act = 0;
  d.bn_max = (flags >> 8) & 0x1ff; d.x3 = (flags >> 3) & 1;
  d.park = 1; d.park_info = &pk;
  if (int e = gemm_launch(d, st)) return e;
  const int wpb = 8;
  launch_pdl(splitk_ln_kernel, dim3((M + wpb - 1) / wpb), dim3(wpb * 32), 0, st, pk, M, N, bias, residual, ldr, gamma, beta, eps,
             (__half*)out16, ld16, out32, ld32, (flags & 4) ? N : 0);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_dwconv_ln(const float* x, int B, int H, int W, int C, const float* w9c, const float* bias, float* y,
                  const float* gamma, const float* beta, float eps, void* out16, int split, cudaStream_t st) {
  if (C % 4 || C > 1024) return set_error("dwconv_ln: C must be a multiple of 4 and <= 1024");
  const long long T = (long long)B * H * W;
  if (split & 4) {   // strip kernel (florence_simt.cu); shapes it does not cover fall through
    const int r = dwconv_ln_v3_launch(x, B, H, W, C, w9c, bias, y, gamma, beta, eps, out16, split & 1, st);
    if (r <= 0) return r;
  }
  const size_t tile_bytes = size_t(H) * W * C * sizeof(float);
  if ((split & 2) && tile_bytes <= 200 * 1024 && B > 0) {   // opt-in tiled variant (see dwconv_ln_tile_kernel)
    static std::atomic<bool> attr{false};
    if (!attr) {
      if (cudaFuncSetAttribute(dwconv_ln_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess)
        return set_error("dwconv_ln: cudaFuncSetAttribute failed");
      attr = true;
    }
    const int threads = (H * W >= 16) ? 512 : 256;
    launch_pdl(dwconv_ln_tile_kernel, dim3(B), dim3(threads), tile_bytes, st, x, H, W, C, w9c, bias, y, gamma, beta, eps, (__half*)out16,
               (split & 1) ? C : 0);
    B2P_CHECK_LAUNCH();
    return 0;
  }
  const int wpb = 8;
  launch_pdl(dwconv_ln_kernel, dim3(int((T + wpb - 1) / wpb)), dim3(wpb * 32), 0, st, x, B, H, W, C, w9c, bias, y, gamma, beta, eps, (__half*)out16, (split & 1) ? C : 0);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_dwconv3x3_res(const float* x, int B, int H, int W, int C, const float* w9c, const float* bias, float* y,
                      cudaStream_t st) {
  launch_pdl(dwconv3x3_res_kernel, dim3(grid_for((long long)B * H * W * C, 256)), dim3(256), 0, st, x, B, H, W, C, w9c, bias, y);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_window_attn(const float* qkv, const float* qkv_bias, int B, int H, int W, int C, int heads, int win, void* out,
                    int split, cudaStream_t st) {
  if (C / heads != 32) return set_error("window_attn: head_dim must be 32");
  if (split & 4) {   // one-window maps: CTA per (image, head group), florence_simt.cu
    if (int e = bind_device()) return e;
    const int r = window_attn_crop_launch(qkv, qkv_bias, B, H, W, C, heads, win, out, split & 1, st);
    if (r <= 0) return r;
  }
  const int nw = ((W + win - 1) / win) * ((H + win - 1) / win);
  // K/V staging sized by the REAL tokens of a window: the 4x4 / 2x2 maps of the 64x64-crop mode need 4 KB / 1 KB, not the
  // 36.9 KB of a full 12x12 window (which capped those launches at 6 one-warp CTAs per SM)
  const int kv_cap = (W < win ? W : win) * (H < win ? H : win);
  const size_t smem = size_t(2) * kv_cap * 32 * sizeof(float);
  if (int e = bind_device()) return e;
  static std::atomic<bool> attr{false};
  if (!attr) {
    cudaFuncSetAttribute(window_attn_kernel<32, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    attr = true;
  }
  if (smem > 64 * 1024) return set_error("window_attn: window too large");
  // (two queries per thread, QB = 2, is slower on the 16x16 map -- 168 registers leave 12 warps per SM;
  //  the one-window maps do use QB = 2, in window_attn_crop_kernel)
  // one thread per query of the window: small maps (4x4, 8x8 in the 64x64-crop mode) get small CTAs so more of them fit per SM
  const int nq = kv_cap;
  const int threads = nq >= 160 ? 160 : ((nq + 31) / 32) * 32;
  launch_pdl(window_attn_kernel<32, 1>, dim3(B * nw * heads), dim3(threads), smem, st, qkv, qkv_bias, B, H, W, C, heads, win, (__half*)out, (split & 1) ? C : 0, kv_cap);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_channel_attn(const float* qkv, int B, int N, int C, int groups, void* out, int split, cudaStream_t st) {
  if (C / groups != 32) return set_error("channel_attn: channels per group must be 32");
  if (split & 4) {   // register-tiled kernel, florence_simt.cu
    const int r = channel_attn_v3_launch(qkv, B, N, C, groups, out, split & 1, st);
    if (r <= 0) return r;
  }
  if ((split & 2) && N <= 16 && B > 0) {   // opt-in small-N variant (see channel_attn_small_kernel)
    launch_pdl(channel_attn_small_kernel, dim3((B * groups + 3) / 4), dim3(128), 0, st, qkv, B, N, C, groups, (__half*)out, (split & 1) ? C : 0);
    B2P_CHECK_LAUNCH();
    return 0;
  }
  launch_pdl(channel_attn_kernel, dim3(B * groups), dim3(256), 0, st, qkv, N, C, groups, (__half*)out, (split & 1) ? C : 0);
  B2P_CHECK_LAUNCH();
  return 0;
}

// Encoder self-attention / decoder cross-attention: explicit K, V.
int b2p_mha(const float* q, long long ldq, const float* k, const float* v, long long ldk, int B, int Lq, int Lk, int heads,
            void* out, long long ldo, int split, cudaStream_t st) {
  if (split & 4) {   // short sequences: warp per (batch, head) with K / V in registers, florence_simt.cu
    const int r = mha_short_launch(q, ldq, k, v, ldk, B, Lq, Lk, heads, out, ldo, split & 1, st);
    if (r <= 0) return r;
  }
  MhaArgs a{};
  a.q = q; a.ldq = ldq; a.k = k; a.v = v; a.ldk = ldk;
  a.B = B; a.Lq = Lq; a.Lk = Lk; a.heads = heads; a.out = (__half*)out; a.ldo = ldo; a.split = (split & 1) ? heads * 64 : 0;
  const int total = B * heads * Lq;
  // (a thread-per-query variant is slower here: its per-thread 256-B rows are uncoalesced)
  launch_pdl(mha_kernel<false>, dim3((total + 7) / 8), dim3(256), 0, st, a);
  B2P_CHECK_LAUNCH();
  return 0;
}

// Decoder self-attention step with KV-cache append at position *step.
int b2p_mha_cached(const float* q, long long ldq, const float* knew, const float* vnew, long long ldnew, float* kcache,
                   float* vcache, int tmax, const int* step, int B, int heads, void* out, long long ldo, int split,
                   cudaStream_t st) {
  MhaArgs a{};
  a.q = q; a.ldq = ldq; a.knew = knew; a.vnew = vnew; a.ldnew = ldnew;
  a.kcache = kcache; a.vcache = vcache; a.tmax = tmax; a.step = step;
  a.B = B; a.Lq = 1; a.Lk = 0; a.heads = heads; a.out = (__half*)out; a.ldo = ldo; a.split = split ? heads * 64 : 0;
  const int total = B * heads;
  launch_pdl(mha_kernel<false>, dim3((total + 7) / 8), dim3(256), 0, st, a);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_encoder_embed(const float* img, int n_img, const float* E, const int* prompt, int n_prompt, const float* P,
                      int B, int C, float* out, cudaStream_t st) {
  launch_pdl(encoder_embed_kernel, dim3(grid_for((long long)B * (n_img + n_prompt) * C, 256)), dim3(256), 0, st, img, n_img, E, prompt,
                                                                                            n_prompt, P, B, C, out);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_decoder_embed(const float* E, const int* seq, int seq_ld, const int* step, const float* P, int B, int C,
                      float* out, cudaStream_t st) {
  launch_pdl(decoder_embed_kernel, dim3(grid_for((long long)B * C, 256)), dim3(256), 0, st, E, seq, seq_ld, step, P, B, C, out);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_projector_prep(const float* x, const float* pos, int B, int HW, int C, void* out, int split, cudaStream_t st) {
  launch_pdl(projector_prep_kernel, dim3(grid_for((long long)B * C, 256)), dim3(256), 0, st, x, pos, B, HW, C, (__half*)out, split ? C : 0);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_greedy_pick(const float* logits, long long ld, int V, int B, int* seq, int seq_ld, int* finished,
                    const int* step, int ngram, int forced_bos, int forced_eos, int eos, int pad, int max_len,
                    float* dump, int* n_unfinished, cudaStream_t st) {
  if (B < 0) return set_error("greedy_pick: B must be >= 0");
  if (B == 0) return 0;
  if (V < 1 || ld < V) return set_error("greedy_pick: need 1 <= V <= ld");
  if (ngram < 0) return set_error("greedy_pick: ngram must be >= 0 (0 = no n-gram ban)");
  if (max_len < 2 || max_len > kPickMaxLen) return set_error("greedy_pick: max_len must be in [2, 8192]");
  if (seq_ld < max_len) return set_error("greedy_pick: seq_ld must be >= max_len");
  if (forced_bos >= V || forced_eos >= V) return set_error("greedy_pick: forced token ids must be < V");
  PickArgs a{};
  a.logits = logits; a.ld = ld; a.V = V; a.seq = seq; a.seq_ld = seq_ld; a.finished = finished; a.step = step;
  a.ngram = ngram; a.forced_bos = forced_bos; a.forced_eos = forced_eos; a.eos = eos; a.pad = pad; a.max_len = max_len;
  a.dump = dump; a.n_unfinished = n_unfinished;
  launch_pdl(greedy_pick_kernel, dim3(B), dim3(1024), size_t(max_len) * sizeof(int), st, a);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_step_advance(int* step, cudaStream_t st) {
  launch_pdl(step_advance_kernel, dim3(1), dim3(1), 0, st, step);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_mha_cached_beam(const float* q, long long ldq, const float* knew, const float* vnew, long long ldnew, float* kcache,
                        float* vcache, int tmax, const int* step, const int* src, int B, int heads, void* out, long long ldo,
                        int split, cudaStream_t st) {
  if (B < 0) return set_error("mha_cached_beam: B must be >= 0");
  if (B == 0) return 0;
  if (!src || tmax < 1) return set_error("mha_cached_beam: needs the ancestor table src [B][tmax]");
  MhaArgs a{};
  a.q = q; a.ldq = ldq; a.knew = knew; a.vnew = vnew; a.ldnew = ldnew;
  a.kcache = kcache; a.vcache = vcache; a.tmax = tmax; a.step = step; a.src = src;
  a.B = B; a.Lq = 1; a.Lk = 0; a.heads = heads; a.out = (__half*)out; a.ldo = ldo; a.split = split ? heads * 64 : 0;
  launch_pdl(mha_kernel<true>, dim3((B * heads + 7) / 8), dim3(256), 0, st, a);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_mha_grouped(const float* q, long long ldq, const float* k, const float* v, long long ldk, int B, int Lq, int Lk,
                    int heads, int rows_per_kv, void* out, long long ldo, int split, cudaStream_t st) {
  if (B < 0) return set_error("mha_grouped: B must be >= 0");
  if (B == 0) return 0;
  if (rows_per_kv < 1) return set_error("mha_grouped: rows_per_kv must be >= 1");
  MhaArgs a{};
  a.q = q; a.ldq = ldq; a.k = k; a.v = v; a.ldk = ldk; a.rows_per_kv = rows_per_kv;
  a.B = B; a.Lq = Lq; a.Lk = Lk; a.heads = heads; a.out = (__half*)out; a.ldo = ldo; a.split = (split & 1) ? heads * 64 : 0;
  launch_pdl(mha_kernel<true>, dim3((B * heads * Lq + 7) / 8), dim3(256), 0, st, a);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_beam_topk(const float* logits, long long ld, int V, int B, int nb, const int* seq, int seq_ld, const int* step,
                  int ngram, int forced_bos, int forced_eos, int max_len, const float* bscore, const int* done,
                  float* cand_score, int* cand_idx, cudaStream_t st) {
  if (B < 0) return set_error("beam_topk: B must be >= 0");
  if (nb < 1 || nb > kBeamMax) return set_error("beam_topk: num_beams must be in [1, 16]");
  if (B % nb) return set_error("beam_topk: B must be a multiple of num_beams");
  if (V < 2 * nb || ld < V) return set_error("beam_topk: need 2 * num_beams <= V <= ld");
  if ((long long)V * nb > 0x7fffffffLL) return set_error("beam_topk: num_beams * V must fit in int");
  if (ngram < 0) return set_error("beam_topk: ngram must be >= 0 (0 = no n-gram ban)");
  if (max_len < 2 || max_len > kPickMaxLen) return set_error("beam_topk: max_len must be in [2, 8192]");
  if (seq_ld < max_len) return set_error("beam_topk: seq_ld must be >= max_len");
  if (forced_bos >= V || forced_eos >= V) return set_error("beam_topk: forced token ids must be < V");
  if (B == 0) return 0;
  BeamTopkArgs a{};
  a.logits = logits; a.ld = ld; a.V = V; a.nb = nb; a.seq = seq; a.seq_ld = seq_ld; a.step = step;
  a.ngram = ngram; a.forced_bos = forced_bos; a.forced_eos = forced_eos; a.max_len = max_len;
  a.bscore = bscore; a.done = done; a.cand_score = cand_score; a.cand_idx = cand_idx;
  const size_t smem = size_t(max_len) * sizeof(int);
  if (nb <= 2) launch_pdl(beam_topk_kernel<4>, dim3(B), dim3(256), smem, st, a);
  else if (nb <= 4) launch_pdl(beam_topk_kernel<8>, dim3(B), dim3(256), smem, st, a);
  else if (nb <= 8) launch_pdl(beam_topk_kernel<16>, dim3(B), dim3(256), smem, st, a);
  else launch_pdl(beam_topk_kernel<32>, dim3(B), dim3(256), smem, st, a);
  B2P_CHECK_LAUNCH();
  return 0;
}

int b2p_beam_update(const float* cand_score, const int* cand_idx, int V, int K, int nb, int* seq, int seq_ld, int* src,
                    int tmax, const int* step, int eos, int pad, int max_len, int early_stopping, float length_penalty,
                    const float* lp_pow, float* bscore, int* parent, int* hyp_seq, float* hyp_score, int* hyp_len,
                    int* hyp_fin, int* heur, int* done, int* n_open, cudaStream_t st) {
  if (K < 0) return set_error("beam_update: K must be >= 0");
  if (nb < 1 || nb > kBeamMax) return set_error("beam_update: num_beams must be in [1, 16]");
  if (V < 2 * nb) return set_error("beam_update: need 2 * num_beams <= V");
  if ((long long)V * nb > 0x7fffffffLL) return set_error("beam_update: num_beams * V must fit in int");
  if (max_len < 2 || max_len > kPickMaxLen) return set_error("beam_update: max_len must be in [2, 8192]");
  if (seq_ld < max_len) return set_error("beam_update: seq_ld must be >= max_len");
  if (tmax < max_len - 1) return set_error("beam_update: tmax must be >= max_len - 1");
  if ((long long)nb * max_len > kBeamSeqInts) return set_error("beam_update: num_beams * max_len must be <= 16384");
  if (early_stopping < 0 || early_stopping > 2) return set_error("beam_update: early_stopping must be 0 (False), 1 (True) or 2 (\"never\")");
  if (!lp_pow) return set_error("beam_update: needs the length-penalty table lp_pow [max_len + 1]");
  if (K == 0) return 0;
  const size_t smem = size_t(2) * nb * max_len * sizeof(int);
  static std::atomic<bool> attr{false};
  if (!attr) {
    if (int e = bind_device()) return e;
    if (cudaFuncSetAttribute(beam_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(2 * kBeamSeqInts * sizeof(int))) != cudaSuccess)
      return set_error("beam_update: cudaFuncSetAttribute failed");
    attr = true;
  }
  BeamUpdateArgs a{};
  a.cand_score = cand_score; a.cand_idx = cand_idx; a.V = V; a.nb = nb; a.seq = seq; a.seq_ld = seq_ld; a.src = src; a.tmax = tmax;
  a.step = step; a.eos = eos; a.pad = pad; a.max_len = max_len; a.early_stopping = early_stopping; a.lp_positive = length_penalty > 0.f;
  a.lp_pow = lp_pow; a.bscore = bscore; a.parent = parent; a.hyp_seq = hyp_seq; a.hyp_score = hyp_score; a.hyp_len = hyp_len;
  a.hyp_fin = hyp_fin; a.heur = heur; a.done = done; a.n_open = n_open;
  launch_pdl(beam_update_kernel, dim3(K), dim3(256), smem, st, a);
  B2P_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
