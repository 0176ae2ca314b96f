// One persistent, warp-specialised wgmma kernel for every dense contraction on the parse hot path:
//   mode 0  C[M,N] = A[M,K] * B[N,K]^T                 (1x1 convs on NHWC, all transformer linears, LM head)
//   mode 1  3x3 stride-1 pad-1 convolution on NHWC      (implicit GEMM: 9 shifted TMA boxes per Cin block)
//   mode 2  3x3 stride-2 pad-1 convolution on NHWC      (implicit GEMM through a 5-D even/odd "parity" view)
// Operands fp16 (or bf16), accumulate fp32 in registers, fused epilogue: +bias, SiLU / exact GELU, +residual,
// store fp16 or fp32 into a channel slice (row stride ldc) of the destination so concats are never
// materialised.  Replaces the cuDNN/cuBLAS library kernels behind ref:util/yolov9.py:120-121 (TorchScript
// YOLOv9-E forward) and ref:util/utils.py:125 (Florence-2 generate).
//
// Roles (384 threads = 3 warpgroups): warp 0 = TMA producer (one elected lane; the rest of its warpgroup exits and the
// warpgroup hands its registers over with setmaxnreg), warpgroups 1 and 2 = consumers: each issues the wgmma of 64 of
// the tile's 128 rows and then runs the epilogue of those rows from its register accumulators.  While the consumers are
// in an epilogue the producer already fills the ring for the next tile.
// Pipelines: smem ring full/empty (TMA <-> wgmma); a stage is empty when both consumer warpgroups have released it.
#include "ptx.cuh"
#include "b2p_internal.h"
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <mutex>
#include <atomic>

namespace b2p {

static constexpr int kThreads = 384;      // producer warpgroup + 2 consumer warpgroups
static constexpr int kConsumerGroups = 2;
static constexpr int kConsumerThreads = kConsumerGroups * 128;
static constexpr int kProducerRegs = 56, kConsumerRegs = 224;   // setmaxnreg: 128 * 56 + 256 * 224 <= 64 K registers
static constexpr int kStagePitch = 36;    // floats per row of the epilogue's staging slices (32 columns + 4: conflict-free float4 reads)
static constexpr int kEpiStageBytes = 8 * 16 * kStagePitch * 4;   // 8 consumer warps x 16 rows
static constexpr int kTileM = 128;
static constexpr int kASlot = 16384;    // 128 rows x 128 B
static constexpr int kMaxStages = 8;

// q = n / d for 0 <= n < 2^31 by multiply-high + shift (d >= 1), precomputed on the host
struct FastDiv {
  uint32_t mul, shr;
  __host__ static FastDiv make(int d) {
    FastDiv f;
    if (d <= 1) { f.mul = 0; f.shr = 0; return f; }          // shr == 0 marks d == 1
    uint32_t l = 0;
    while ((1u << l) < uint32_t(d)) ++l;                     // ceil(log2 d)
    const unsigned long long m = ((1ull << (32 + l)) + uint32_t(d) - 1) / uint32_t(d);   // ceil(2^(32+l) / d)  (33 bits)
    f.mul = uint32_t(m - (1ull << 32));
    f.shr = l;
    return f;
  }
  __device__ __forceinline__ int div(int n) const {
    if (shr == 0) return n;
    const uint32_t t = __umulhi(uint32_t(n), mul);
    return int((((uint32_t(n) - t) >> 1) + t) >> (shr - 1));   // Granlund-Montgomery round-up method, d in [2, 2^31)
  }
};

struct GemmArgs {
  int mode, M, N, num_kb, bk, bn;
  FastDiv d_ksplit, d_ntiles, d_mtiles, d_perimg, d_tilesx, d_cinb;   // divisors of the item -> tile decode
  int cin_blocks, tw, th, tiles_x, tiles_y, Ho, Wo, batch;
  int m_tiles, n_tiles, stages, ldpar;
  int nb;                // images per tile (small maps: a TMA box spans nb consecutive images)
  int tw_valid;          // valid output columns per tile row (== tw except in halo mode, where tw is the halo pitch)
  int stagesA, cin;      // separate-pipeline modes: A ring depth; Cin
  uint32_t a_slot;       // bytes per A slot (single ring: per A half, 128 rows x bk)
  // sep: A and B move through SEPARATE pipelines (always in halo mode 3, where one A tile feeds nine weight taps).
  // bres (implies sep): the WHOLE weight matrix of this launch (n_tiles == 1) stays resident in shared memory -- every B
  // k-block is loaded once per CTA, on its first work item, and the persistent loop afterwards streams only A tiles.  For
  // the small-channel layers (N, Cin <= 64..256 on the 160x160 / 80x80 maps: 10+ tiles per CTA) the weight re-loads and
  // their barrier round trips are the per-tile critical path.
  int sep, bres, taps;
  int ksplit, kb_per;    // split-K: work item = (m tile, n tile, k slice); the last CTA to arrive for a tile reduces + stores
  uint32_t a_bytes, b_bytes, b_slot;
  int bf16;
  uint64_t desc_hi;   // high 32 bits of the smem matrix descriptor (SBO, version, layout), shifted in place
  void* out;
  long long ldc;
  int out_f32;
  const float* bias;
  const void* res;
  long long ldr;
  int act, vec_ok;
  int split;   // > 0: fp16 output in the fp16x3 operand layout: hi at column n, lo at column split + n (lo-plane offset)
  int res_lo;  // > 0: the fp16 residual is a hi/lo pair too, lo at column res_lo + n
  // fp16x3 operands: A rows are [hi(K) | lo(K)] (conv: per pixel [hi(Cin) | lo(Cin)]), W rows [hi | lo] likewise.  Each
  // pipeline stage holds A_hi, A_lo, B_hi, B_lo of ONE logical k-block (each loaded once) and the consumers issue the
  // three products hi*hi + hi*lo + lo*hi into the same fp32 accumulator.  The k-blocks are 32 wide (64B swizzle): a
  // 64-wide fp16x3 stage at BN=256 is 96 KiB, so only two would fit and one stage would load while the other is read;
  // 32-wide stages give the ring four.  The k16 steps, and so every sum, run in the same order either way.
  int mt_fast;   // tile order: 1 = M tiles fastest (concurrent CTAs share a B tile: weights larger than activations, e.g. the LM head)
  int x3, lo_a, lo_b, b_tap;   // lo_a / lo_b: column offset of the lo half in A / B; b_tap: B columns per conv tap
  float* ws;   // split-K partial tiles [tile][slice][128][bn] fp32
  int* counters;   // split-K {arrived, finished} counters per output tile (self-resetting)
  int sk_last;     // split-K variant: 1 = last arriver reduces (wait-free, B2P_SPLITK_LAST=1), 0 = distributed reduction
  int park;        // 1 = park-only: every (tile, k slice) leaves its raw fp32 accumulators in ws and the kernel ends; the
                   // following kernel (splitk_ln_kernel) sums the slices, adds bias + residual and applies LayerNorm
  unsigned long long* trace;   // B2P_TRACE=1 only, else null: [CTA][16] globaltimer stamps (see trace_stamp)
  // TMA epilogue (mode 0, direct launches only, see plan_epilogue): each 64-byte-wide column chunk of the whole 128-row
  // tile is built in one of two shared-memory staging buffers and written by one TMA store (tmC); the residual of the
  // chunk arrives by TMA (tmR) into one of two residual buffers, issued two chunks ahead (the first two at item start, so
  // they land under the tile's MMAs).  epi_bytes = the epilogue's shared-memory region either way.
  int tma_epi, out_planes, res_planes;   // planes: 2 = a [hi | lo] fp16 pair (split output / res_lo), 1 = one plane
  uint32_t epi_buf, res_buf, epi_bytes;  // bytes of one staging / residual buffer, of the whole region
};

// Shared-memory matrix descriptor (PTX ISA "wgmma matrix descriptor"), K-major operand, swizzled:
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (=1, unused for swizzled K-major) | [32,46) SBO >> 4
//   [49,52) matrix base offset (0: every slot is 1024-B aligned) | [62,64) layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B.
// SBO = byte distance between consecutive 8-row groups (8 rows x row pitch).
__host__ __device__ inline uint64_t make_desc_hi(int bk) {
  const uint64_t sbo = (bk == 64) ? 1024 : 512;
  const uint64_t layout = (bk == 64) ? 1 : 2;
  return (uint64_t(1) << 16) | ((sbo >> 4) << 32) | (layout << 62);
}

__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float silu_fn(float x) {
  return x * fast_rcp(1.0f + fast_ex2(x * -1.4426950408889634f));   // SiLU: 2 MUFU + 3 FP32, ~2 ulp
}
// exact (erf) GELU, Florence-2 parity: erf by Abramowitz-Stegun 7.1.26 (|err| < 1.5e-7) on MUFU rcp/ex2 instead
// of the ~25-instruction libdevice erff: the GELU epilogues were instruction-bound
__device__ __forceinline__ float gelu_fn(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = fast_rcp(fmaf(0.3275911f, z, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = 1.0f - p * t * fast_ex2(z * z * -1.4426950408889634f);   // erf(|x|/sqrt2)
  return 0.5f * x + 0.5f * fabsf(x) * e;                                      // 0.5 x (1 + sign(x) erf)
}
__device__ __forceinline__ float act_fn(float x, int act) {
  if (act == 1) return silu_fn(x);
  if (act == 2) return gelu_fn(x);
  return x;
}
// Activation of N accumulator columns.  The switch on the (runtime) activation code sits OUTSIDE the element loop: with
// act_fn(x[j], act) inside it the compiler kept one basic block per element (uniform branch, then the dependent
// FMUL -> MUFU.EX2 -> FADD -> MUFU.RCP -> FMUL chain), so the 16 chains run back to back at full MUFU latency instead of
// interleaved.
template <int N>
__device__ __forceinline__ void act_n(float (&x)[N], int act) {
  if (act == 1) {
#pragma unroll
    for (int j = 0; j < N; ++j) x[j] = silu_fn(x[j]);
  } else if (act == 2) {
#pragma unroll
    for (int j = 0; j < N; ++j) x[j] = gelu_fn(x[j]);
  }
}

struct EpiCtx {
  __half* outh; float* outf; const __half* resh; const float* resf;
};

// bias + activation + residual + store of 16 consecutive output columns [nb, nb+16) of one row.
// pre: bias of the 16 columns already in registers (loaded before the accumulator wait), or nullptr
__device__ __forceinline__ void epi_store16(const GemmArgs& g, const EpiCtx& e, float (&x)[16], int nb, long long pix, bool valid,
                                            const float4* pre = nullptr) {
  const bool full = (nb + 16 <= g.N);
  if (full && g.vec_ok) {
    if (g.bias) {
      const float4* bp = reinterpret_cast<const float4*>(g.bias + nb);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 b = pre ? pre[q] : __ldg(bp + q);
        x[4 * q + 0] += b.x; x[4 * q + 1] += b.y; x[4 * q + 2] += b.z; x[4 * q + 3] += b.w;
      }
    }
    act_n(x, g.act);
    if (!valid) return;
    if (g.res) {
      if (g.out_f32) {
        const float4* rp = reinterpret_cast<const float4*>(e.resf + pix * g.ldr + nb);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 t = rp[q];
          x[4 * q] += t.x; x[4 * q + 1] += t.y; x[4 * q + 2] += t.z; x[4 * q + 3] += t.w;
        }
      } else {
        uint4 rr_[2];
        const uint4* rp = reinterpret_cast<const uint4*>(e.resh + pix * g.ldr + nb);
        rr_[0] = rp[0]; rr_[1] = rp[1];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const __half2* hp = reinterpret_cast<const __half2*>(&rr_[q]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 f = __half22float2(hp[k]);
            x[8 * q + 2 * k] += f.x;
            x[8 * q + 2 * k + 1] += f.y;
          }
        }
        if (g.res_lo) {
          const uint4* rl = reinterpret_cast<const uint4*>(e.resh + pix * g.ldr + g.res_lo + nb);
          rr_[0] = rl[0]; rr_[1] = rl[1];
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const __half2* hp = reinterpret_cast<const __half2*>(&rr_[q]);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 f = __half22float2(hp[k]);
              x[8 * q + 2 * k] += f.x;
              x[8 * q + 2 * k + 1] += f.y;
            }
          }
        }
      }
    }
    if (g.out_f32) {
      float4* op = reinterpret_cast<float4*>(e.outf + pix * g.ldc + nb);
#pragma unroll
      for (int q = 0; q < 4; ++q) op[q] = make_float4(x[4 * q], x[4 * q + 1], x[4 * q + 2], x[4 * q + 3]);
    } else {
      uint4 pk[2];
      __half2* hp = reinterpret_cast<__half2*>(pk);
#pragma unroll
      for (int k = 0; k < 8; ++k) hp[k] = __floats2half2_rn(x[2 * k], x[2 * k + 1]);
      uint4* op = reinterpret_cast<uint4*>(e.outh + pix * g.ldc + nb);
      op[0] = pk[0];
      op[1] = pk[1];
      if (g.split) {
        uint4 lo[2];
        __half2* lp = reinterpret_cast<__half2*>(lo);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float2 hf = __half22float2(hp[k]);
          lp[k] = __floats2half2_rn(x[2 * k] - hf.x, x[2 * k + 1] - hf.y);
        }
        uint4* o3 = reinterpret_cast<uint4*>(e.outh + pix * g.ldc + g.split + nb);
        o3[0] = lo[0];
        o3[1] = lo[1];
      }
    }
  } else {
    // ragged tail / unaligned destination: scalar path
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = nb + j;
      if (n < g.N) {
        float t = x[j];
        if (g.bias) t += __ldg(g.bias + n);
        t = act_fn(t, g.act);
        if (valid) {
          if (g.res) {
            t += g.out_f32 ? e.resf[pix * g.ldr + n] : __half2float(e.resh[pix * g.ldr + n]);
            if (g.res_lo) t += __half2float(e.resh[pix * g.ldr + g.res_lo + n]);
          }
          if (g.out_f32) e.outf[pix * g.ldc + n] = t;
          else {
            const __half hh = __float2half_rn(t);
            e.outh[pix * g.ldc + n] = hh;
            if (g.split) e.outh[pix * g.ldc + g.split + n] = __float2half_rn(t - __half2float(hh));
          }
        }
      }
    }
  }
}

// Phase stamps of a traced launch (B2P_TRACE=1, tools/trace_gemm.py): where a launch's microseconds go.
// Slots past kTrExit are not stamps but sums over all of the CTA's items: kTrSumMain = item start -> accumulators ready
// (main loop, TMA waits included), kTrSumEpi = accumulators ready -> item end (epilogue, split-K reduction included);
// kTrMark = start of the current phase.  They live in the stamp buffer: a register held across the main loop makes the
// BN = 256 instantiation spill.
enum { kTrEntry = 0, kTrPrologue, kTrDepWait, kTrFirstTma, kTrFirstFull, kTrFirstAccDone, kTrFirstEpiStart, kTrLastEpiEnd, kTrExit,
       kTrSumMain, kTrSumEpi, kTrMark };
__device__ __forceinline__ unsigned long long trace_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned long long& trace_at(const GemmArgs& g, int slot) { return g.trace[blockIdx.x * 16 + slot]; }
__device__ __forceinline__ void trace_stamp(const GemmArgs& g, int slot) {
  if (g.trace) trace_at(g, slot) = trace_now();
}
// adds the time since the last mark to the sum `slot` and marks now (call from one thread)
__device__ __forceinline__ void trace_phase(const GemmArgs& g, int slot) {
  if (g.trace) {
    const unsigned long long t = trace_now();
    trace_at(g, slot) += t - trace_at(g, kTrMark);
    trace_at(g, kTrMark) = t;
  }
}

// TMA epilogue (GemmArgs::tma_epi).  A buffer holds [plane][128 rows][64 B] in the TMA 64-byte swizzle: 16-byte unit u of
// row r sits at unit u ^ ((r >> 1) & 3), which makes the fragment's shared-memory accesses below bank-conflict free.
static constexpr uint32_t kEpiPlane = kTileM * 64;
// bias pair load that stays in program order (asm volatile): hoisted out of the chunk loop, the __ldg loads of a whole
// BN = 256 tile would hold 128 registers next to the 128 accumulators
__device__ __forceinline__ float2 ldg_f2_in_order(const float* p) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float2 lds_f2(uint32_t a) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ float2 lds_h2(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return __half22float2(*reinterpret_cast<const __half2*>(&v));
}
__device__ __forceinline__ void sts_f2(uint32_t a, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void sts_h2(uint32_t a, __half2 h) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(*reinterpret_cast<const uint32_t*>(&h)) : "memory");
}
// residual of column chunk c of the tile (mt, n0) into residual buffer c & 1 (one thread)
__device__ __forceinline__ void epi_res_load(const GemmArgs& g, const CUtensorMap* tmR, int c, int mt, int n0, uint32_t rsb, uint32_t bar_res) {
  const int cols = g.out_f32 ? 16 : 32;
  const uint32_t bar = bar_res + 8u * uint32_t(c & 1);
  const uint32_t dst = rsb + uint32_t(c & 1) * g.res_buf;
  mbar_expect_tx(bar, g.res_buf);
  if (g.res_planes == 2) tma_load_3d(dst, tmR, bar, n0 + c * cols, mt * kTileM, 0);
  else tma_load_2d(dst, tmR, bar, n0 + c * cols, mt * kTileM);
}
// The epilogue of one direct mode-0 tile straight from the wgmma fragment (lane l of consumer warp w holds rows 16w + l/4
// and 16w + l/4 + 8, and of each 8-column group the columns 2(l%4), +1), one 64-byte column chunk at a time.  Per element
// the fp32 order of epi_store16: acc + bias -> activation -> + residual hi -> + residual lo -> round (lo = x - hi).
// Staging buffer (sbuf & 1) is rewritten only after the store issued from it two chunks earlier has read it.
template <int BN, bool F32>
__device__ __forceinline__ void epi_tma(const GemmArgs& g, const CUtensorMap* tmC, const CUtensorMap* tmR, const float (&acc)[BN / 2],
                                        int mt, int n0, int row, int ctid, uint32_t stg, uint32_t bar_res, uint32_t& sbuf,
                                        uint32_t& rphase) {
  constexpr int kCols = F32 ? 16 : 32;     // columns of a 64-byte chunk
  constexpr int kGroups = kCols / 8;       // 8-column fragment groups per chunk
  if constexpr (BN % kCols == 0) {
    const int q = threadIdx.x & 3;
    // byte offsets of this thread's column pair of group 0 in rows `row` and `row + 8`; group jj is at offset ^ (jj << 4)
    // (fp32: ^ (jj << 5)) since the swizzle XORs 16-byte unit indices
    const uint32_t sw = ((uint32_t(row) >> 1) & 3u) << 4;
    const uint32_t in_row = F32 ? ((uint32_t(q >> 1) << 4) ^ sw) | (uint32_t(q & 1) << 3) : sw | (uint32_t(q) << 2);
    const uint32_t offA = uint32_t(row) * 64u + in_row, offB = offA + 8u * 64u;
    const uint32_t rsb = stg + 2 * g.epi_buf;
#pragma unroll
    for (int c = 0; c < BN / kCols; ++c) {
      float x[4 * kGroups];
#pragma unroll
      for (int jj = 0; jj < kGroups; ++jj) {
        const int a = (c * kGroups + jj) * 4;
        const int col = n0 + c * kCols + 8 * jj + 2 * q;
        float2 b = make_float2(0.f, 0.f);
        if (g.bias && col < g.N) b = ldg_f2_in_order(g.bias + col);
        x[4 * jj] = acc[a] + b.x; x[4 * jj + 1] = acc[a + 1] + b.y;
        x[4 * jj + 2] = acc[a + 2] + b.x; x[4 * jj + 3] = acc[a + 3] + b.y;
      }
      act_n(x, g.act);
      constexpr uint32_t kStep = F32 ? 32u : 16u;
      if (g.res) {
        mbar_wait(bar_res + 8u * uint32_t(c & 1), (rphase >> (c & 1)) & 1u);
        rphase ^= 1u << (c & 1);
        const uint32_t rb = rsb + uint32_t(c & 1) * g.res_buf;
#pragma unroll
        for (int jj = 0; jj < kGroups; ++jj) {
          const uint32_t oa = offA ^ (uint32_t(jj) * kStep), ob = offB ^ (uint32_t(jj) * kStep);
          if constexpr (F32) {
            const float2 ta = lds_f2(rb + oa), tb = lds_f2(rb + ob);
            x[4 * jj] += ta.x; x[4 * jj + 1] += ta.y; x[4 * jj + 2] += tb.x; x[4 * jj + 3] += tb.y;
          } else {
            for (int pl = 0; pl < g.res_planes; ++pl) {
              const float2 ta = lds_h2(rb + pl * kEpiPlane + oa), tb = lds_h2(rb + pl * kEpiPlane + ob);
              x[4 * jj] += ta.x; x[4 * jj + 1] += ta.y; x[4 * jj + 2] += tb.x; x[4 * jj + 3] += tb.y;
            }
          }
        }
      }
      const uint32_t sb = stg + (sbuf & 1u) * g.epi_buf;
#pragma unroll
      for (int jj = 0; jj < kGroups; ++jj) {
        const uint32_t oa = offA ^ (uint32_t(jj) * kStep), ob = offB ^ (uint32_t(jj) * kStep);
        if constexpr (F32) {
          sts_f2(sb + oa, x[4 * jj], x[4 * jj + 1]);
          sts_f2(sb + ob, x[4 * jj + 2], x[4 * jj + 3]);
        } else {
          const __half2 ha = __floats2half2_rn(x[4 * jj], x[4 * jj + 1]), hb = __floats2half2_rn(x[4 * jj + 2], x[4 * jj + 3]);
          sts_h2(sb + oa, ha);
          sts_h2(sb + ob, hb);
          if (g.out_planes == 2) {
            const float2 fa = __half22float2(ha), fb = __half22float2(hb);
            sts_h2(sb + kEpiPlane + oa, __floats2half2_rn(x[4 * jj] - fa.x, x[4 * jj + 1] - fa.y));
            sts_h2(sb + kEpiPlane + ob, __floats2half2_rn(x[4 * jj + 2] - fb.x, x[4 * jj + 3] - fb.y));
          }
        }
      }
      fence_proxy_async_smem();
      if (ctid == 0) bulk_wait_read<0>();   // the other buffer's store has read it: it may be rewritten after the barrier
      asm volatile("bar.sync 2, %0;" ::"n"(kConsumerThreads) : "memory");
      if (ctid == 0) {
        if (g.out_planes == 2) tma_store_3d(tmC, sb, n0 + c * kCols, mt * kTileM, 0);
        else tma_store_2d(tmC, sb, n0 + c * kCols, mt * kTileM);
        bulk_commit();
        if (g.res && c + 2 < BN / kCols) epi_res_load(g, tmR, c + 2, mt, n0, rsb, bar_res);
      }
      ++sbuf;
    }
  }
}

// All k-steps of one (A, B) stage: 64 rows of this warpgroup x BN columns, fp32 accumulate in registers.  a_lo / b_lo are
// the low descriptor words (start address >> 4 | LBO field); advancing K by 16 elements inside the swizzle span is +2.
template <int BN, bool kBf16>
__device__ __forceinline__ void mma_stage(float (&acc)[BN / 2], uint32_t a_lo, uint32_t b_lo, uint32_t dhi, int ksteps, uint32_t b_rows16,
                                          uint32_t accum) {
  for (int k = 0; k < ksteps; ++k) {
    const uint64_t da = (uint64_t(dhi) << 32) | (a_lo + 2u * k), db = (uint64_t(dhi) << 32) | (b_lo + 2u * k);
    wgmma_tile<kBf16, BN, 0>(acc, da, db, b_rows16, k == 0 ? accum : 1u);
  }
}
// fp16x3 operands: per k-step hi*hi (+)=, hi*lo +=, lo*hi += into the same accumulator
template <int BN>
__device__ __forceinline__ void mma_stage_x3(float (&acc)[BN / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo, uint32_t dhi,
                                             int ksteps, uint32_t b_rows16, uint32_t accum) {
  for (int k = 0; k < ksteps; ++k) {
    const uint64_t hi = uint64_t(dhi) << 32;
    const uint64_t dah = hi | (a_hi + 2u * k), dal = hi | (a_lo + 2u * k), dbh = hi | (b_hi + 2u * k), dbl = hi | (b_lo + 2u * k);
    wgmma_tile<false, BN, 0>(acc, dah, dbh, b_rows16, k == 0 ? accum : 1u);
    wgmma_tile<false, BN, 0>(acc, dah, dbl, b_rows16, 1u);
    wgmma_tile<false, BN, 0>(acc, dal, dbh, b_rows16, 1u);
  }
}

// kTma: the instantiation of the launches planned with the TMA epilogue (direct mode-0 tiles only).  It is a kernel of its
// own: compiled next to the register epilogue and the split-K paths, the TMA epilogue makes ptxas spill at BN = 192 / 256
// (a register cap of 168 at 384 threads, 128 of them accumulators).
template <int BN, bool kTma>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
                  const __grid_constant__ CUtensorMap tmR, const GemmArgs g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t a_part = g.x3 ? 2u * g.a_slot : g.a_slot;                          // single ring: [A_hi][A_lo] | [A]
  const uint32_t stage_bytes = g.sep ? g.b_slot : a_part + (g.x3 ? 2u : 1u) * g.b_slot;
  const uint32_t a_region = g.sep ? uint32_t(g.stagesA) * g.a_slot : 0u;   // separate pipelines: [A slots][B slots]
  float* epi_stage = reinterpret_cast<float*>(smem + a_region + size_t(g.stages) * stage_bytes);   // [8 warps][16 rows][kStagePitch]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(epi_stage) + g.epi_bytes);
  const uint32_t bar_full = smem_u32(bars);
  const uint32_t bar_empty = bar_full + 8 * g.stages;
  const uint32_t bar_afull = bar_empty + 8 * g.stages;     // separate pipelines only
  const uint32_t bar_aempty = bar_afull + 8 * g.stagesA;
  uint32_t* s_flag = reinterpret_cast<uint32_t*>(bars + 2 * g.stages + 2 * g.stagesA);
  const uint32_t bar_res = smem_u32(bars + 2 * g.stages + 2 * g.stagesA + 1);   // TMA epilogue: residual buffer 0 / 1 full

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;              // 0 = producer warpgroup, 1 / 2 = consumers (rows 0..63 / 64..127 of the tile)

  // Programmatic dependent launch: this grid is persistent (<= one CTA per SM, all resident), so the next kernel in
  // the stream may start launching right away; its CTAs run their prologue on SMs as they free up and then block in
  // griddepcontrol.wait until this grid has completed and flushed.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (threadIdx.x == 0) trace_stamp(g, kTrEntry);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (kTma) {
      tma_prefetch_desc(&tmC);
      if (g.res) tma_prefetch_desc(&tmR);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < g.stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, kConsumerGroups);
    }
    for (int a = 0; a < g.stagesA; ++a) {
      mbar_init(bar_afull + 8 * a, 1);
      mbar_init(bar_aempty + 8 * a, kConsumerGroups);
    }
    if (kTma) {
      mbar_init(bar_res, 1);
      mbar_init(bar_res + 8, 1);
    }
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) trace_stamp(g, kTrPrologue);
  // everything above touched only this CTA's shared memory; global reads/writes start below
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (threadIdx.x == 0) trace_stamp(g, kTrDepWait);

  const int total_items = g.m_tiles * g.n_tiles * g.ksplit;   // item = (mt * n_tiles + nt) * ksplit + ks
  const uint32_t smem_base = smem_u32(smem);

  if (wg == 0) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp != 0) return;
    // ------------------------------------------------------------ TMA producer
    // Warp-converged: all lanes run the loop and wait on the "empty" barriers, one elected lane issues the TMA
    // instructions; loop state lives in registers, item -> tile coordinates by multiply-shift division.
    const int n_stages = g.stages, n_stagesA = g.stagesA, ksplit = g.ksplit, kb_per = g.kb_per, num_kb = g.num_kb;
    const int mode = g.mode, bk = g.bk, bn = g.bn, cin = g.cin, cin_blocks = g.cin_blocks, b_tap = g.b_tap, ldpar = g.ldpar;
    const int th = g.th, tw_valid = g.tw_valid, nb = g.nb, lo_a = g.lo_a, lo_b = g.lo_b, taps = g.taps;
    const bool sep = g.sep != 0, bres = g.bres != 0, x3 = g.x3 != 0, mt_fast = g.mt_fast != 0;
    const uint32_t a_bytes = g.a_bytes, b_bytes = g.b_bytes, a_slot = g.a_slot, b_slot = g.b_slot;
    const FastDiv d_ksplit = g.d_ksplit, d_ntiles = g.d_ntiles, d_mtiles = g.d_mtiles, d_perimg = g.d_perimg, d_tilesx = g.d_tilesx,
                  d_cinb = g.d_cinb;
    const uint32_t b_base = smem_base + a_region;
    int stage = 0, stageA = 0;
    uint32_t phase = 0, phaseA = 0;
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
      const int tile = d_ksplit.div(item);
      const int ks = item - tile * ksplit;
      int nt, mt;
      if (mt_fast) { nt = d_mtiles.div(tile); mt = tile - nt * g.m_tiles; }
      else { mt = d_ntiles.div(tile); nt = tile - mt * g.n_tiles; }
      const int n0 = nt * bn;
      int img = 0, y0 = 0, x0 = 0;
      if (mode != 0) {
        img = d_perimg.div(mt);
        const int r = mt - img * g.tiles_x * g.tiles_y;
        const int ty = d_tilesx.div(r);
        y0 = ty * th;
        x0 = (r - ty * g.tiles_x) * tw_valid;
        img *= nb;   // nb > 1 only when one tile covers whole images (per_img == 1)
      }
      const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
      if (sep) {
        // separate pipelines.  Halo mode (3): ONE (th+2) x (tw+2) input tile per channel block feeds all nine taps (the MMA
        // side shifts the smem descriptor start address by (ky*pitch + kx) rows); only the weights stream per tap.
        // Other modes: one A tile per k-block.  Resident weights (bres): B slot (unit*taps + tap) is filled on this CTA's
        // first item only and never released.
        const bool first_item = (item == int(blockIdx.x));
        for (int u = kb0; u < kb1; ++u) {
          mbar_wait(bar_aempty + 8 * stageA, phaseA ^ 1);
          const uint32_t fa = bar_afull + 8 * stageA;
          const uint32_t dstA = smem_base + uint32_t(stageA) * a_slot;
          mbar_expect_tx_elect(fa, a_bytes);
          int bcol0;
          if (mode == 3) {
            tma_load_4d_elect(dstA, &tmA, fa, u * bk, x0 - 1, y0 - 1, img);
            bcol0 = u * bk;                                   // + tap * cin below
          } else if (mode == 0) {
            tma_load_2d_elect(dstA, &tmA, fa, u * bk, mt * kTileM);
            bcol0 = u * bk;
          } else {
            const int tap = d_cinb.div(u);
            const int c0 = (u - tap * cin_blocks) * bk;
            const int ky = (tap * 11) >> 5, kx = tap - ky * 3;     // tap / 3 for tap in 0..8
            bcol0 = tap * b_tap + c0;
            if (mode == 1) {
              tma_load_4d_elect(dstA, &tmA, fa, c0, x0 + kx - 1, y0 + ky - 1, img);
            } else {
              const int py = (ky != 1), px = (kx != 1);
              const int yo = y0 - (ky == 0), xo = x0 - (kx == 0);
              tma_load_5d_elect(dstA, &tmA, fa, c0 + px * ldpar, xo, py, yo, img);
            }
          }
          if (item == blockIdx.x && u == kb0 && lane == 0) trace_stamp(g, kTrFirstTma);
          if (++stageA == n_stagesA) { stageA = 0; phaseA ^= 1; }
          if (bres) {
            if (first_item) {
              for (int tap = 0; tap < taps; ++tap) {
                const int slot = (u - kb0) * taps + tap;
                const uint32_t fb = bar_full + 8 * slot;
                mbar_expect_tx_elect(fb, b_bytes);
                tma_load_2d_elect(b_base + uint32_t(slot) * b_slot, &tmB, fb, (mode == 3) ? tap * cin + bcol0 : bcol0, n0);
              }
            }
            continue;
          }
          for (int tap = 0; tap < taps; ++tap) {
            mbar_wait(bar_empty + 8 * stage, phase ^ 1);
            const uint32_t fb = bar_full + 8 * stage;
            mbar_expect_tx_elect(fb, b_bytes);
            tma_load_2d_elect(b_base + uint32_t(stage) * b_slot, &tmB, fb, (mode == 3) ? tap * cin + bcol0 : bcol0, n0);
            if (++stage == n_stages) { stage = 0; phase ^= 1; }
          }
        }
        continue;
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
        const uint32_t fb = bar_full + 8 * stage;
        const uint32_t sa = smem_base + uint32_t(stage) * stage_bytes;
        const uint32_t sb = sa + a_part;
        mbar_expect_tx_elect(fb, x3 ? 2u * (a_bytes + b_bytes) : a_bytes + b_bytes);
        int bcol = kb * bk;
        int tap = 0, c0 = 0, ky = 0, kx = 0;
        if (mode != 0) {
          tap = d_cinb.div(kb);
          c0 = (kb - tap * cin_blocks) * bk;
          ky = (tap * 11) >> 5; kx = tap - ky * 3;
          bcol = tap * b_tap + c0;
        }
        for (int half = 0; half <= int(x3); ++half) {     // half 1 = the lo parts (fp16x3 operands only)
          const uint32_t dst = sa + uint32_t(half) * a_slot;
          const int ca = half * lo_a;
          if (mode == 0) {
            tma_load_2d_elect(dst, &tmA, fb, ca + kb * bk, mt * kTileM);
          } else if (mode == 1) {
            tma_load_4d_elect(dst, &tmA, fb, ca + c0, x0 + kx - 1, y0 + ky - 1, img);
          } else {
            // input row 2*oy + (ky-1): ky=0 -> (oy-1, odd), ky=1 -> (oy, even), ky=2 -> (oy, odd); same in x.
            const int py = (ky != 1), px = (kx != 1);
            const int yo = y0 - (ky == 0), xo = x0 - (kx == 0);
            tma_load_5d_elect(dst, &tmA, fb, ca + c0 + px * ldpar, xo, py, yo, img);
          }
        }
        tma_load_2d_elect(sb, &tmB, fb, bcol, n0);
        if (x3) tma_load_2d_elect(sb + b_slot, &tmB, fb, bcol + lo_b, n0);
        if (item == blockIdx.x && kb == kb0 && lane == 0) trace_stamp(g, kTrFirstTma);
        if (++stage == n_stages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- consumers: wgmma main loop + epilogue
  // Two warpgroups share every pipeline stage: warpgroup cw multiplies rows [64 cw, 64 cw + 64) of the A tile with the whole
  // B tile into its own register accumulators, and a stage goes back to the producer when both have read it.  One wgmma
  // group stays in flight: the stage of group n-1 is released after group n has been committed.
  setmaxnreg_inc<kConsumerRegs>();
  const int cw = wg - 1;
  const int ctid = threadIdx.x - 128;                 // 0..255 over the consumer threads
  const bool wg_leader = (threadIdx.x & 127) == 0;    // arrives on the "empty" barriers for its warpgroup
  const int n_stages = g.stages, n_stagesA = g.stagesA, ksplit = g.ksplit, kb_per = g.kb_per, num_kb = g.num_kb;
  const bool sep = g.sep != 0, bres = g.bres != 0, halo = (g.mode == 3), x3 = g.x3 != 0, bf16 = g.bf16 != 0;
  const int ksteps = g.bk >> 4;
  const uint32_t a_slot = g.a_slot, b_slot = g.b_slot;
  const uint32_t dhi = uint32_t(g.desc_hi >> 32), dlo = uint32_t(g.desc_hi);       // descriptor halves (dlo = the LBO field)
  const uint32_t row16 = uint32_t(16 * 2 * g.bk) >> 4;                              // 16 operand rows, in descriptor units
  const uint32_t wg_rows = uint32_t(cw) * 4u * row16;                               // this warpgroup's 64-row offset into an A tile
  const uint32_t row_shift = (uint32_t(g.tw) * uint32_t(2 * g.bk)) >> 4, col_shift = uint32_t(2 * g.bk) >> 4;   // halo taps
  const uint32_t b_base = smem_base + a_region;
  int stage = 0, stageA = 0;
  uint32_t phase = 0, phaseA = 0;
  bool b_ready = false;   // resident weights: every slot has landed once the first item has been issued
  auto lo_of = [dlo](uint32_t addr) { return ((addr & 0x3FFFFu) >> 4) | dlo; };

  EpiCtx e;
  e.outh = reinterpret_cast<__half*>(g.out);
  e.outf = reinterpret_cast<float*>(g.out);
  e.resh = reinterpret_cast<const __half*>(g.res);
  e.resf = reinterpret_cast<const float*>(g.res);
  // Epilogue: each warp passes its 16 accumulator rows through its own slice of shared memory, 32 columns at a time, so
  // that a lane ends up with 16 consecutive columns of one row (lane & 15 = row, lane >> 4 = which half of the 32).
  float* my_stage = epi_stage + ((cw * 4 + (warp & 3)) * 16) * kStagePitch;
  const int piece = lane >> 4;
  // this thread's row of the tile: its position inside the (tw x th [x nb images]) tile never changes
  const int r = cw * 64 + (warp & 3) * 16 + (lane & 15);
  const int e_mode = g.mode, e_bn = g.bn, e_th = g.th, e_twv = g.tw_valid, e_nb = g.nb;
  const int e_Ho = g.Ho, e_Wo = g.Wo, e_batch = g.batch, e_tiles_x = g.tiles_x, e_per_img = g.tiles_x * g.tiles_y;
  const bool e_mtfast = g.mt_fast != 0;
  const FastDiv e_dks = g.d_ksplit, e_dnt = g.d_ntiles, e_dmt = g.d_mtiles, e_dpi = g.d_perimg, e_dtx = g.d_tilesx;
  int r_sub = 0, r_ty = 0, r_tx = 0;
  if (e_mode != 0) {
    const int rows_img = g.tw * g.th;                  // rows of one image inside the tile
    r_sub = (e_nb > 1) ? r / rows_img : 0;
    const int rloc = r - r_sub * rows_img;
    r_ty = rloc / g.tw;
    r_tx = rloc - r_ty * g.tw;
  }
  const bool r_ok = (r_sub < e_nb) && (r_ty < e_th) && (r_tx < e_twv);

  uint32_t epi_sbuf = 0, epi_rphase = 0;   // TMA epilogue: staging buffers used so far; residual buffers' mbarrier parities
  for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
    if (ctid == 0) trace_stamp(g, kTrMark);
    const int tile = e_dks.div(item);
    const int ks = item - tile * ksplit;
    if (kTma && g.res && ctid == 0) {
      // the tile's first two residual chunks land under its MMAs
      const int mt_ = e_mtfast ? tile - e_dmt.div(tile) * g.m_tiles : e_dnt.div(tile);
      const int n0_ = (e_mtfast ? e_dmt.div(tile) : tile - mt_ * g.n_tiles) * e_bn;
      const uint32_t rsb = smem_u32(epi_stage) + 2 * g.epi_buf;
      epi_res_load(g, &tmR, 0, mt_, n0_, rsb, bar_res);
      if (BN > (g.out_f32 ? 16 : 32)) epi_res_load(g, &tmR, 1, mt_, n0_, rsb, bar_res);
    }
    const int kb0 = ks * kb_per, kb1 = min(num_kb, kb0 + kb_per);
    float acc[BN / 2];           // this thread's fragment of the 64 x BN accumulator (layout: ptx.cuh)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    uint32_t accum = 0;          // the first MMA of an item overwrites the accumulator
    uint32_t prev_b = 0, prev_a = 0;   // "empty" barriers of the wgmma group still in flight (0 = nothing to release)
    auto retire = [&](uint32_t next_b, uint32_t next_a) {
      if (wg_leader) {
        if (prev_b) mbar_arrive(prev_b);
        if (prev_a) mbar_arrive(prev_a);
      }
      prev_b = next_b; prev_a = next_a;
    };
    if (sep) {
      for (int u = kb0; u < kb1; ++u) {
        mbar_wait(bar_afull + 8 * stageA, phaseA);
        const uint32_t a0 = lo_of(smem_base + uint32_t(stageA) * a_slot) + wg_rows;
        if (item == blockIdx.x && u == kb0 && ctid == 0) trace_stamp(g, kTrFirstFull);
        const int taps_y = halo ? 3 : 1;
        int slot = bres ? (u - kb0) * (halo ? 9 : 1) : stage;
        for (int ky = 0; ky < taps_y; ++ky) {
          for (int kx = 0; kx < taps_y; ++kx) {
            if (!b_ready) {
              // resident weights: slot (unit, tap) completes its one and only phase (parity 0) during the first item
              mbar_wait(bar_full + 8 * slot, bres ? 0u : phase);
            }
            // halo mode: shifted view of the halo tile.  The 128B/64B swizzle pattern is anchored at the 1024-B aligned slot
            // base (that is how TMA wrote it), so the "matrix base offset" field stays 0 even though the start address
            // points into the middle of an atom: the XOR phase is taken from the address bits, as for the K-advance.
            const uint32_t a_lo = a0 + uint32_t(ky) * row_shift + uint32_t(kx) * col_shift;
            const uint32_t b_lo = lo_of(b_base + uint32_t(slot) * b_slot);
            wgmma_fence_operand(acc);
            wgmma_fence();
            if (bf16) mma_stage<BN, true>(acc, a_lo, b_lo, dhi, ksteps, row16, accum);
            else mma_stage<BN, false>(acc, a_lo, b_lo, dhi, ksteps, row16, accum);
            wgmma_commit();
            accum = 1;
            wgmma_wait<1>();
            const bool last_tap = (ky == taps_y - 1) && (kx == taps_y - 1);
            retire(bres ? 0u : bar_empty + 8 * stage, last_tap ? bar_aempty + 8 * stageA : 0u);
            if (bres) {
              ++slot;
            } else {
              if (++stage == n_stages) { stage = 0; phase ^= 1; }
              slot = stage;
            }
          }
        }
        if (++stageA == n_stagesA) { stageA = 0; phaseA ^= 1; }
      }
      if (bres) b_ready = true;
    } else {
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase);
        if (item == blockIdx.x && kb == kb0 && ctid == 0) trace_stamp(g, kTrFirstFull);
        const uint32_t sa = smem_base + uint32_t(stage) * stage_bytes;
        const uint32_t sb = sa + a_part;
        wgmma_fence_operand(acc);
        wgmma_fence();
        if (x3) mma_stage_x3<BN>(acc, lo_of(sa) + wg_rows, lo_of(sa + a_slot) + wg_rows, lo_of(sb), lo_of(sb + b_slot), dhi, ksteps, row16, accum);
        else if (bf16) mma_stage<BN, true>(acc, lo_of(sa) + wg_rows, lo_of(sb), dhi, ksteps, row16, accum);
        else mma_stage<BN, false>(acc, lo_of(sa) + wg_rows, lo_of(sb), dhi, ksteps, row16, accum);
        wgmma_commit();
        accum = 1;
        wgmma_wait<1>();
        retire(bar_empty + 8 * stage, 0u);
        if (++stage == n_stages) { stage = 0; phase ^= 1; }
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operand(acc);
    retire(0u, 0u);
    if (item == blockIdx.x && ctid == 0) { trace_stamp(g, kTrFirstAccDone); trace_stamp(g, kTrFirstEpiStart); }
    if (ctid == 0) trace_phase(g, kTrSumMain);

    // -------------------------------------------------------------- epilogue of this item
    int nt, mt;
    if (e_mtfast) { nt = e_dmt.div(tile); mt = tile - nt * g.m_tiles; }
    else { mt = e_dnt.div(tile); nt = tile - mt * g.n_tiles; }
    const int n0 = nt * e_bn;
    if constexpr (kTma) {
      const int row = cw * 64 + (warp & 3) * 16 + (lane >> 2);
      const uint32_t stg = smem_u32(epi_stage);
      if (g.out_f32) epi_tma<BN, true>(g, &tmC, &tmR, acc, mt, n0, row, ctid, stg, bar_res, epi_sbuf, epi_rphase);
      else epi_tma<BN, false>(g, &tmC, &tmR, acc, mt, n0, row, ctid, stg, bar_res, epi_sbuf, epi_rphase);
      if (ctid == 0) trace_phase(g, kTrSumEpi);
      continue;
    }
    long long pix;
    bool valid;
    if (e_mode == 0) {
      pix = (long long)mt * kTileM + r;
      valid = pix < g.M;
    } else {
      const int img0 = e_dpi.div(mt);
      const int rr = mt - img0 * e_per_img;
      const int img = img0 * e_nb + r_sub;
      const int tyi = e_dtx.div(rr);
      const int oy = tyi * e_th + r_ty;
      const int ox = (rr - tyi * e_tiles_x) * e_twv + r_tx;
      valid = r_ok && (img < e_batch) && (oy < e_Ho) && (ox < e_Wo);
      pix = ((long long)img * e_Ho + oy) * e_Wo + ox;
    }
    const bool direct = (ksplit == 1 && !g.park);
    // split-K: every slice parks its raw fp32 partial tile, then the partials are summed in slice order (deterministic) and
    // the epilogue runs -- by the last CTA to arrive (sk_last: nobody waits for anybody, so partially resident grids cannot
    // deadlock) or, by default, distributed over the tile's ksplit CTAs (see below).
    float* wsp = direct ? nullptr : g.ws + ((size_t(tile) * ksplit + ks) * kTileM + r) * e_bn;
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += 32) {
      float* wrow = my_stage + (lane >> 2) * kStagePitch + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (c0 + 8 * j < BN) {
          const int a = (c0 / 8 + j) * 4;
          *reinterpret_cast<float2*>(wrow + 8 * j) = make_float2(acc[a], acc[a + 1]);
          *reinterpret_cast<float2*>(wrow + 8 * kStagePitch + 8 * j) = make_float2(acc[a + 2], acc[a + 3]);
        }
      }
      __syncwarp();
      const int c = c0 + piece * 16;
      const bool mine = (c < BN) && (direct ? (n0 + c < g.N) : true);
      float x[16];
      if (mine) {
        const float4* rp = reinterpret_cast<const float4*>(my_stage + (lane & 15) * kStagePitch + piece * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 t = rp[q];
          x[4 * q] = t.x; x[4 * q + 1] = t.y; x[4 * q + 2] = t.z; x[4 * q + 3] = t.w;
        }
      }
      __syncwarp();
      if (!mine) continue;
      if (direct) {
        epi_store16(g, e, x, n0 + c, pix, valid);
      } else {
        float4* wp = reinterpret_cast<float4*>(wsp + c);
#pragma unroll
        for (int q = 0; q < 4; ++q) wp[q] = make_float4(x[4 * q], x[4 * q + 1], x[4 * q + 2], x[4 * q + 3]);
      }
    }
    if (!direct && !g.park) {
      // (park-only launches stop here: the consumer kernel starts after this grid has completed)
      if (g.sk_last) {
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        volatile uint32_t* s_last = s_flag;
        if (ctid == 0) {
          int* cnt = g.counters + 2 * tile;
          const bool last = (atomicAdd(cnt, 1) == ksplit - 1);
          if (last) *cnt = 0;   // every slice has arrived: the next user of this counter is a later launch / graph replay
          *s_last = last ? 1u : 0u;
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        if (*s_last) {
          __threadfence();
          const int chunks = e_bn >> 4;
          const float* base = g.ws + size_t(tile) * ksplit * kTileM * e_bn;
          int img0 = 0, rr = 0, tyi = 0;
          if (e_mode != 0) {
            img0 = e_dpi.div(mt);
            rr = mt - img0 * e_per_img;
            tyi = e_dtx.div(rr);
          }
          const int rows_img = g.tw * g.th, tw_ = g.tw;
          for (int w = ctid; w < kTileM * chunks; w += kConsumerThreads) {
            const int rr_ = w / chunks, c = (w - rr_ * chunks) << 4;
            if (n0 + c >= g.N) continue;
            long long pix2;
            bool valid2;
            if (e_mode == 0) {
              pix2 = (long long)mt * kTileM + rr_;
              valid2 = pix2 < g.M;
            } else {
              const int sub = (e_nb > 1) ? rr_ / rows_img : 0;
              const int rloc = rr_ - sub * rows_img;
              const int img = img0 * e_nb + sub;
              const int ty = rloc / tw_, tx = rloc - ty * tw_;
              const int oy = tyi * e_th + ty;
              const int ox = (rr - tyi * e_tiles_x) * e_twv + tx;
              valid2 = (sub < e_nb) && (img < e_batch) && (ty < e_th) && (tx < e_twv) && (oy < e_Ho) && (ox < e_Wo);
              pix2 = ((long long)img * e_Ho + oy) * e_Wo + ox;
            }
            float x[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) x[j] = 0.f;
            for (int sidx = 0; sidx < ksplit; ++sidx) {
              const float4* pp = reinterpret_cast<const float4*>(base + (size_t(sidx) * kTileM + rr_) * e_bn + c);
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float4 t = __ldcg(pp + q);
                x[4 * q] += t.x; x[4 * q + 1] += t.y; x[4 * q + 2] += t.z; x[4 * q + 3] += t.w;
              }
            }
            epi_store16(g, e, x, n0 + c, pix2, valid2);
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");   // s_flag is rewritten by the next item
      } else {
        // default: DISTRIBUTED reduction -- each of the ksplit CTAs of a tile waits for the tile's arrival counter and then
        // reduces its share of the 128 rows (slice order => deterministic sums): the partials are re-read by ksplit SMs in
        // parallel instead of one.  The price is an inter-CTA wait: safe because the grid is at most one wave and the hardware
        // dispatches the CTAs of an earlier launch before those of later ones; a wait longer than ~2 s traps.
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        int* cnt = g.counters + 2 * tile;
        if (ctid == 0) {
          atomicAdd(cnt, 1);
          long long t0 = clock64();
          while (*reinterpret_cast<volatile int*>(cnt) < ksplit) {
            if (clock64() - t0 > 4000000000LL) __trap();   // (no printf: see mbar_wait)
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        __threadfence();
        const int rows_per = (kTileM + ksplit - 1) / ksplit;
        const int row0 = ks * rows_per, row1 = min(kTileM, row0 + rows_per);
        const int chunks = e_bn >> 4;
        const float* base = g.ws + size_t(tile) * ksplit * kTileM * e_bn;
        for (int w = ctid; w < (row1 - row0) * chunks; w += kConsumerThreads) {
          const int rr_ = row0 + w / chunks, c = (w % chunks) << 4;
          if (n0 + c >= g.N) continue;
          long long pix2;
          bool valid2;
          if (e_mode == 0) {
            pix2 = (long long)mt * kTileM + rr_;
            valid2 = pix2 < g.M;
          } else {
            const int img0 = mt / e_per_img;
            const int rr = mt - img0 * e_per_img;
            const int rows_img = g.tw * g.th;
            const int sub = (e_nb > 1) ? rr_ / rows_img : 0;
            const int rloc = rr_ - sub * rows_img;
            const int img = img0 * e_nb + sub;
            const int ty = rloc / g.tw, tx = rloc - ty * g.tw;
            const int oy = (rr / e_tiles_x) * e_th + ty;
            const int ox = (rr % e_tiles_x) * e_twv + tx;
            valid2 = (sub < e_nb) && (img < e_batch) && (ty < e_th) && (tx < e_twv) && (oy < e_Ho) && (ox < e_Wo);
            pix2 = ((long long)img * e_Ho + oy) * e_Wo + ox;
          }
          float x[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) x[j] = 0.f;
          // two slices per round trip: the loads of both are in flight before the first add (one slice at a time costs one L2
          // latency per slice); the adds keep the slice order
          const size_t sl_stride = size_t(kTileM) * e_bn;
          const float* pbase = base + size_t(rr_) * e_bn + c;
          int sidx = 0;
          for (; sidx + 2 <= ksplit; sidx += 2) {
            const float4* p0 = reinterpret_cast<const float4*>(pbase + size_t(sidx) * sl_stride);
            const float4* p1 = reinterpret_cast<const float4*>(pbase + size_t(sidx + 1) * sl_stride);
            float4 t0[4], t1[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) { t0[q] = __ldcg(p0 + q); t1[q] = __ldcg(p1 + q); }
#pragma unroll
            for (int q = 0; q < 4; ++q) { x[4 * q] += t0[q].x; x[4 * q + 1] += t0[q].y; x[4 * q + 2] += t0[q].z; x[4 * q + 3] += t0[q].w; }
#pragma unroll
            for (int q = 0; q < 4; ++q) { x[4 * q] += t1[q].x; x[4 * q + 1] += t1[q].y; x[4 * q + 2] += t1[q].z; x[4 * q + 3] += t1[q].w; }
          }
          if (sidx < ksplit) {
            const float4* pp = reinterpret_cast<const float4*>(pbase + size_t(sidx) * sl_stride);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float4 t = __ldcg(pp + q);
              x[4 * q] += t.x; x[4 * q + 1] += t.y; x[4 * q + 2] += t.z; x[4 * q + 3] += t.w;
            }
          }
          epi_store16(g, e, x, n0 + c, pix2, valid2);
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        if (ctid == 0) {
          // the last CTA to finish its share resets both counters for the next launch / graph replay
          if (atomicAdd(cnt + 1, 1) == ksplit - 1) { cnt[1] = 0; cnt[0] = 0; __threadfence(); }
        }
      }
    }
    if (ctid == 0) trace_phase(g, kTrSumEpi);
  }
  if (kTma && ctid == 0) bulk_wait_all();   // the stores are performed before the grid completes (PDL dependents)
  if (ctid == 0) { trace_stamp(g, kTrLastEpiEnd); trace_stamp(g, kTrExit); }
}

// ------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int encode(CUtensorMap* m, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                  const cuuint64_t* strides_bytes, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode();
  if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable");
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, dtype, rank,
                  const_cast<void*>(base), dims, strides_bytes, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed: CUresult %d (rank %d, dims %llu %llu, box %u %u)", int(r),
             rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return set_error(buf);
  }
  return 0;
}

static int g_num_sms = 0;
// Split-K scratch is per stream (two streams may run split-K GEMMs concurrently): a few slots are allocated up
// front (never inside a graph capture) and handed to streams at their first launch; a slot goes back to the free list when
// its stream is destroyed through stream_destroy.  A graph bakes in the slot of the stream it was captured on.
static constexpr int kWsSlots = 24;
static float* g_ws[kWsSlots] = {};
static int* g_counters[kWsSlots] = {};
static cudaStream_t g_ws_owner[kWsSlots] = {};
static bool g_ws_taken[kWsSlots] = {};
static std::mutex g_ws_mu;
static int ws_slot_locked(cudaStream_t st) {
  for (int i = 0; i < kWsSlots; ++i)
    if (g_ws_taken[i] && g_ws_owner[i] == st) return i;
  return -1;
}
static int ws_slot_for(cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_ws_mu);
  const int have = ws_slot_locked(st);
  if (have >= 0) return have;
  for (int i = 0; i < kWsSlots; ++i)
    if (!g_ws_taken[i]) { g_ws_taken[i] = true; g_ws_owner[i] = st; return i; }
  return -1;   // more concurrent streams than slots: the caller disables split-K for this launch
}
static constexpr size_t kWsBytes = size_t(64) << 20;     // split-K partial tiles (per slot)
static constexpr int kMaxCounterTiles = 1 << 12;   // split-K only ever covers < #SMs tiles

static int g_max_smem = 0;

// B2P_TRACE=1 (debugging aid, tools/trace_gemm.py): launches carry a stamp buffer and leave per-CTA
// globaltimer stamps; b2p_trace_read() hands them out together with the launch shapes.
static constexpr int kTraceCap = 1024, kTraceCtas = 160, kTraceSlots = 16;
static unsigned long long* g_trace = nullptr;
static int g_trace_n = 0;
static int g_trace_meta[kTraceCap][8];
static std::mutex g_trace_mu;

// one instantiation per N tile: the accumulator fragment (BN / 2 registers per consumer thread) is sized at compile time
typedef void (*GemmKernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const GemmArgs);
static constexpr int kNumBn = 8;
static const int kBnCand[kNumBn] = {256, 192, 128, 96, 64, 48, 32, 16};
// [N tile][TMA epilogue]
static const GemmKernel kGemmKernels[kNumBn][2] = {
    {gemm_wgmma_kernel<256, false>, gemm_wgmma_kernel<256, true>}, {gemm_wgmma_kernel<192, false>, gemm_wgmma_kernel<192, true>},
    {gemm_wgmma_kernel<128, false>, gemm_wgmma_kernel<128, true>}, {gemm_wgmma_kernel<96, false>, gemm_wgmma_kernel<96, true>},
    {gemm_wgmma_kernel<64, false>, gemm_wgmma_kernel<64, true>},   {gemm_wgmma_kernel<48, false>, gemm_wgmma_kernel<48, true>},
    {gemm_wgmma_kernel<32, false>, gemm_wgmma_kernel<32, true>},   {gemm_wgmma_kernel<16, false>, gemm_wgmma_kernel<16, true>}};

static std::mutex g_setup_mu;
static int device_setup() {
  if (int e = bind_device()) return e;
  std::lock_guard<std::mutex> lk(g_setup_mu);
  if (g_num_sms) return 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return set_error("cudaGetDevice failed (no CUDA device?)");
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return set_error("cudaGetDeviceProperties failed");
  if (p.major != 9) return set_error("libb200parse requires an sm_90 (Hopper H100) device");
  g_num_sms = p.multiProcessorCount;
  g_max_smem = int(p.sharedMemPerBlockOptin);
  for (int i = 0; i < kNumBn; ++i)
    for (int t = 0; t < 2; ++t)
      if (cudaFuncSetAttribute(kGemmKernels[i][t], cudaFuncAttributeMaxDynamicSharedMemorySize, g_max_smem) != cudaSuccess)
        return set_error("cudaFuncSetAttribute(max dynamic smem) failed");
  if (getenv("B2P_TRACE")) {
    if (cudaMalloc(&g_trace, sizeof(unsigned long long) * kTraceCap * kTraceCtas * kTraceSlots) != cudaSuccess)
      return set_error("B2P_TRACE: setup of the traced kernel failed");
    cudaMemset(g_trace, 0, sizeof(unsigned long long) * kTraceCap * kTraceCtas * kTraceSlots);
  }
  for (int i = 0; i < kWsSlots; ++i) {
    if (cudaMalloc(&g_ws[i], kWsBytes) != cudaSuccess || cudaMalloc(&g_counters[i], 2 * kMaxCounterTiles * sizeof(int)) != cudaSuccess)
      return set_error("cudaMalloc for the split-K workspace failed");
    cudaMemset(g_counters[i], 0, 2 * kMaxCounterTiles * sizeof(int));
  }
  return 0;
}


// Environment knobs of the planner, read once per process by gemm_knobs(); plan_gemm() itself never reads the environment.
struct GemmKnobs {
  bool no_halo;       // B2P_NO_HALO: stride-1 convs use the per-tap path (mode 1) instead of the halo tile (mode 3)
  bool no_halo32;     // B2P_NO_HALO32: no halo tile at 32-wide k-blocks
  bool no_bres;       // B2P_NO_BRES: never keep the weights resident
  bool no_split;      // B2P_NO_SPLITK: never split K
  bool sk_last;       // B2P_SPLITK_LAST: split-K reduced by the last arriving CTA instead of the distributed reduction
  bool few_ctas;      // unset B2P_DENSE_GRIDS: single-wave launches pay a charge per occupied SM
  double cta_penalty; // B2P_CTA_PENALTY: microseconds charged per CTA (default 0.02)
  int max_grid;       // B2P_MAX_GRID: experiment, cap the grid of launches that do not split K (0 = none)
  bool no_tma_epi;    // B2P_NO_TMA_EPI: every launch keeps the register epilogue (per-thread global loads and stores)
};
static const GemmKnobs& gemm_knobs() {
  static const GemmKnobs k = [] {
    GemmKnobs v{};
    v.no_halo = getenv("B2P_NO_HALO") != nullptr;
    v.no_halo32 = getenv("B2P_NO_HALO32") != nullptr;
    v.no_bres = getenv("B2P_NO_BRES") != nullptr;
    v.no_split = getenv("B2P_NO_SPLITK") != nullptr;
    v.sk_last = getenv("B2P_SPLITK_LAST") != nullptr;
    v.few_ctas = getenv("B2P_DENSE_GRIDS") == nullptr;
    v.cta_penalty = getenv("B2P_CTA_PENALTY") ? atof(getenv("B2P_CTA_PENALTY")) : 0.02;
    v.max_grid = getenv("B2P_MAX_GRID") ? atoi(getenv("B2P_MAX_GRID")) : 0;
    v.no_tma_epi = getenv("B2P_NO_TMA_EPI") != nullptr;
    return v;
  }();
  return k;
}

// Choose the N tile and the split-K factor with a small time model (microseconds per CTA):
//   per k-block  max(MMA issue, smem fill): MMA = 128 * bn * bk MACs at 2048 fp16 MACs per clock and SM, ~1.7 GHz under
//   load; fill = (A + B bytes) at ~40 GB/s per SM (the L2's ~5.5 TB/s shared by 132 SMs)
//   per item     ~2.5 us pipeline fill/drain + epilogue (~0.012 us per output column) + split-K park/reduce.
// The constants are estimates from the H100 data sheet, not fitted to measurements.
static void pick_tiling(int N, int m_tiles, int num_kb, int bk, uint32_t a_bytes, int bn_max, bool allow_split, bool x3,
                        int num_sms, int max_smem, const GemmKnobs& kn, int* bn_out, int* ksplit_out) {
  // single-wave launches: a charge per occupied SM (B2P_DENSE_GRIDS=1 selects the model that spreads every launch over as
  // many SMs as it can)
  const bool few_ctas = kn.few_ctas;
  const double cta_penalty = kn.cta_penalty;
  const int n16 = (N + 15) / 16 * 16;
  double best_cost = -1;
  int best = 16, best_ks = 1;
  for (int c : kBnCand) {
    if (c > bn_max) continue;
    if (c > n16 && c != 16) {
      bool smaller_covers = false;
      for (int d : kBnCand) if (d < c && d >= n16) smaller_covers = true;
      if (smaller_covers) continue;
    }
    const long n_tiles = (N + c - 1) / c;
    const long tiles = n_tiles * m_tiles;
    // fp16x3 operands: three MMAs and two (hi, lo) tile pairs per logical k-block
    const double t_mma = (x3 ? 3.0 : 1.0) * double(c) * bk / 16.0 / 1700.0;
    const double t_fill = (x3 ? 2.0 : 1.0) * (double(a_bytes) + double(c) * bk * 2.0) / 40000.0;
    if (x3 && 2 * (2 * kASlot + 2 * ((c * bk * 2 + 1023) & ~1023)) + 2048 + kEpiStageBytes > max_smem) continue;   // needs >= 2 stages
    const double t_kb = t_mma > t_fill ? t_mma : t_fill;
    int max_ks = 1;
    if (allow_split && tiles * 2 <= num_sms && tiles * 2 <= kMaxCounterTiles) {
      max_ks = int(num_sms / tiles);            // one wave of (tile, slice) items (a performance choice: nothing spins)
      if (max_ks > num_kb / 2) max_ks = num_kb / 2;
      if (max_ks > 32) max_ks = 32;
      if (max_ks < 1) max_ks = 1;
    }
    for (int ks = 1; ks <= max_ks; ++ks) {
      const int kb_per = (num_kb + ks - 1) / ks;
      const int ks_eff = (num_kb + kb_per - 1) / kb_per;
      if (ks_eff != ks) continue;
      if (ks > 1 && size_t(tiles) * ks * 128 * c * 4 > kWsBytes) continue;
      const long items = tiles * ks;
      const long waves = (items + num_sms - 1) / num_sms;
      // split-K overhead: park one fp32 partial tile + read one tile's worth back (distributed reduce) at ~100 GB/s/SM
      double t_split = ks > 1 ? 2.0 + 2.0 * (128.0 * c * 4.0 / 100000.0) : 0.0;
      double t_kb_ = t_kb;
      double occupancy_penalty = 0.0;
      if (few_ctas && waves == 1) {
        // a single-wave launch is latency-bound whatever its tiling (split-K's park / arrive / reduce, the fill rate of a CTA
        // of a sparse grid), so equal-latency tilings are resolved by a charge per occupied SM: the sparser grid leaves SMs
        // to the other streams of the pipelined parser
        if (ks > 1) t_split = 5.0 + double(ks) * (128.0 * c * 4.0 / 100000.0);
        if (items < 128) t_kb_ = t_mma > t_fill * 0.7 ? t_mma : t_fill * 0.7;
        occupancy_penalty = cta_penalty * double(items);
      }
      const double per_item = 2.5 + kb_per * t_kb_ + 0.012 * c + t_split;
      const double cost = waves * per_item + occupancy_penalty;
      if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = c; best_ks = ks; }
    }
  }
  *bn_out = best;
  *ksplit_out = best_ks;
}

// What cuTensorMapEncodeTiled is asked to encode: dims (elements), strides of dims 1.. (bytes), box (elements).
struct TmaGeom {
  int rank;
  cuuint64_t dims[5], strides[4];
  cuuint32_t box[5];
  CUtensorMapSwizzle swizzle;   // must span exactly one box row (bk * 2 bytes) and match the wgmma descriptors' layout
  bool f32;                     // fp32 elements (else fp16, or bf16 for bf16 operands)
};
static int swizzle_bytes(CUtensorMapSwizzle s) {
  return s == CU_TENSOR_MAP_SWIZZLE_128B ? 128 : s == CU_TENSOR_MAP_SWIZZLE_64B ? 64 : s == CU_TENSOR_MAP_SWIZZLE_32B ? 32 : 0;
}
static int desc_swizzle_bytes(uint64_t desc_hi) {   // layout field [62,64) of the smem matrix descriptor
  const int layout = int(desc_hi >> 62);
  return layout == 1 ? 128 : layout == 2 ? 64 : layout == 3 ? 32 : 0;
}
// One launch, fully planned on the host: the kernel arguments (minus the split-K workspace, counters and trace buffer,
// which belong to the launching stream), both tensor maps' geometry, the grid and the dynamic shared memory.
struct GemmPlan {
  GemmArgs g;
  TmaGeom ta, tb, tc, tr;   // tc / tr: TMA epilogue output / residual
  int kb_merge, grid;
  size_t smem;
};

// The epilogue, decided after the tiling and the ring: the TMA epilogue (GemmArgs::tma_epi) for direct mode-0 launches with
// 16-byte aligned rows whose staging and residual buffers fit in the shared memory the ring leaves, giving up ring stages
// down to 2 (resident weights: A stages) if needed -- but never an fp16x3 stage: those rings are as deep as their
// k-blocks allow only just.  Otherwise the register epilogue (epi_store16).
static void plan_epilogue(const ConvGemm& d, int max_smem, const GemmKnobs& kn, int stage_bytes, GemmPlan* p) {
  GemmArgs& g = p->g;
  g.epi_bytes = kEpiStageBytes;
  const int esz = d.out_f32 ? 4 : 2, cols = 64 / esz;
  if (kn.no_tma_epi || d.mode != 0 || g.ksplit != 1 || g.park || !g.vec_ok || d.N % (16 / esz) != 0 || g.bn % cols != 0) return;
  const int out_planes = g.split ? 2 : 1, res_planes = !d.res ? 0 : (g.res_lo ? 2 : 1);
  const uint32_t epi_buf = out_planes * kEpiPlane, res_buf = res_planes * kEpiPlane;
  const long long epi_bytes = 2LL * (epi_buf + res_buf);
  const long long need = (long long)p->smem - kEpiStageBytes + epi_bytes - max_smem;   // bytes the ring must give up
  if (need > 0) {
    const long long unit = g.bres ? g.a_slot : stage_bytes;
    const int give = int((need + unit - 1) / unit);
    int& ring = g.bres ? g.stagesA : g.stages;
    if (g.x3 || ring - give < 2) return;
    ring -= give;
    p->smem -= size_t(give) * size_t(unit);
  }
  p->smem += epi_bytes - kEpiStageBytes;
  g.tma_epi = 1;
  g.out_planes = out_planes; g.res_planes = res_planes;
  g.epi_buf = epi_buf; g.res_buf = res_buf; g.epi_bytes = uint32_t(epi_bytes);
  const cuuint64_t N = cuuint64_t(d.N), M = cuuint64_t(d.M);
  const cuuint32_t bc = cuuint32_t(cols);
  // [hi | lo] pairs: one more dimension of size 2, the lo plane at column offset split / res_lo
  p->tc = out_planes == 2 ? TmaGeom{3, {N, M, 2}, {cuuint64_t(d.ldc) * esz, cuuint64_t(g.split) * esz}, {bc, kTileM, 2}}
                          : TmaGeom{2, {N, M}, {cuuint64_t(d.ldc) * esz}, {bc, kTileM}};
  if (res_planes) {
    p->tr = res_planes == 2 ? TmaGeom{3, {N, M, 2}, {cuuint64_t(d.ldr) * esz, cuuint64_t(g.res_lo) * esz}, {bc, kTileM, 2}}
                            : TmaGeom{2, {N, M}, {cuuint64_t(d.ldr) * esz}, {bc, kTileM}};
  }
  p->tc.swizzle = p->tr.swizzle = CU_TENSOR_MAP_SWIZZLE_64B;
  p->tc.f32 = p->tr.f32 = d.out_f32 != 0;
}

// Plans one launch for a device with num_sms SMs and max_smem bytes of opt-in shared memory per block; makes every
// host-side rejection of gemm_launch and touches no device state.  have_ws: a split-K workspace slot is available for the
// launching stream (otherwise K is never split and park-only launches are refused).
static int plan_gemm(const ConvGemm& d, int num_sms, int max_smem, const GemmKnobs& kn, bool have_ws, GemmPlan* p) {
  *p = GemmPlan{};
  GemmArgs& g = p->g;
  TmaGeom& ta = p->ta;
  TmaGeom& tb = p->tb;
  const int Ktot = (d.mode == 0) ? d.K : 9 * d.Cin;
  const int kred = (d.mode == 0) ? d.K : d.Cin;
  // fp16x3 operands always stream 32-wide k-blocks (GemmArgs::x3).  The tiling and split-K choice is still made for 64-wide
  // blocks where K allows them (kb_merge = 2), so split-K slices start at the same K offsets and every sum keeps its order.
  const int bk = (kred % 64 == 0 && !d.x3) ? 64 : 32;
  const int kb_merge = (d.x3 && kred % 64 == 0) ? 2 : 1;
  p->kb_merge = kb_merge;
  if (d.mode != 0 && kred % 32 != 0) return set_error("conv3x3: Cin must be a multiple of 32");
  if (d.mode == 0 && (d.K % 8 != 0 || d.lda % 8 != 0)) return set_error("gemm: K and lda must be multiples of 8");
  if ((reinterpret_cast<uintptr_t>(d.A) & 15) || (reinterpret_cast<uintptr_t>(d.B) & 15)) return set_error("gemm: operands must be 16-byte aligned");
  const bool halo = (d.mode == 1) && !kn.no_halo && (bk == 64 || !kn.no_halo32) && !d.x3;
  if (d.x3 && (kred % bk != 0)) return set_error("gemm: fp16x3 operands need K (Cin) to be a multiple of 32");
  if (d.x3 && d.bf16) return set_error("gemm: fp16x3 operands are fp16");
  const int xk = d.x3 ? 2 : 1;   // operand rows carry [hi | lo]
  g.x3 = d.x3 ? 1 : 0;
  // lo-plane offset of A: [hi(K) | lo(K)] rows by default; a channel slice of a wider [hi(Ctot) | lo(Ctot)] pixel passes Ctot
  const long long lo_a = d.x3 ? (d.lo_a > 0 ? d.lo_a : (long long)kred) : 0;
  const long long a_span = d.x3 ? lo_a + kred : (long long)kred;   // columns of A the tensor map must cover
  if (d.x3 && (lo_a % 8 != 0 || lo_a < kred)) return set_error("gemm: fp16x3 lo-plane offset of A must be a multiple of 8 and >= K");
  g.lo_a = int(lo_a); g.lo_b = kred;
  g.b_tap = xk * d.Cin;
  g.mode = halo ? 3 : d.mode;
  g.N = d.N;
  g.bk = bk;
  g.cin = d.Cin;
  g.desc_hi = make_desc_hi(bk);
  g.out = d.out; g.ldc = d.ldc; g.out_f32 = d.out_f32; g.bias = d.bias; g.res = d.res; g.ldr = d.ldr; g.act = d.act;
  g.split = (d.split_out && !d.out_f32) ? int(d.lo_out > 0 ? d.lo_out : d.N) : 0;
  if (g.split && ((d.N % 8) || (g.split % 8))) return set_error("gemm: split (fp16x3) output needs N % 8 == 0 and an 8-aligned lo-plane offset");
  if (g.split && (g.split < d.N || d.ldc < (long long)g.split + d.N)) return set_error("gemm: split (fp16x3) output rows are [hi(N) .. | lo(N) ..]: ldc must be >= lo offset + N");
  g.res_lo = (d.res && !d.out_f32 && d.lo_res > 0) ? int(d.lo_res) : 0;
  if (g.res_lo % 8) return set_error("gemm: residual lo-plane offset must be a multiple of 8");

  if (d.mode == 0) {
    g.M = d.M;
    g.tw_valid = 0;
    g.num_kb = (d.K + bk - 1) / bk;
    g.m_tiles = (d.M + kTileM - 1) / kTileM;
    g.a_bytes = kTileM * bk * 2;
    if (d.x3 && d.lda < a_span) return set_error("gemm: fp16x3 A rows are [hi(K) .. | lo(K) ..]: lda must be >= lo offset + K");
    ta = TmaGeom{2, {cuuint64_t(a_span), cuuint64_t(d.M)}, {cuuint64_t(d.lda) * 2}, {cuuint32_t(bk), cuuint32_t(kTileM)}};
  } else {
    const int s = (d.mode == 2) ? 2 : 1;
    if (s == 2 && ((d.H & 1) || (d.W & 1))) return set_error("conv3x3 s2: H and W must be even");
    if (d.lda % 8 != 0) return set_error("conv3x3: input pixel stride must be a multiple of 8 channels");
    if (d.x3 && d.lda < a_span) return set_error("conv3x3: fp16x3 pixels are [hi(Cin) .. | lo(Cin) ..]: pixel stride must be >= lo offset + Cin");
    g.Ho = d.H / s; g.Wo = d.W / s; g.batch = d.batch;
    g.cin_blocks = d.Cin / bk;
    g.num_kb = 9 * g.cin_blocks;
    // spatial tile tw x th <= 128 output pixels: maximise useful rows per 128-row MMA tile
    int btw = 1, bth = 1; double bu = -1;
    for (int tw = 1; tw <= g.Wo && tw <= 128; ++tw) {
      int th = 128 / tw; if (th > g.Ho) th = g.Ho; if (th < 1) continue;
      const long tiles = long((g.Wo + tw - 1) / tw) * ((g.Ho + th - 1) / th);
      const double u = double(g.Ho) * g.Wo / (double(tiles) * 128.0);
      if (u > bu + 1e-9 || (u > bu - 1e-9 && tw > btw)) { bu = u; btw = tw; bth = th; }
    }
    if (halo) {
      // halo tile: (th+2) x (tw+2) input pixels loaded once per 64-channel block; the 128 MMA rows are 128 consecutive
      // positions of that tile (row pitch tw+2), so 2 of every tw+2 rows are halo columns and carry no output.
      btw = 1; bth = 1; bu = -1;
      for (int tw = 1; tw <= g.Wo && tw <= 126; ++tw) {
        int th = 128 / (tw + 2); if (th > g.Ho) th = g.Ho; if (th < 1) continue;
        const long tiles = long((g.Wo + tw - 1) / tw) * ((g.Ho + th - 1) / th);
        const double u = double(g.Ho) * g.Wo / (double(tiles) * 128.0);
        if (u > bu + 1e-9 || (u > bu - 1e-9 && tw > btw)) { bu = u; btw = tw; bth = th; }
      }
      g.tw = btw + 2; g.tw_valid = btw; g.th = bth;
      g.num_kb = g.cin_blocks;                                  // pipeline unit = one channel block (9 taps)
      g.a_bytes = uint32_t(bth + 2) * (btw + 2) * uint32_t(2 * bk);
      g.a_slot = (uint32_t(2 * (btw + 2) + 2 + 128) * uint32_t(2 * bk) + 1023) & ~1023u;
    } else {
      g.tw = btw; g.tw_valid = btw; g.th = bth;
      g.a_bytes = uint32_t(btw) * bth * bk * 2;
    }
    g.nb = 1;
    g.tiles_x = (g.Wo + btw - 1) / btw; g.tiles_y = (g.Ho + bth - 1) / bth;
    if (!halo && g.tiles_x == 1 && g.tiles_y == 1 && btw == g.Wo && bth == g.Ho && btw * bth * 2 <= 128 && d.batch > 1) {
      // tiny maps (DaViT stages at 64x64 crops: 8x8, 4x4, 2x2 outputs): one TMA box spans nb whole images so the 128
      // MMA rows are full instead of 64/16/4 valid ones
      int nb = 128 / (btw * bth);
      if (nb > d.batch) nb = d.batch;
      g.nb = nb;
      g.a_bytes *= uint32_t(nb);
    }
    g.m_tiles = (g.nb > 1) ? (d.batch + g.nb - 1) / g.nb : g.tiles_x * g.tiles_y * d.batch;
    const cuuint64_t ld = cuuint64_t(d.lda);
    if (halo) {
      ta = TmaGeom{4, {cuuint64_t(d.Cin), cuuint64_t(d.W), cuuint64_t(d.H), cuuint64_t(d.batch)}, {ld * 2, ld * 2 * d.W, ld * 2 * d.W * d.H},
                   {cuuint32_t(bk), cuuint32_t(btw + 2), cuuint32_t(bth + 2), 1}};
    } else if (d.mode == 1) {
      ta = TmaGeom{4, {cuuint64_t(a_span), cuuint64_t(d.W), cuuint64_t(d.H), cuuint64_t(d.batch)}, {ld * 2, ld * 2 * d.W, ld * 2 * d.W * d.H},
                   {cuuint32_t(bk), cuuint32_t(btw), cuuint32_t(bth), cuuint32_t(g.nb)}};
    } else {
      // (x parity, channel) merged in dim0: element (n, 2*yo+py, 2*xo+px, c) at c + px*ld  (+ xo*2ld + py*W*ld + yo*2W*ld)
      g.ldpar = int(d.lda);   // producer adds px * ldA to the channel coordinate
      ta = TmaGeom{5, {ld + cuuint64_t(a_span), cuuint64_t(d.W / 2), 2, cuuint64_t(d.H / 2), cuuint64_t(d.batch)},
                   {ld * 4, ld * 2 * d.W, ld * 4 * d.W, ld * 2 * d.W * d.H}, {cuuint32_t(bk), cuuint32_t(btw), 1, cuuint32_t(bth), cuuint32_t(g.nb)}};
    }
  }
  int bn = 16, ksplit = 1;
  pick_tiling(d.N, g.m_tiles, g.num_kb / kb_merge, (halo ? 9 * bk : bk) * kb_merge, g.a_bytes * kb_merge, d.bn_max > 0 ? d.bn_max : 256,
              have_ws, d.x3 != 0, num_sms, max_smem, kn, &bn, &ksplit);
  // Resident weights: one N tile, no split-K, at least one full wave of M tiles, and the whole weight matrix + a >= 2-deep
  // A ring must fit in shared memory (see GemmArgs::bres).
  bool bres = false;
  int res_slots = 0, res_stagesA = 0;
  const uint32_t a_slot_sep = halo ? g.a_slot : uint32_t(kASlot);
  if (!kn.no_bres && !d.x3 && d.N <= 256 && g.m_tiles >= num_sms && (d.bn_max <= 0 || d.bn_max >= d.N)) {
    static const int cand[] = {16, 32, 48, 64, 96, 128, 192, 256};
    int bnr = 256;
    for (int c : cand) if (c >= d.N) { bnr = c; break; }
    const uint32_t bslot = (uint32_t(bnr) * bk * 2 + 1023) & ~1023u;
    res_slots = halo ? g.cin_blocks * 9 : g.num_kb;
    const long long bar_bytes = 8LL * (2 * res_slots + 4 + 2 * 8) + 64;
    const long long avail = (long long)max_smem - 1024 - kEpiStageBytes - ((bar_bytes + 1023) & ~1023LL) - (long long)res_slots * bslot;
    if (avail >= 2LL * a_slot_sep) {
      bres = true;
      bn = bnr;
      ksplit = 1;
      res_stagesA = int(avail / a_slot_sep);
      if (res_stagesA > 8) res_stagesA = 8;
    }
  }
  if (d.park) {
    if (d.mode != 0 || !have_ws) return set_error("gemm (park-only): needs mode 0 and a split-K workspace slot for this stream");
    if (size_t(g.m_tiles) * ((d.N + bn - 1) / bn) * ksplit * 128 * bn * 4 > kWsBytes) return set_error("gemm (park-only): partial tiles exceed the workspace");
    bres = false;
  }
  g.park = d.park ? 1 : 0;
  g.bres = bres ? 1 : 0;
  g.sep = (halo || bres) ? 1 : 0;
  g.taps = halo ? 9 : 1;
  g.bn = bn;
  g.sk_last = kn.sk_last ? 1 : 0;
  g.ksplit = ksplit;
  g.kb_per = kb_merge * ((g.num_kb / kb_merge + ksplit - 1) / ksplit);
  g.n_tiles = (d.N + bn - 1) / bn;
  // co-scheduled CTAs should share the LARGER operand through L2: weights bigger than activations -> M tiles fastest
  g.mt_fast = (d.mode == 0 && g.m_tiles > 1 && (long long)d.N > (long long)d.M) ? 1 : 0;
  g.b_bytes = uint32_t(bn) * bk * 2;
  g.b_slot = (g.b_bytes + 1023) & ~1023u;
  g.bf16 = d.bf16 ? 1 : 0;
  tb = TmaGeom{2, {cuuint64_t(xk) * cuuint64_t(Ktot), cuuint64_t(d.N)}, {cuuint64_t(xk) * cuuint64_t(Ktot) * 2}, {cuuint32_t(bk), cuuint32_t(bn)}};
  ta.swizzle = tb.swizzle = (bk == 64) ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  g.d_ksplit = FastDiv::make(g.ksplit); g.d_ntiles = FastDiv::make(g.n_tiles); g.d_mtiles = FastDiv::make(g.m_tiles);
  g.d_perimg = FastDiv::make(d.mode != 0 ? g.tiles_x * g.tiles_y : 1); g.d_tilesx = FastDiv::make(d.mode != 0 ? g.tiles_x : 1);
  g.d_cinb = FastDiv::make(d.mode != 0 ? g.cin_blocks : 1);
  if (!g.sep) g.a_slot = uint32_t(kTileM) * bk * 2;     // single ring: one A half per slot
  const int stage_bytes = g.sep ? int(g.b_slot) : xk * (int(g.a_slot) + int(g.b_slot));
  int stages, bar_space = 512;
  if (bres) {
    g.a_slot = a_slot_sep;
    g.stagesA = res_stagesA;
    stages = res_slots;                                   // every B k-block (x tap) owns a slot for the whole launch
    bar_space = int((8LL * (2 * stages + 4 + 2 * g.stagesA) + 64 + 1023) & ~1023LL);
  } else if (halo) {
    // B ring first (up to 8 taps in flight), then as deep an A ring as fits (2..4 halo tiles)
    stages = (max_smem - 1024 - 512 - kEpiStageBytes - 2 * int(g.a_slot)) / stage_bytes;
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages < 2) stages = 2;
    int sa = (max_smem - 1024 - 512 - kEpiStageBytes - stages * stage_bytes) / int(g.a_slot);
    g.stagesA = sa > 4 ? 4 : (sa < 2 ? 2 : sa);
  } else {
    g.stagesA = 0;
    stages = (max_smem - 1024 - 512 - kEpiStageBytes) / stage_bytes;
    if (stages > kMaxStages) stages = kMaxStages;
    if (stages > g.kb_per && g.kb_per >= 2 && g.ksplit == 1) stages = g.kb_per;
    if (stages < 2) stages = 2;
  }
  const int a_region = g.sep ? g.stagesA * int(g.a_slot) : 0;
  g.stages = stages;
  p->smem = size_t(a_region) + size_t(stages) * stage_bytes + 1024 + kEpiStageBytes + bar_space;
  if (p->smem > size_t(max_smem)) return set_error("gemm: internal error, shared-memory plan exceeds the device limit");
  // vector epilogue needs 16-byte aligned rows in out / residual and bias
  const int esz = d.out_f32 ? 4 : 2;
  g.vec_ok = ((reinterpret_cast<uintptr_t>(d.out) & 15) == 0) && ((d.ldc * esz) % 16 == 0) &&
             (!d.res || (((reinterpret_cast<uintptr_t>(d.res) & 15) == 0) && ((d.ldr * esz) % 16 == 0))) &&
             (!d.bias || ((reinterpret_cast<uintptr_t>(d.bias) & 15) == 0));
  plan_epilogue(d, max_smem, kn, stage_bytes, p);
  const int total = g.m_tiles * g.n_tiles * g.ksplit;
  int grid = total < num_sms ? total : num_sms;
  if (kn.max_grid > 0 && grid > kn.max_grid && ksplit == 1) grid = kn.max_grid;
  p->grid = grid;
  return 0;
}

static int encode(CUtensorMap* m, int bf16, const TmaGeom& t, const void* base) {
  const CUtensorMapDataType dt = t.f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  return encode(m, dt, t.rank, base, t.dims, t.strides, t.box, t.swizzle);
}

static void plan_fields(const GemmPlan& p, int* out);
// the plan of the calling thread's most recent launch (b2p_gemm_last_plan): the one actually launched, after the stream's
// split-K workspace slot was looked up
static thread_local int t_last_plan[kGemmPlanFields];
static thread_local bool t_have_last_plan = false;

int gemm_launch(const ConvGemm& d, cudaStream_t st) {
  if (int e = device_setup()) return e;
  const GemmKnobs& kn = gemm_knobs();
  const int slot = (kn.no_split || d.no_split) ? -1 : ws_slot_for(st);
  GemmPlan p;
  if (int e = plan_gemm(d, g_num_sms, g_max_smem, kn, slot >= 0, &p)) return e;
  GemmArgs& g = p.g;
  g.ws = slot >= 0 ? g_ws[slot] : nullptr;
  g.counters = slot >= 0 ? g_counters[slot] : nullptr;
  CUtensorMap tmA, tmB, tmC{}, tmR{};
  if (int e = encode(&tmA, d.bf16, p.ta, d.A)) return e;
  if (int e = encode(&tmB, d.bf16, p.tb, d.B)) return e;
  if (g.tma_epi) {
    if (int e = encode(&tmC, 0, p.tc, d.out)) return e;
    if (g.res_planes)
      if (int e = encode(&tmR, 0, p.tr, d.res)) return e;
  }
  const int grid = p.grid, bn = g.bn, ksplit = g.ksplit;
  const int Ktot = (d.mode == 0) ? d.K : 9 * d.Cin;
  static const bool dbg = getenv("B2P_DEBUG") != nullptr;
  static const bool no_pdl = getenv("B2P_NO_PDL") != nullptr;
  if (grid <= 0) return 0;
  if (dbg)
    fprintf(stderr, "b2p_gemm mode=%d M=%d N=%d Ktot=%d bk=%d bn=%d tw=%d th=%d m_tiles=%d n_tiles=%d stages=%d grid=%d act=%d f32=%d res=%d ksplit=%d x3=%d bres=%d stagesA=%d\n",
            g.mode, d.mode == 0 ? d.M : g.m_tiles * 128, d.N, Ktot, g.bk, bn, g.tw, g.th, g.m_tiles, g.n_tiles, g.stages, grid,
            d.act, d.out_f32, d.res != nullptr, ksplit, g.x3, g.bres, g.stagesA);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = p.smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = no_pdl ? 0 : 1;
  if (g_trace && grid <= kTraceCtas) {
    std::lock_guard<std::mutex> lk(g_trace_mu);
    if (g_trace_n < kTraceCap) {
      const int m[8] = {g.mode, d.mode == 0 ? d.M : g.m_tiles * 128, d.N, Ktot, bn, ksplit, g.x3, grid};
      for (int i = 0; i < 8; ++i) g_trace_meta[g_trace_n][i] = m[i];
      g.trace = g_trace + size_t(g_trace_n) * kTraceCtas * kTraceSlots;
      ++g_trace_n;
    }
  }
  GemmKernel kern = nullptr;
  for (int i = 0; i < kNumBn; ++i) if (kBnCand[i] == bn) kern = kGemmKernels[i][g.tma_epi];
  if (!kern) return set_error("gemm: internal error, no kernel instantiation for the chosen N tile");
  cudaError_t ce = cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, tmR, g);
  if (ce == cudaSuccess) ce = cudaGetLastError();
  if (ce != cudaSuccess) return set_error(cudaGetErrorString(ce));
  count_launch();
  plan_fields(p, t_last_plan);
  t_have_last_plan = true;
  if (d.park_info) {
    d.park_info->ws = g.ws; d.park_info->bn = bn; d.park_info->ksplit = g.ksplit; d.park_info->n_tiles = g.n_tiles;
    d.park_info->m_tiles = g.m_tiles; d.park_info->mt_fast = g.mt_fast;
  }
  return 0;
}

// Elements from a tensor map's base pointer up to one past the last element it can address.
static long long tma_extent(const TmaGeom& t) {
  long long e = (long long)t.dims[0];
  for (int i = 1; i < t.rank; ++i) e += (long long)(t.dims[i] - 1) * (long long)(t.strides[i - 1] / 2);
  return e;
}

static void plan_fields(const GemmPlan& p, int* out) {
  const GemmArgs& g = p.g;
  auto sat = [](long long v) { return int(v > 0x7fffffffLL ? 0x7fffffffLL : v); };
  const int f[] = {g.mode, g.bk, g.bn, g.ksplit, g.kb_per, p.kb_merge, g.stages, g.stagesA, g.sep, g.bres, g.nb, g.tw, g.tw_valid,
                   g.th, g.m_tiles, g.n_tiles, g.mt_fast, p.grid, int(p.smem), g.vec_ok, g.split, g.res_lo, g.park,
                   g.x3, g.num_kb, g.taps, int(g.a_bytes), int(g.a_slot), int(g.b_bytes), int(g.b_slot), g.tiles_x, g.tiles_y,
                   p.ta.rank, int(p.ta.box[0]), int(p.ta.box[1]), int(p.ta.box[2]), int(p.ta.box[3]), int(p.ta.box[4]),
                   int(p.tb.box[0]), int(p.tb.box[1]), sat(tma_extent(p.ta)), sat(tma_extent(p.tb)),
                   swizzle_bytes(p.ta.swizzle), swizzle_bytes(p.tb.swizzle), desc_swizzle_bytes(g.desc_hi)};
  static_assert(sizeof(f) / sizeof(f[0]) == kGemmPlanFields, "b2p_gemm_plan field count");
  for (int i = 0; i < kGemmPlanFields; ++i) out[i] = f[i];
}

// Host-only planner (b2p_gemm_plan): see include/b200parse.h for the field order of `out`.  The plan assumes the launching
// stream owns a split-K workspace slot (gemm_launch plans without split-K once kWsSlots streams own one).
int gemm_plan_host(const ConvGemm& d, int num_sms, int max_smem, int* out) {
  if (num_sms < 1 || max_smem < 1) return set_error("gemm_plan: num_sms and max_smem must be positive");
  const GemmKnobs& kn = gemm_knobs();
  GemmPlan p;
  if (int e = plan_gemm(d, num_sms, max_smem, kn, !(kn.no_split || d.no_split), &p)) return e;
  plan_fields(p, out);
  return 0;
}

// Host-only epilogue planner (b2p_gemm_epilogue_plan): see include/b200parse.h for the field order of `out`.
int gemm_epilogue_plan_host(const ConvGemm& d, int num_sms, int max_smem, int* out) {
  if (num_sms < 1 || max_smem < 1) return set_error("gemm_plan: num_sms and max_smem must be positive");
  const GemmKnobs& kn = gemm_knobs();
  GemmPlan p;
  if (int e = plan_gemm(d, num_sms, max_smem, kn, !(kn.no_split || d.no_split), &p)) return e;
  const GemmArgs& g = p.g;
  auto sat = [](cuuint64_t v) { return int(v > 0x7fffffffULL ? 0x7fffffffULL : v); };
  const int cols = d.out_f32 ? 16 : 32;
  const int f[] = {g.tma_epi, g.tma_epi ? cols : 0, g.tma_epi ? g.bn / cols : 0, g.tma_epi ? 2 : 0, g.out_planes,
                   g.tma_epi && g.res_planes ? 2 : 0, g.res_planes, int(g.epi_bytes), g.stages, g.stagesA, int(p.smem),
                   p.tc.rank, int(p.tc.box[0]), int(p.tc.box[1]), int(p.tc.box[2]), sat(p.tc.strides[0]), sat(p.tc.strides[1]),
                   p.tr.rank, int(p.tr.box[0]), int(p.tr.box[1]), int(p.tr.box[2]), sat(p.tr.strides[0]), sat(p.tr.strides[1]),
                   swizzle_bytes(p.tc.swizzle)};
  static_assert(sizeof(f) / sizeof(f[0]) == kEpiPlanFields, "b2p_gemm_epilogue_plan field count");
  for (int i = 0; i < kEpiPlanFields; ++i) out[i] = f[i];
  return 0;
}

int gemm_last_plan(int* out) {
  if (!t_have_last_plan) return set_error("gemm_last_plan: this thread has launched no GEMM/conv");
  for (int i = 0; i < kGemmPlanFields; ++i) out[i] = t_last_plan[i];
  return 0;
}

// -> number of traced launches since the last call; stamps [n][kTraceCtas = 160][16] (ns, 0 = not written), meta [n][8] =
// {mode, M, N, K, bn, ksplit, x3, grid}.  Synchronises the device.
int trace_read(unsigned long long* stamps, int* meta, int max_launches) {
  if (!g_trace) return set_error("tracing is off (set B2P_TRACE=1 before the first GEMM launch)");
  cudaDeviceSynchronize();
  std::lock_guard<std::mutex> lk(g_trace_mu);
  const int n = g_trace_n < max_launches ? g_trace_n : max_launches;
  const size_t per = size_t(kTraceCtas) * kTraceSlots;
  if (n > 0 && cudaMemcpy(stamps, g_trace, sizeof(unsigned long long) * per * n, cudaMemcpyDeviceToHost) != cudaSuccess)
    return set_error("trace_read: copy failed");
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 8; ++j) meta[i * 8 + j] = g_trace_meta[i][j];
  cudaMemset(g_trace, 0, sizeof(unsigned long long) * per * kTraceCap);
  g_trace_n = 0;
  return n;
}

// ------------------------------------------------------------------------ streams and their split-K workspace slots
int stream_create(cudaStream_t* out) {
  if (!out) return set_error("stream_create: out is null");
  if (int e = bind_device()) return e;
  if (cudaStreamCreateWithFlags(out, cudaStreamNonBlocking) != cudaSuccess) return set_error("cudaStreamCreateWithFlags failed");
  return 0;
}

int stream_destroy(cudaStream_t st) {
  if (!st) return set_error("stream_destroy: the default stream is not destroyed");
  // the slot is released under the lock before the handle can be reused by a new stream
  std::lock_guard<std::mutex> lk(g_ws_mu);
  const int i = ws_slot_locked(st);
  if (i >= 0) { g_ws_taken[i] = false; g_ws_owner[i] = nullptr; }
  if (cudaStreamDestroy(st) != cudaSuccess) return set_error("cudaStreamDestroy failed");
  return 0;
}

int ws_slot(cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_ws_mu);
  return ws_slot_locked(st);
}

// Every split-K launch leaves its tiles' arrival counters at zero (the last CTA of a tile resets them), so with the device
// idle a non-zero counter word is a launch that did not complete its reduction, or two launches that shared a slot.
int ws_audit(int* nonzero_host, int max_slots) {
  if (!nonzero_host && max_slots > 0) return set_error("ws_audit: nonzero_host is null");
  if (int e = bind_device()) return e;
  if (cudaDeviceSynchronize() != cudaSuccess) return set_error("ws_audit: cudaDeviceSynchronize failed");
  static int words[2 * kMaxCounterTiles];
  std::lock_guard<std::mutex> lk(g_ws_mu);
  for (int i = 0; i < kWsSlots && i < max_slots; ++i) {
    nonzero_host[i] = -1;
    if (!g_ws_taken[i]) continue;
    if (cudaMemcpy(words, g_counters[i], sizeof words, cudaMemcpyDeviceToHost) != cudaSuccess)
      return set_error("ws_audit: counter copy failed");
    int n = 0;
    for (int w = 0; w < 2 * kMaxCounterTiles; ++w) n += words[w] != 0;
    nonzero_host[i] = n;
  }
  return kWsSlots;
}

}  // namespace b2p
