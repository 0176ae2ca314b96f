// Lossless PNG of the annotated Set-of-Marks frame (8-bit RGB) on the device: the encode that ends get_som_labeled_img
// (ref:util/utils.py:493-494, PIL's Image.save(format="PNG")), SURVEY.md 8f.
//
// Stream layout (the pigz construction, as the host encoder som_overlay.encode_png writes it): every row gets the Up
// filter; the filtered rows are cut into bands of whole rows (about 32 KiB each); each band is deflated on its own and
// ends byte-aligned -- a dynamic-Huffman block followed by an empty stored block (sync flush), or, when smaller, stored
// blocks; the last band sets BFINAL.  The concatenation is one zlib stream inside one IDAT chunk.  Back-references may
// reach into earlier bands (their bytes are already in the decoder's window).
//
// Four launches on the caller's stream:
//   png_filter_kernel   rgb -> filtered rows (filter byte 2, then Raw(x) - Prior(x) mod 256)
//   png_band_kernel     one CTA per band: LZ77 match finding (a hash table of the band's earlier positions, same-key lanes
//                       of the warp, the previous byte / pixel / row, all checked by direct comparison), a greedy parse with
//                       one-step lazy matching, the Adler-32 partial sums,
//                       length-limited Huffman codes, and the band's bytes written into its workspace slot
//   png_place_kernel    one CTA per band: the band's output offset (sum of the earlier bands' sizes), the copy behind the
//                       zlib header, and the band's CRC-32
//   png_finish_kernel   signature, IHDR, IDAT length, zlib header, Adler-32 (combined across bands), IDAT CRC (band CRCs
//                       combined with the x^(8n) mod P "zeros" operator, as zlib's crc32_combine), IEND, total length
//
// The worst case is every band stored, so the output bound and the workspace follow from H and W alone (png_plan).
#include <cuda_runtime.h>
#include <stdint.h>

#include "b2p_internal.h"

namespace b2p {

static constexpr int kPngThreads = 256;
static constexpr int kPngBandTarget = 32768;   // filtered bytes per band (whole rows, at least one)
static constexpr int kHashBits = 13;
static constexpr int kWindow = 32768;
static constexpr int kMaxMatch = 258;
static constexpr int kStoredMax = 65535;
static constexpr long long kHeadBytes = 43;     // signature 8, IHDR 25, IDAT length + tag 8, zlib header 2
static constexpr long long kTailBytes = 20;     // Adler-32 4, IDAT CRC 4, IEND 12
static constexpr unsigned kAdlerMod = 65521u;
static constexpr unsigned kCrcPoly = 0xedb88320u;

struct PngPlan {
  long long pitch, rows_per_band, bands, band_bytes, last_bytes;   // filtered bytes per row / band / last band
  long long stage_stride;                                          // workspace slot per band (bytes, multiple of 16)
  long long filt_off, tok_off, stage_off, info_off, ws_bytes, out_bytes;
};

struct BandInfo {          // per band, in the workspace
  long long out_bytes;     // bytes the band contributes to the zlib stream
  long long offset;        // its offset behind the zlib header (png_place_kernel)
  unsigned adler_a, adler_b, crc, pad;
};

__host__ __device__ static long long stored_bytes(long long n) { return n + 5 * ((n + kStoredMax - 1) / kStoredMax); }
static long long align_up(long long v, long long a) { return (v + a - 1) / a * a; }

// Host-side plan: band geometry, workspace layout, worst-case output.  Returns -1 (with the message recorded) when H or W
// is < 1 or the worst case does not fit one IDAT chunk (length <= 2^31 - 1).
static int png_plan(int H, int W, PngPlan* p) {
  if (H < 1 || W < 1) return set_error("b2p_png: H and W must be >= 1");
  p->pitch = 1 + 3LL * W;
  p->rows_per_band = p->pitch >= kPngBandTarget ? 1 : kPngBandTarget / p->pitch;
  if (p->rows_per_band > H) p->rows_per_band = H;
  p->bands = (H + p->rows_per_band - 1) / p->rows_per_band;
  p->band_bytes = p->rows_per_band * p->pitch;
  p->last_bytes = (H - (p->bands - 1) * p->rows_per_band) * p->pitch;
  const long long stream = (p->bands - 1) * stored_bytes(p->band_bytes) + stored_bytes(p->last_bytes);
  if (2 + stream + 4 > 2147483647LL) return set_error("b2p_png: the frame's worst-case IDAT exceeds 2^31 - 1 bytes");
  p->out_bytes = kHeadBytes + stream + kTailBytes;
  const long long filt = (long long)H * p->pitch;
  p->stage_stride = align_up(stored_bytes(p->band_bytes), 16);
  p->filt_off = 0;
  p->tok_off = align_up(filt + 16, 256);
  p->stage_off = p->tok_off + align_up(4 * filt, 256);
  p->info_off = p->stage_off + align_up(p->bands * p->stage_stride, 256);
  p->ws_bytes = p->info_off + align_up(p->bands * (long long)sizeof(BandInfo), 256);
  return 0;
}

// ------------------------------------------------------------------------------------------------------------ device code

__global__ void png_filter_kernel(const unsigned char* __restrict__ rgb, int H, int W, unsigned char* __restrict__ filt) {
  const long long pitch = 1 + 3LL * W, n = (long long)H * pitch, row = 3LL * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long y = i / pitch, c = i - y * pitch;
    unsigned char v = 2;
    if (c) {
      v = rgb[y * row + c - 1];
      if (y) v = (unsigned char)(v - rgb[(y - 1) * row + c - 1]);
    }
    filt[i] = v;
  }
}

// bytes of a[0..max) equal to b[0..max) from the start (a > b, both inside the filtered stream)
__device__ __forceinline__ int match_len(const unsigned char* __restrict__ f, long long a, long long b, int max) {
  int n = 0;
  while (n < max && f[a + n] == f[b + n]) ++n;
  return n;
}

__host__ __device__ __forceinline__ long long lmin(long long a, long long b) { return a < b ? a : b; }

// deflate length code (257..285) and extra bits of a match length 3..258
__device__ __forceinline__ void len_code(int len, int* code, int* nextra, int* extra) {
  const int l = len - 3;
  if (l < 8) { *code = 257 + l; *nextra = 0; *extra = 0; return; }
  if (l == 255) { *code = 285; *nextra = 0; *extra = 0; return; }
  const int nb = 31 - __clz(l);
  *code = 257 + 4 * (nb - 1) + ((l >> (nb - 2)) & 3);
  *nextra = nb - 2;
  *extra = l & ((1 << (nb - 2)) - 1);
}

// deflate distance code (0..29) and extra bits of a distance 1..32768
__device__ __forceinline__ void dist_code(int dist, int* code, int* nextra, int* extra) {
  const int d = dist - 1;
  if (d < 4) { *code = d; *nextra = 0; *extra = 0; return; }
  const int nb = 31 - __clz(d);
  *code = 2 * nb + ((d >> (nb - 1)) & 1);
  *nextra = nb - 1;
  *extra = d & ((1 << (nb - 1)) - 1);
}

// Huffman code lengths <= limit for freq[0..n) (n <= 286), one thread.  Symbols with freq 0 get length 0; if fewer than
// two symbols are used, symbols 0 / 1 are added with weight 1 so the code is complete (zlib's inflate accepts a lone
// one-bit code only for distances).  sorted / A: scratch of n entries.  Optimal lengths by Moffat and Katajainen's
// in-place algorithm over the frequency-sorted symbols, then the Kraft sum is restored at the limit by moving leaves.
__device__ void huff_lengths(const unsigned* freq, int n, int limit, unsigned char* lens, int* sorted, unsigned* A) {
  int m = 0;
  for (int s = 0; s < n; ++s) { lens[s] = 0; if (freq[s]) sorted[m++] = s; }
  for (int s = 0; m < 2 && s < n; ++s) {
    bool have = false;
    for (int i = 0; i < m; ++i) have |= sorted[i] == s;
    if (!have) sorted[m++] = s;
  }
  // insertion sort by (weight, symbol); m <= 286
  for (int i = 1; i < m; ++i) {
    const int s = sorted[i];
    const unsigned w = freq[s] ? freq[s] : 1u;
    int j = i - 1;
    while (j >= 0) {
      const int t = sorted[j];
      const unsigned wt = freq[t] ? freq[t] : 1u;
      if (wt < w || (wt == w && t < s)) break;
      sorted[j + 1] = t; --j;
    }
    sorted[j + 1] = s;
  }
  for (int i = 0; i < m; ++i) A[i] = freq[sorted[i]] ? freq[sorted[i]] : 1u;
  // phase 1: internal node weights and parent pointers
  A[0] += A[1];
  int root = 0, leaf = 2;
  for (int next = 1; next < m - 1; ++next) {
    if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; }
    else A[next] = A[leaf++];
    if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; }
    else A[next] += A[leaf++];
  }
  // phase 2: internal node depths
  A[m - 2] = 0;
  for (int next = m - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
  // phase 3: leaf depths
  int avail = 1, used = 0, depth = 0, next = m - 1;
  root = m - 2;
  while (avail > 0) {
    while (root >= 0 && (int)A[root] == depth) { ++used; --root; }
    while (avail > used) { A[next--] = depth; --avail; }
    avail = 2 * used; ++depth; used = 0;
  }
  // A[i] is now the length of sorted[i] (non-increasing in i).  Limit: fold longer codes to the limit, then split
  // shorter leaves until the Kraft sum is exactly 1 again.
  int count[33];
  for (int l = 0; l < 33; ++l) count[l] = 0;
  for (int i = 0; i < m; ++i) count[A[i] > (unsigned)limit ? limit : A[i]]++;
  unsigned long long total = 0;
  for (int l = 1; l <= limit; ++l) total += (unsigned long long)count[l] << (limit - l);
  while (total > (1ull << limit)) {
    count[limit]--;
    for (int l = limit - 1; l > 0; --l)
      if (count[l]) { count[l]--; count[l + 1] += 2; break; }
    total--;
  }
  // least frequent symbols get the longest codes
  int i = 0;
  for (int l = limit; l >= 1; --l)
    for (int k = 0; k < count[l]; ++k) lens[sorted[i++]] = (unsigned char)l;
}

// canonical codes, bit-reversed for LSB-first output
__device__ void huff_codes(const unsigned char* lens, int n, unsigned short* codes) {
  int bl[16] = {0}, next[16];
  for (int s = 0; s < n; ++s) bl[lens[s]]++;
  bl[0] = 0;
  int code = 0;
  for (int l = 1; l < 16; ++l) { code = (code + bl[l - 1]) << 1; next[l] = code; }
  for (int s = 0; s < n; ++s) {
    const int l = lens[s];
    if (!l) { codes[s] = 0; continue; }
    codes[s] = (unsigned short)(__brev((unsigned)next[l]++) >> (32 - l));
  }
}

__device__ __forceinline__ void put_bits(unsigned* buf, unsigned long long pos, unsigned v, int n) {
  if (!n) return;
  const unsigned long long w = pos >> 5;
  const int s = (int)(pos & 31);
  atomicOr(buf + w, v << s);
  if (s + n > 32) atomicOr(buf + w + 1, v >> (32 - s));
}

// tokens: literal byte (bit 31 clear) or match: bit 31 | (dist - 1) << 8 | (len - 3)
static constexpr unsigned kMatchBit = 0x80000000u;

__global__ void __launch_bounds__(kPngThreads) png_band_kernel(const unsigned char* __restrict__ filt, PngPlan p,
                                                              unsigned* __restrict__ tok_all, unsigned char* __restrict__ stage_all,
                                                              BandInfo* __restrict__ info) {
  __shared__ int table[1 << kHashBits];
  __shared__ unsigned short c_len[kPngThreads], c_dist[kPngThreads];
  __shared__ unsigned char c_byte[kPngThreads];
  __shared__ unsigned lfreq[286], dfreq[30], cfreq[19];
  __shared__ unsigned char llen[286 + 30], clen[19];
  __shared__ unsigned short lcode[286], dcode[30], ccode[19];
  __shared__ unsigned char rle_sym[286 + 30], rle_extra[286 + 30];
  __shared__ int sort_scratch[286];
  __shared__ unsigned a_scratch[286];
  __shared__ unsigned long long red_a[kPngThreads / 32], red_b[kPngThreads / 32];
  __shared__ long long s_pos, s_ntok, s_extra_bits;
  __shared__ int s_hlit, s_hdist, s_hclen, s_nrle, s_stored;
  __shared__ unsigned long long s_header_bits, s_bits;
  __shared__ unsigned long long s_scan[kPngThreads];

  const int tid = threadIdx.x;
  const long long band = blockIdx.x;
  const bool last = band == p.bands - 1;
  const long long bs = band * p.band_bytes;
  const long long n = last ? p.last_bytes : p.band_bytes;
  const long long be = bs + n;
  unsigned* tok = tok_all + bs;
  unsigned char* stage = stage_all + band * p.stage_stride;

  for (int i = tid; i < (1 << kHashBits); i += kPngThreads) table[i] = -1;
  for (int i = tid; i < 286; i += kPngThreads) lfreq[i] = 0;
  if (tid < 30) dfreq[tid] = 0;
  if (tid < 19) cfreq[tid] = 0;
  if (tid == 0) { s_pos = bs; s_ntok = 0; s_extra_bits = 0; }
  __syncthreads();

  unsigned long long sum_a = 0, sum_b = 0;   // Adler-32 partial sums of this thread's bytes (band-relative weights)
  for (long long base = bs; base < be; base += kPngThreads) {
    const long long q = base + tid;
    int best = 0, bdist = 0, h = -1;
    if (q < be) {
      const unsigned x = filt[q];
      c_byte[tid] = (unsigned char)x;
      sum_a += x;
      sum_b += (unsigned long long)x * (unsigned long long)(be - q);
      const int maxl = (int)lmin(kMaxMatch, be - q);
      if (maxl >= 3) {
        const unsigned key = x | (unsigned)filt[q + 1] << 8 | (unsigned)filt[q + 2] << 16;
        h = (int)((key * 2654435761u) >> (32 - kHashBits));
        // candidates, longest match wins (ties: the first, i.e. the nearer-coded one): the nearest earlier lane of this warp
        // with the same three bytes, the hash table's latest position of an earlier chunk, the previous byte and pixel,
        // and the same bytes one row up
        const unsigned lanes = __match_any_sync(__activemask(), key) & ((1u << (tid & 31)) - 1);
        long long cands[5];
        int nc = 0;
        if (lanes) cands[nc++] = q - ((tid & 31) - (31 - __clz(lanes)));
        const int cand = table[h];
        if (cand >= 0) cands[nc++] = bs + cand;
        cands[nc++] = q - 1;
        cands[nc++] = q - 3;
        cands[nc++] = q - p.pitch;
        for (int k = 0; k < nc && best < maxl; ++k) {
          const long long c = cands[k];
          if (c < 0 || q - c > kWindow || (int)(q - c) == bdist) continue;
          const int l = match_len(filt, q, c, maxl);
          if (l > best) { best = l; bdist = (int)(q - c); }
        }
        if (best < 3 || (best == 3 && bdist > 4096)) best = 0;   // a far 3-byte match costs more than three literals
      }
      sum_a %= kAdlerMod;
      sum_b %= kAdlerMod;
      c_len[tid] = (unsigned short)best;
      c_dist[tid] = (unsigned short)(bdist - 1);
    }
    __syncthreads();
    if (h >= 0) atomicMax(&table[h], (int)(q - bs));
    if (tid == 0) {
      long long pos = s_pos, nt = s_ntok, eb = s_extra_bits;
      const long long end = min(base + kPngThreads, be);
      while (pos < end) {
        const int i = (int)(pos - base);
        int L = c_len[i];
        if (L && pos + 1 < end && c_len[i + 1] > L) L = 0;   // one-step lazy match: a longer one starts at the next byte
        if (L) {
          const int D = c_dist[i] + 1;
          int lc, ln, lx, dc, dn, dx;
          len_code(L, &lc, &ln, &lx);
          dist_code(D, &dc, &dn, &dx);
          lfreq[lc]++; dfreq[dc]++; eb += ln + dn;
          tok[nt++] = kMatchBit | (unsigned)(D - 1) << 8 | (unsigned)(L - 3);
          pos += L;
        } else {
          lfreq[c_byte[i]]++;
          tok[nt++] = c_byte[i];
          pos += 1;
        }
      }
      s_pos = pos; s_ntok = nt; s_extra_bits = eb;
    }
    __syncthreads();
  }

  // Adler-32 partial sums of the band: a = sum x, b = sum (n - i) x_i  (mod 65521)
  for (int o = 16; o; o >>= 1) {
    sum_a += __shfl_down_sync(0xffffffffu, sum_a, o);
    sum_b += __shfl_down_sync(0xffffffffu, sum_b, o);
  }
  if ((tid & 31) == 0) { red_a[tid >> 5] = sum_a; red_b[tid >> 5] = sum_b; }
  __syncthreads();

  // Huffman codes and the size of the dynamic block
  if (tid == 0) {
    lfreq[256] = 1;
    huff_lengths(lfreq, 286, 15, llen, sort_scratch, a_scratch);
    huff_lengths(dfreq, 30, 15, llen + 286, sort_scratch, a_scratch);
    int hlit = 286, hdist = 30;
    while (hlit > 257 && !llen[hlit - 1]) --hlit;
    while (hdist > 1 && !llen[286 + hdist - 1]) --hdist;
    // the code-length sequence of litlen[0..hlit) ++ dist[0..hdist), run-length coded with 16 / 17 / 18
    unsigned char seq[286 + 30];
    const int N = hlit + hdist;
    for (int i = 0; i < hlit; ++i) seq[i] = llen[i];
    for (int i = 0; i < hdist; ++i) seq[hlit + i] = llen[286 + i];
    int nr = 0;
    for (int i = 0; i < N;) {
      const int v = seq[i];
      int run = 1;
      while (i + run < N && seq[i + run] == v) ++run;
      i += run;
      if (v == 0) {
        while (run >= 11) { const int r = min(run, 138); rle_sym[nr] = 18; rle_extra[nr++] = (unsigned char)(r - 11); run -= r; }
        if (run >= 3) { rle_sym[nr] = 17; rle_extra[nr++] = (unsigned char)(run - 3); run = 0; }
        while (run > 0) { rle_sym[nr] = 0; rle_extra[nr++] = 0; --run; }
      } else {
        rle_sym[nr] = (unsigned char)v; rle_extra[nr++] = 0; --run;
        while (run >= 3) { const int r = min(run, 6); rle_sym[nr] = 16; rle_extra[nr++] = (unsigned char)(r - 3); run -= r; }
        while (run > 0) { rle_sym[nr] = (unsigned char)v; rle_extra[nr++] = 0; --run; }
      }
    }
    for (int i = 0; i < nr; ++i) cfreq[rle_sym[i]]++;
    huff_lengths(cfreq, 19, 7, clen, sort_scratch, a_scratch);
    const int order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    int hclen = 19;
    while (hclen > 4 && !clen[order[hclen - 1]]) --hclen;
    unsigned long long hb = 3 + 5 + 5 + 4 + 3ull * hclen;
    for (int i = 0; i < nr; ++i) {
      const int s = rle_sym[i];
      hb += clen[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
    }
    unsigned long long bits = hb + (unsigned long long)s_extra_bits;
    for (int s = 0; s < 286; ++s) bits += (unsigned long long)lfreq[s] * llen[s];
    for (int s = 0; s < 30; ++s) bits += (unsigned long long)dfreq[s] * llen[286 + s];
    const long long dyn = last ? (long long)((bits + 7) >> 3) : (long long)((bits + 3 + 7) >> 3) + 4;
    const long long sto = stored_bytes(n);
    s_stored = dyn >= sto;
    s_hlit = hlit; s_hdist = hdist; s_hclen = hclen; s_nrle = nr;
    s_header_bits = hb; s_bits = bits;
    huff_codes(llen, 286, lcode);
    huff_codes(llen + 286, 30, dcode);
    huff_codes(clen, 19, ccode);
    unsigned long long A = 0, B = 0;
    for (int w = 0; w < kPngThreads / 32; ++w) { A += red_a[w]; B += red_b[w]; }
    info[band].out_bytes = s_stored ? sto : dyn;
    info[band].adler_a = (unsigned)(A % kAdlerMod);
    info[band].adler_b = (unsigned)(B % kAdlerMod);
  }
  __syncthreads();

  if (s_stored) {   // stored blocks of <= 65535 bytes; BFINAL only on the last block of the last band
    const long long nblk = (n + kStoredMax - 1) / kStoredMax, total = n + 5 * nblk;
    for (long long o = tid; o < total; o += kPngThreads) {
      const long long blk = o / (kStoredMax + 5), r = o - blk * (kStoredMax + 5);
      const long long len = lmin(kStoredMax, n - blk * kStoredMax);
      unsigned char v;
      if (r == 0) v = (last && blk == nblk - 1) ? 1 : 0;
      else if (r == 1) v = (unsigned char)(len & 255);
      else if (r == 2) v = (unsigned char)(len >> 8);
      else if (r == 3) v = (unsigned char)(~len & 255);
      else if (r == 4) v = (unsigned char)((~len >> 8) & 255);
      else v = filt[bs + blk * kStoredMax + r - 5];
      stage[o] = v;
    }
    return;
  }

  // dynamic block: zero the slot, write the header (one thread), then the tokens at their prefix-summed bit offsets
  unsigned* words = reinterpret_cast<unsigned*>(stage);
  const long long nbytes = last ? (long long)((s_bits + 7) >> 3) : (long long)((s_bits + 3 + 7) >> 3) + 4;
  for (long long w = tid; w < (nbytes + 3) / 4; w += kPngThreads) words[w] = 0;
  __syncthreads();
  if (tid == 0) {
    const int order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    unsigned long long o = 0;
    put_bits(words, o, (last ? 1u : 0u) | (2u << 1), 3); o += 3;
    put_bits(words, o, (unsigned)(s_hlit - 257), 5); o += 5;
    put_bits(words, o, (unsigned)(s_hdist - 1), 5); o += 5;
    put_bits(words, o, (unsigned)(s_hclen - 4), 4); o += 4;
    for (int i = 0; i < s_hclen; ++i) { put_bits(words, o, clen[order[i]], 3); o += 3; }
    for (int i = 0; i < s_nrle; ++i) {
      const int s = rle_sym[i];
      put_bits(words, o, ccode[s], clen[s]); o += clen[s];
      const int ne = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
      put_bits(words, o, rle_extra[i], ne); o += ne;
    }
  }
  const long long ntok = s_ntok;
  unsigned long long off = s_header_bits;
  for (long long t0 = 0; t0 < ntok; t0 += kPngThreads) {
    const long long t = t0 + tid;
    unsigned v = 0;
    int nb = 0, lc = 0, ln = 0, lx = 0, dc = 0, dn = 0, dx = 0;
    if (t < ntok) {
      v = tok[t];
      if (v & kMatchBit) {
        len_code((int)(v & 255) + 3, &lc, &ln, &lx);
        dist_code((int)((v >> 8) & 0x7fff) + 1, &dc, &dn, &dx);
        nb = llen[lc] + ln + llen[286 + dc] + dn;
      } else {
        nb = llen[v];
      }
    }
    // block-wide exclusive scan of the token bit lengths
    s_scan[tid] = (unsigned long long)nb;
    __syncthreads();
    for (int d = 1; d < kPngThreads; d <<= 1) {
      const unsigned long long add = tid >= d ? s_scan[tid - d] : 0;
      __syncthreads();
      s_scan[tid] += add;
      __syncthreads();
    }
    const unsigned long long pos = off + s_scan[tid] - nb;
    const unsigned long long chunk_bits = s_scan[kPngThreads - 1];
    if (t < ntok) {
      if (v & kMatchBit) {
        unsigned long long o = pos;
        put_bits(words, o, lcode[lc], llen[lc]); o += llen[lc];
        put_bits(words, o, (unsigned)lx, ln); o += ln;
        put_bits(words, o, dcode[dc], llen[286 + dc]); o += llen[286 + dc];
        put_bits(words, o, (unsigned)dx, dn);
      } else {
        put_bits(words, pos, lcode[v], llen[v]);
      }
    }
    off += chunk_bits;
    __syncthreads();
  }
  if (tid == 0) {
    put_bits(words, off, lcode[256], llen[256]);   // end of block
    if (!last) {                                    // sync flush: empty stored block, 3 zero bits, pad, 00 00 ff ff
      const long long b = (long long)((off + llen[256] + 3 + 7) >> 3);
      stage[b] = 0; stage[b + 1] = 0; stage[b + 2] = 0xff; stage[b + 3] = 0xff;
    }
  }
}

// reflected CRC-32 polynomial arithmetic (bit 31 = x^0): a * b mod P
__device__ __forceinline__ unsigned crc_mulmod(unsigned a, unsigned b) {
  unsigned m = 1u << 31, r = 0;
  for (;;) {
    if (a & m) {
      r ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return r;
}

// x^(8 n) mod P from x2n[k] = x^(2^k) mod P
__device__ __forceinline__ unsigned crc_x8n(const unsigned* x2n, unsigned long long n) {
  unsigned r = 1u << 31;
  int k = 3;
  while (n) {
    if (n & 1) r = crc_mulmod(x2n[k & 31], r);
    n >>= 1; ++k;
  }
  return r;
}

// CRC of data1 || data2 from crc(data1), crc(data2) and len(data2)
__device__ __forceinline__ unsigned crc_shift(const unsigned* x2n, unsigned crc1, unsigned long long len2) {
  return crc_mulmod(crc_x8n(x2n, len2), crc1);
}

__device__ void crc_tables(unsigned* table, unsigned* x2n) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    unsigned c = (unsigned)i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kCrcPoly : c >> 1;
    table[i] = c;
  }
  if (threadIdx.x == 0) {
    unsigned v = 1u << 30;   // x^1
    x2n[0] = v;
    for (int k = 1; k < 32; ++k) { v = crc_mulmod(v, v); x2n[k] = v; }
  }
}

__device__ __forceinline__ unsigned crc_bytes(const unsigned* table, const unsigned char* d, long long n) {
  unsigned c = 0xffffffffu;
  for (long long i = 0; i < n; ++i) c = table[(c ^ d[i]) & 255] ^ (c >> 8);
  return c ^ 0xffffffffu;
}

__global__ void __launch_bounds__(kPngThreads) png_place_kernel(PngPlan p, const unsigned char* __restrict__ stage_all,
                                                               BandInfo* __restrict__ info, unsigned char* __restrict__ out) {
  __shared__ unsigned table[256], x2n[32];
  __shared__ unsigned long long red[kPngThreads / 32];
  __shared__ unsigned crc_red;
  const int tid = threadIdx.x;
  const long long band = blockIdx.x;
  crc_tables(table, x2n);
  unsigned long long s = 0;
  for (long long j = tid; j < band; j += kPngThreads) s += (unsigned long long)info[j].out_bytes;
  for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  if (tid == 0) crc_red = 0;
  __syncthreads();
  long long offset = 0;
  for (int w = 0; w < kPngThreads / 32; ++w) offset += (long long)red[w];
  const long long nb = info[band].out_bytes;
  const unsigned char* src = stage_all + band * p.stage_stride;
  unsigned char* dst = out + kHeadBytes + offset;
  for (long long i = tid; i < nb; i += kPngThreads) dst[i] = src[i];
  // CRC of the band: one contiguous segment per thread, combined by shifting each past the bytes that follow it
  const long long seg = (nb + kPngThreads - 1) / kPngThreads;
  const long long s0 = lmin(nb, tid * seg), s1 = lmin(nb, s0 + seg);
  unsigned c = 0;
  if (s1 > s0) c = crc_shift(x2n, crc_bytes(table, src + s0, s1 - s0), (unsigned long long)(nb - s1));
  atomicXor(&crc_red, c);
  __syncthreads();
  if (tid == 0) { info[band].offset = offset; info[band].crc = crc_red; }
}

__device__ __forceinline__ void put_be32(unsigned char* d, unsigned v) {
  d[0] = (unsigned char)(v >> 24); d[1] = (unsigned char)(v >> 16); d[2] = (unsigned char)(v >> 8); d[3] = (unsigned char)v;
}

__global__ void __launch_bounds__(kPngThreads) png_finish_kernel(PngPlan p, int H, int W, const BandInfo* __restrict__ info,
                                                                unsigned char* __restrict__ out, long long* __restrict__ out_len) {
  __shared__ unsigned table[256], x2n[32];
  __shared__ unsigned crc_red, s_adler;
  const int tid = threadIdx.x;
  crc_tables(table, x2n);
  if (tid == 0) crc_red = 0;
  __syncthreads();
  const BandInfo& lastb = info[p.bands - 1];
  const long long total = lastb.offset + lastb.out_bytes;   // bytes of all bands
  unsigned c = 0;
  for (long long k = tid; k < p.bands; k += kPngThreads) {
    const long long after = total - info[k].offset - info[k].out_bytes + 4;   // later bands, then the Adler-32
    c ^= crc_shift(x2n, info[k].crc, (unsigned long long)after);
  }
  atomicXor(&crc_red, c);
  if (tid == 0) {
    // Adler-32 over the bands in order: b += n_k a + B_k, a += A_k
    unsigned long long a = 1, b = 0;
    for (long long k = 0; k < p.bands; ++k) {
      const unsigned long long nk = (unsigned long long)((k == p.bands - 1) ? p.last_bytes : p.band_bytes) % kAdlerMod;
      b = (b + nk * a + info[k].adler_b) % kAdlerMod;
      a = (a + info[k].adler_a) % kAdlerMod;
    }
    s_adler = (unsigned)(b << 16 | a);
    const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    for (int i = 0; i < 8; ++i) out[i] = sig[i];
    unsigned char* ih = out + 8;
    put_be32(ih, 13);
    ih[4] = 'I'; ih[5] = 'H'; ih[6] = 'D'; ih[7] = 'R';
    put_be32(ih + 8, (unsigned)W);
    put_be32(ih + 12, (unsigned)H);
    ih[16] = 8; ih[17] = 2; ih[18] = 0; ih[19] = 0; ih[20] = 0;   // depth 8, RGB, deflate, adaptive filtering, no interlace
    put_be32(ih + 21, crc_bytes(table, ih + 4, 17));
    unsigned char* id = out + 33;
    put_be32(id, (unsigned)(2 + total + 4));
    id[4] = 'I'; id[5] = 'D'; id[6] = 'A'; id[7] = 'T';
    id[8] = 0x78; id[9] = 0x01;                                   // deflate, 32 KiB window, check bits
  }
  __syncthreads();
  if (tid == 0) {
    unsigned char* tail = out + kHeadBytes + total;
    put_be32(tail, s_adler);
    const unsigned head_crc = crc_bytes(table, out + 37, 6);      // "IDAT" + zlib header
    const unsigned idat_crc = crc_shift(x2n, head_crc, (unsigned long long)(total + 4)) ^ crc_red ^ crc_bytes(table, tail, 4);
    put_be32(tail + 4, idat_crc);
    unsigned char* ie = tail + 8;
    put_be32(ie, 0);
    ie[4] = 'I'; ie[5] = 'E'; ie[6] = 'N'; ie[7] = 'D';
    put_be32(ie + 8, crc_bytes(table, ie + 4, 4));
    *out_len = kHeadBytes + total + kTailBytes;
  }
}

}  // namespace b2p

using namespace b2p;

extern "C" {

int b2p_png_plan_host(int H, int W, long long* sizes_host) {
  PngPlan p{};
  if (png_plan(H, W, &p)) return -1;
  if (sizes_host) {
    sizes_host[0] = p.bands;
    sizes_host[1] = p.ws_bytes;
    sizes_host[2] = p.out_bytes;
  }
  return 0;
}

int b2p_png_encode(const unsigned char* rgb, int H, int W, void* ws, long long ws_bytes, unsigned char* out, long long out_cap,
                   long long* out_len, cudaStream_t st) {
  PngPlan p{};
  if (png_plan(H, W, &p)) return -1;
  if (!rgb || !ws || !out || !out_len) return set_error("b2p_png_encode: null pointer");
  if (ws_bytes < p.ws_bytes) return set_error("b2p_png_encode: workspace smaller than b2p_png_plan_host's");
  if (out_cap < p.out_bytes) return set_error("b2p_png_encode: output capacity below b2p_png_plan_host's worst case");
  if (bind_device()) return -1;
  unsigned char* w = static_cast<unsigned char*>(ws);
  unsigned char* filt = w + p.filt_off;
  unsigned* tok = reinterpret_cast<unsigned*>(w + p.tok_off);
  unsigned char* stage = w + p.stage_off;
  BandInfo* info = reinterpret_cast<BandInfo*>(w + p.info_off);
  const long long nf = (long long)H * p.pitch;
  const unsigned fgrid = (unsigned)lmin((nf + 255) / 256, 132LL * 16);
  png_filter_kernel<<<fgrid, 256, 0, st>>>(rgb, H, W, filt);
  B2P_CHECK_LAUNCH();
  png_band_kernel<<<(unsigned)p.bands, kPngThreads, 0, st>>>(filt, p, tok, stage, info);
  B2P_CHECK_LAUNCH();
  png_place_kernel<<<(unsigned)p.bands, kPngThreads, 0, st>>>(p, stage, info, out);
  B2P_CHECK_LAUNCH();
  png_finish_kernel<<<1, kPngThreads, 0, st>>>(p, H, W, info, out, out_len);
  B2P_CHECK_LAUNCH();
  return 0;
}

}  // extern "C"
