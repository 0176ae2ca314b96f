/* libb200parse.so -- C ABI of the CUDA-native (H100, sm_90a) OmniParser parse hot path.
 *
 * The reference (microsoft/OmniParser) has no FFI layer: its hot path is three Python functions
 * (util/utils.py: get_yolo_model :72-85, get_caption_model_processor :48-69, get_som_labeled_img :417-496) whose
 * arithmetic lives in third-party wheels (TorchScript/cuDNN, torchvision::nms, cv2, PIL, HF transformers).
 * Each entry point below replaces one of those library call sites; the reference file:line it stands in for is
 * cited per function.  omniparser_b200/_lib.py is the ctypes binding a maintainer would add (INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes only (no torch types); every pointer is DEVICE memory unless its name
 * ends in _host; all launches are asynchronous on `stream`; return 0 on success, -1 on error with the message in
 * b2p_last_error(); the caller owns every buffer; a process uses one GPU (cudaSetDevice before the first call).
 * Feature maps are NHWC fp16 "channel slices": base pointer already offset to the first channel, `ld` = channels
 * per pixel of the owning buffer, so concatenations are pointer arithmetic.
 */
#ifndef B200PARSE_H
#define B200PARSE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* b2p_stream_t; /* == cudaStream_t */

/* ---- library state ---- */
const char* b2p_last_error(void);
long long b2p_launch_count(void); /* kernels launched by this library since load (bench.py gpu_launches) */
int b2p_abi_version(void);
/* Debugging aid, not on the hot path: with B2P_TRACE=1 in the environment every GEMM/conv launch is handed a stamp
 * buffer and its kernel leaves globaltimer stamps per CTA (a runtime branch, off otherwise); this returns the launches recorded since the
 * last call: stamps [n][160][16] (ns; slots: entry, prologue, dependency wait, first TMA, first full stage, first
 * accumulator issued, first epilogue start, last epilogue end, exit), meta [n][8] = {mode, M, N, K, bn, ksplit, x3, grid}. */
int b2p_trace_read(unsigned long long* stamps, int* meta, int max_launches);

/* ---- streams and split-K workspace slots (host only) ----
 * Split-K GEMM/conv launches park partial tiles in a workspace slot owned by the launching stream (under graph capture: the
 * capture stream, whose slot the graph bakes in); a stream claims one of 24 slots at its first GEMM/conv launch.  Streams that
 * may run concurrently must therefore be distinct handles.
 * b2p_stream_create: a new non-blocking stream on the current device (cudaStreamCreateWithFlags), outside any pool.
 * b2p_stream_destroy: destroys a stream and releases its slot; the caller ensures the stream is idle and that no graph
 *   captured on it is replayed afterwards.
 * b2p_ws_slot: the slot the stream owns, or -1; never claims one.
 * b2p_ws_audit: synchronises the device, then nonzero_host[i] (i < max_slots) = the number of non-zero arrival-counter words
 *   of slot i, or -1 if no stream owns it; returns the number of slots (24).  A completed split-K launch leaves its counters
 *   at zero, so with the device idle every owned slot should report 0.  For tests and debugging. */
int b2p_stream_create(b2p_stream_t* out);
int b2p_stream_destroy(b2p_stream_t st);
int b2p_ws_slot(b2p_stream_t st);
int b2p_ws_audit(int* nonzero_host, int max_slots);

/* ---- dense contractions (wgmma + TMA), ref:util/yolov9.py:120-121 and ref:util/utils.py:125 ----
 * flags: bit0 operands bf16 (else fp16) | bit1 output fp32 (else fp16) | bit2 fp16 output in the "fp16x3" operand
 * layout [hi(N) | lo(N)] (ldc >= 2N) | bit3 fp16x3 OPERANDS: A rows [hi(K) | lo(K)] (lda >= 2K; conv: pixels
 * [hi(Cin) | lo(Cin)]), weight rows [hi | lo] likewise (conv: per tap), K / Cin the logical sizes; the kernel loads each
 * half once per k-block and accumulates hi*hi + hi*lo + lo*hi in fp32 | bit4 never split K (tuning) | bits 8.. maximum N tile (0 = auto).
 * act: 0 none, 1 SiLU, 2 exact GELU.
 * out = act(A[M,K] * B[N,K]^T + bias[N]) + residual (residual has the dtype of out). */
int b2p_gemm(const void* A, long long lda, const void* B, int M, int N, int K, void* out, long long ldc,
             const float* bias, const void* residual, long long ldr, int act, int flags, b2p_stream_t stream);
/* 3x3, pad 1, stride 1|2 convolution as implicit GEMM; weight [Cout][9*Cin] ordered (ky, kx, c). */
int b2p_conv3x3(const void* in, long long ld_in, int batch, int H, int W, int Cin, int stride, const void* weight,
                int Cout, void* out, long long ldc, const float* bias, const void* residual, long long ldr, int act,
                int flags, b2p_stream_t stream);

/* `_planes` forms (fp16x3 operands that are channel slices of a wider [hi(Ctot) | lo(Ctot)] pixel / row): explicit
 * lo-plane offsets in elements -- lo_a: A's lo half at column lo_a + k (default K / Cin); lo_out: with flags bit2 the
 * output's lo half at column lo_out + n (default N); lo_res: the fp16 residual is a hi/lo pair whose lo half sits at
 * column lo_res + n (default 0: the residual has no lo half).  This is what the parity-grade (fp16x3) detector mode uses:
 * every YOLOv9-E feature map stays a hi/lo pair inside its concat buffer (ref:util/yolov9.py:120-121 in fp32). */
int b2p_gemm_planes(const void* A, long long lda, const void* B, int M, int N, int K, void* out, long long ldc,
                    const float* bias, const void* residual, long long ldr, int act, int flags, long long lo_a,
                    long long lo_out, long long lo_res, b2p_stream_t stream);
int b2p_conv3x3_planes(const void* in, long long ld_in, int batch, int H, int W, int Cin, int stride, const void* weight,
                       int Cout, void* out, long long ldc, const float* bias, const void* residual, long long ldr, int act,
                       int flags, long long lo_a, long long lo_out, long long lo_res, b2p_stream_t stream);

/* Host only (no device is touched): the plan the launch of b2p_conv3x3_planes (stride 1 | 2) or of b2p_gemm_planes
 * (stride 0, with M = batch and K = Cin; H and W ignored) would make on a device with num_sms SMs and max_smem bytes of
 * opt-in shared memory per block, under the same B2P_* environment knobs; flags as there, plus bit5: the park-only GEMM of
 * b2p_gemm_ln.  Makes every host-side rejection the launch makes.  It assumes the launching stream owns a split-K workspace
 * slot: a launch on a stream that finds all 24 slots taken by other streams is planned without split-K instead (and a
 * park-only one is refused); b2p_gemm_last_plan tells what was launched.  plan_host receives 45 ints:
 *   0 mode (0 GEMM, 1 conv s1 per tap, 2 conv s2 parity view, 3 conv s1 halo tile), 1 bk, 2 bn, 3 ksplit, 4 kb_per,
 *   5 kb_merge, 6 stages, 7 stagesA, 8 sep, 9 bres, 10 nb, 11 tw, 12 tw_valid, 13 th, 14 m_tiles, 15 n_tiles, 16 mt_fast,
 *   17 grid, 18 smem (bytes), 19 vec_ok, 20 split (lo-plane offset of the output, 0 = none), 21 res_lo, 22 park,
 *   23 x3, 24 num_kb, 25 taps, 26 a_bytes, 27 a_slot, 28 b_bytes, 29 b_slot, 30 tiles_x, 31 tiles_y,
 *   32 rank of A's tensor map, 33-37 its box (elements, unused dims 0), 38-39 B's box,
 *   40 / 41 elements from A / B to one past the last element their tensor maps can address (saturating at 2^31-1),
 *   42 / 43 swizzle span (bytes) of A's / B's tensor map, 44 swizzle span of the wgmma shared-memory descriptors.
 * kb_per, num_kb and bk count the 32- or 64-wide k-blocks the kernel streams (halo mode: channel blocks of nine taps). */
int b2p_gemm_plan(const void* in, long long ld_in, int batch, int H, int W, int Cin, int stride, const void* weight, int Cout,
                  void* out, long long ldc, const float* bias, const void* residual, long long ldr, int act, int flags,
                  long long lo_a, long long lo_out, long long lo_res, int num_sms, int max_smem, int* plan_host);
/* Host only: the same 45 fields for the most recent GEMM/conv launch made by the calling thread (-1 if it made none). */
int b2p_gemm_last_plan(int* plan_host);
/* Host only: the epilogue of the plan b2p_gemm_plan makes for the same arguments.  epi_host receives 24 ints:
 *   0 TMA epilogue (1) or register epilogue (0), 1 columns per chunk, 2 chunks per tile, 3 staging buffers,
 *   4 output planes (2 = fp16 [hi | lo] pair), 5 residual buffers, 6 residual planes (0 = no residual),
 *   7 shared memory of the epilogue (bytes), 8 stages, 9 stagesA, 10 smem (as b2p_gemm_plan fields 6, 7, 18),
 *   11 rank of the output tensor map, 12-14 its box (elements, unused dims 0), 15-16 its global strides of dims 1, 2 (bytes),
 *   17-22 the same for the residual tensor map (rank 0 = none), 23 swizzle span (bytes) of both.
 * Fields 11-23 are 0 for the register epilogue. */
int b2p_gemm_epilogue_plan(const void* in, long long ld_in, int batch, int H, int W, int Cin, int stride, const void* weight, int Cout,
                           void* out, long long ldc, const float* bias, const void* residual, long long ldr, int act, int flags,
                           long long lo_a, long long lo_out, long long lo_res, int num_sms, int max_smem, int* epi_host);

/* ---- YOLOv9-E graph helpers (inside the TorchScript archive, ref:util/yolov9.py:120-121) ----
 * `_x3` forms: every map is an fp16 hi/lo pair (lo plane `lo*` elements after the hi plane, 0 = plain fp16); the
 * arithmetic runs on the exact fp32 sums hi + lo and the result is re-split. */
int b2p_adown_pool(const void* x, long long ldx, int B, int H, int W, int C, void* x1, long long ld1, void* x2,
                   long long ld2, b2p_stream_t stream);
int b2p_adown_pool_x3(const void* x, long long ldx, int B, int H, int W, int C, void* x1, long long ld1, void* x2,
                      long long ld2, long long lox, long long lo1, long long lo2, b2p_stream_t stream);
int b2p_maxpool_s1(const void* x, long long ldx, int B, int H, int W, int C, int k, void* y, long long ldy,
                   b2p_stream_t stream);
int b2p_maxpool_s1_x3(const void* x, long long ldx, int B, int H, int W, int C, int k, void* y, long long ldy,
                      long long lox, long long loy, b2p_stream_t stream);
int b2p_upsample2x(const void* x, long long ldx, int B, int H, int W, int C, void* y, long long ldy,
                   b2p_stream_t stream);
int b2p_upsample2x_x3(const void* x, long long ldx, int B, int H, int W, int C, void* y, long long ldy, long long lox,
                      long long loy, b2p_stream_t stream);
/* explicit 3x3 / pad-1 im2col of an NHWC f16 map -> [B*Ho*Wo][9*C] (tap-major), for convs whose output map is far
 * smaller than one 128-pixel implicit-GEMM tile (DaViT patch-embed convs of the 64x64-crop mode, hf:modeling_florence2.py
 * ConvEmbed, reached from ref:util/utils.py:125 generate) */
int b2p_im2col3x3(const void* x, long long ldx, int B, int H, int W, int C, int stride, int halves, void* out,
                  b2p_stream_t stream);   /* halves = 2: fp16x3 pixels [hi(C) | lo(C)] -> rows [hi: 9C | lo: 9C] */
int b2p_cbfuse(int nsrc, const void* const* srcs_host, const long long* lds_host, const int* shifts_host,
               const void* last, long long ldl, int B, int H, int W, int C, void* y, long long ldy,
               b2p_stream_t stream);
int b2p_cbfuse_x3(int nsrc, const void* const* srcs_host, const long long* lds_host, const int* shifts_host,
                  const long long* los_host, const void* last, long long ldl, int B, int H, int W, int C, void* y,
                  long long ldy, long long lol, long long loy, b2p_stream_t stream);

/* ---- detector pre/post-processing ----
 * b2p_letterbox: PIL Image.resize(LANCZOS) + paste on a 114 canvas, ref:util/yolov9.py:73-84 (bit-exact).  Returns an
 *                error without launching when a size is < 1 (Pillow raises) or the resized image does not lie inside
 *                the canvas; b2p_resize_u8 likewise for sizes < 1.
 * b2p_im2col_u8: /255 (ref:util/yolov9.py:85) or CLIP rescale+normalise (ref:util/utils.py:121) via `lut` [3][256]
 *                + im2col of the 3-channel stem conv; split != 0 writes the fp16x3 layout.
 * b2p_yolo_decode: ref:util/yolov9.py:89-108 (_decode) and :123-129 (class max, strict conf filter, un-letterbox).
 * b2p_batched_nms: torchvision.ops.batched_nms + [:max_det] + clamp, ref:util/yolov9.py:131-135 (bit-exact).
 * b2p_lanczos_coeffs_host: Pillow's coefficient table on the host (unit-testable without a GPU). */
int b2p_lanczos_coeffs_host(int in_size, int out_size, int* ksize_host, int* bounds_host, int* kk_host, int kk_capacity);
int b2p_letterbox(const unsigned char* src, int B, int H, int W, int Wr, int Hr, int Tw, int Th, int pad_l, int pad_t,
                  unsigned char* tmp, unsigned char* canvas, b2p_stream_t stream);
/* Ragged letterbox: b2p_letterbox for a batch of screenshots of DIFFERENT sizes onto one canvas (Tw, Th), in at most two
 * launches, with the same arithmetic (ref:util/yolov9.py:73-84 per image; bit-exact).
 * b2p_letterbox_batch_plan_host (host only, no device touched): geom_host [B][6] = per image (H, W, Wr, Hr, pad_l, pad_t) ->
 *   desc_host [B][12] int64 per image: 0 byte offset of the image in the flat src buffer ([H][W][3], images back to back),
 *   1 byte offset of its horizontal-pass output in tmp ([H][Wr][3], -1 when Wr == W: Pillow skips that pass), 2-7 H, W,
 *   Wr, Hr, pad_l, pad_t, 8 / 9 element offset in the table buffer and ksize of the horizontal table (-1 / -1 when Wr == W),
 *   10 / 11 the same for the vertical table (-1 / -1 when Hr == H);
 *   tables_host: int32 tables ([out][2] bounds, then [out][ksize] 22-bit weights), one per distinct (in, out) pair of the
 *   batch, from a bounded host cache (256 pairs, least recently used evicted);
 *   sizes_host [3] = table ints, tmp bytes, src bytes the batch needs.
 *   tables_host == NULL is a size query: only sizes_host is written.  Refused before anything is written: B outside
 *   [1, 65535], a size < 1, a resized image outside the canvas, tables_capacity (ints) < the tables' size.
 * b2p_letterbox_batch: desc_host is the plan's descriptor array on the host (validated, and read for the launch
 *   geometry), desc / tables its device copies; src / tmp are the flat buffers the descriptors address, canvas
 *   [B][Th][Tw][3].  No allocation and no synchronous copy. */
int b2p_letterbox_batch_plan_host(int B, const int* geom_host, int Tw, int Th, long long* desc_host, int* tables_host,
                                  long long tables_capacity, long long* sizes_host);
int b2p_letterbox_batch(const unsigned char* src, int B, const long long* desc_host, const long long* desc, const int* tables,
                        int Tw, int Th, unsigned char* tmp, unsigned char* canvas, b2p_stream_t stream);
/* Pillow-exact u8 resize, filter 0 LANCZOS / 1 BICUBIC (CLIP processor resample=3, ref:util/utils.py:123 CPU branch) */
int b2p_resize_u8(const unsigned char* src, int B, int H, int W, int Wr, int Hr, int filter, unsigned char* tmp,
                  unsigned char* out, b2p_stream_t stream);
int b2p_im2col_u8(const unsigned char* img, int B, int H, int W, int k, int s, int p, int Kpad, const float* lut,
                  void* out, int split, b2p_stream_t stream);
int b2p_yolo_decode(const float* const* cls_host, const float* const* box_host, const int* Hs_host, const int* Ws_host,
                    int nc, int B, float conf, const float* pad_l, const float* pad_t, const float* scale, int cap,
                    float* cand_box, float* cand_score, int* cand_cls, int* cand_count, float* dense_ltrb,
                    float* dense_score, b2p_stream_t stream);
int b2p_batched_nms(const float* box, const float* score, const int* cls, const int* count, int B, int cap,
                    double iou_thr, int max_det, const float* img_w, const float* img_h, int* keep_idx, float* out_box,
                    float* out_score, int* out_count, b2p_stream_t stream);

/* ---- overlap filter on the device, ref:util/utils.py:241-319 (remove_overlap_new), :411-415 (int_box_area), :432, :444-451 ----
 * Per screenshot b: the detector's kept boxes box_px[b][0..count[b]) (pixels, fp32, b2p_batched_nms output) and ocr_count[b]
 * OCR boxes as fp32 RATIO boxes (int_box_area-filtered on the host, where their strings stay).  Same float64 arithmetic,
 * comparisons and list order as the reference.  Outputs: icon_state[b][i] = 0 dropped | 1 kept, needs a caption | 2 kept,
 * labelled by OCR text; label_mask[b][i][max_ocr/32] bit k = OCR box k labels icon i; ocr_removed[b][k]; icon_ratio = the
 * fp32 ratio boxes (:432); crop_box / crop_img = the state-1 boxes of the whole batch in order (the crop list of
 * b2p_crop_resize); crop_counts[0..B) per screenshot, crop_counts[B] the total.  `arrive` is a zeroed int the kernel resets. */
int b2p_overlap_filter(const float* box_px, const int* count, int B, int max_det, const float* img_w, const float* img_h,
                       const float* ocr_ratio, const int* ocr_count, int max_ocr, double iou_thr, int* icon_state,
                       unsigned* label_mask, int* ocr_removed, float* icon_ratio, float* crop_box, int* crop_img,
                       int* crop_counts, int* arrive, b2p_stream_t stream);

/* ---- crop + resize, ref:util/utils.py:97-103 (numpy slice + cv2.resize(.., (64,64)), bit-exact) ---- */
int b2p_crop_resize(const unsigned char* imgs, const int* img_hw, const long long* img_off, const float* boxes_ratio,
                    const int* box_img, int n_box, int out_hw, unsigned char* out, int* status, b2p_stream_t stream);

/* ---- PNG encode of the Set-of-Marks overlay, ref:util/utils.py:493-494 (PIL Image.save(format="PNG")), lossless ----
 * Up filter on every row; the filtered rows in bands of whole rows (about 32 KiB each), each deflated on its own (LZ77,
 * dynamic Huffman or stored blocks, whichever is smaller) and ended byte-aligned by a sync flush; one zlib stream in one
 * IDAT chunk.  The bytes differ from PIL's and from som_overlay.encode_png's; the decoded pixels are the frame's.
 * b2p_png_plan_host (host only): sizes_host [3] = band count, workspace bytes, worst-case output bytes (every band
 *   stored).  Refused: H or W < 1, a worst-case IDAT longer than 2^31 - 1 bytes.
 * b2p_png_encode: rgb [H][W][3] contiguous u8 -> out[0..*out_len) (out_len: a device int64), asynchronous on `stream`.
 *   Refused before any launch: what the plan refuses, null pointers, ws_bytes or out_cap below the plan's.  Never writes
 *   past the plan's worst case (<= out_cap). */
int b2p_png_plan_host(int H, int W, long long* sizes_host);
int b2p_png_encode(const unsigned char* rgb, int H, int W, void* ws, long long ws_bytes, unsigned char* out, long long out_cap,
                   long long* out_len, b2p_stream_t stream);

/* ---- Florence-2 (HF generate, ref:util/utils.py:125): non-GEMM kernels; `split` selects the fp16x3 layout ---- */
int b2p_layernorm(const float* x, long long ldx, const float* gamma, const float* beta, float eps, int T, int C,
                  void* out16, long long ld16, float* out32, long long ld32, int split, b2p_stream_t stream);
/* LayerNorm(A * B^T + bias + residual) for the decoder's split-K GEMMs that feed a LayerNorm (hf:models/bart/modeling_bart.py:
 * 312-391: out-proj / cross out-proj / fc2 + residual + layer norm): the GEMM parks its raw partial tiles, one more kernel sums
 * the k slices, adds bias + residual and normalises.  flags as b2p_gemm (bit 3: fp16x3 operands, bit 2: out16 as [hi | lo]). */
int b2p_gemm_ln(const void* A, long long lda, const void* B, int M, int N, int K, const float* bias, const float* residual,
                long long ldr, const float* gamma, const float* beta, float eps, void* out16, long long ld16, float* out32,
                long long ld32, int flags, b2p_stream_t stream);
int b2p_dwconv3x3_res(const float* x, int B, int H, int W, int C, const float* w9c, const float* bias, float* y,
                      b2p_stream_t stream);
int b2p_dwconv_ln(const float* x, int B, int H, int W, int C, const float* w9c, const float* bias, float* y,
                  const float* gamma, const float* beta, float eps, void* out16, int split, b2p_stream_t stream);
int b2p_window_attn(const float* qkv, const float* qkv_bias, int B, int H, int W, int C, int heads, int win, void* out,
                    int split, b2p_stream_t stream);
int b2p_channel_attn(const float* qkv, int B, int N, int C, int groups, void* out, int split, b2p_stream_t stream);
int b2p_mha(const float* q, long long ldq, const float* k, const float* v, long long ldk, int B, int Lq, int Lk,
            int heads, void* out, long long ldo, int split, b2p_stream_t stream);
int b2p_mha_cached(const float* q, long long ldq, const float* knew, const float* vnew, long long ldnew, float* kcache,
                   float* vcache, int tmax, const int* step, int B, int heads, void* out, long long ldo, int split,
                   b2p_stream_t stream);
int b2p_encoder_embed(const float* img, int n_img, const float* E, const int* prompt, int n_prompt, const float* P,
                      int B, int C, float* out, b2p_stream_t stream);
int b2p_decoder_embed(const float* E, const int* seq, int seq_ld, const int* step, const float* P, int B, int C,
                      float* out, b2p_stream_t stream);
int b2p_projector_prep(const float* x, const float* pos, int B, int HW, int C, void* out, int split,
                       b2p_stream_t stream);
/* HF greedy step with no_repeat_ngram / forced BOS / forced EOS processors, hf:generation/utils.py:2727-2805.  Writes
 * seq[b][*step + 1]; *step + 1 must be <= max_len - 1.  The ban list is never truncated (up to max_len - 1 entries in
 * shared memory).  Refused before any launch: B < 0, V < 1, ld < V, ngram < 0, max_len outside [2, 8192],
 * seq_ld < max_len, forced ids >= V.  B == 0 launches nothing. */
int b2p_greedy_pick(const float* logits, long long ld, int V, int B, int* seq, int seq_ld, int* finished,
                    const int* step, int ngram, int forced_bos, int forced_eos, int eos, int pad, int max_len,
                    float* dump, int* n_unfinished, b2p_stream_t stream);
int b2p_step_advance(int* step, b2p_stream_t stream);

/* ---- Florence-2 beam search, HF's _beam_search (hf:generation/utils.py:3076-3386, helpers :2876-3072) ----
 * Decoder rows r = crop * nb + beam (B = K * nb), 1 <= nb <= 16; decoder prompt length 1 (decoder_start at seq[r][0]).
 *
 * Tie rule (ours: torch.topk leaves the order of exact ties unspecified): every selection takes the higher score first and,
 * on equal scores, the lower index -- the flat index beam * V + token in the per-crop top 2 nb, the position in that list when
 * the running beams are picked, the merged index (old hypotheses 0..nb-1, then candidates) when hypotheses are merged.
 * Two kinds of ties that torch may break differently never reach the output:
 *  - the -1e9 placeholders (initial beams 1..nb-1, and candidates that did not finish, whose s / L^lp - 1e9 rounds to
 *    -1e9 in fp32): a crop stops only when every hypothesis slot holds a finished sequence with a real score (the early-stop
 *    heuristic cannot fail while a slot is empty, and at max_len the top nb candidates all finish), and tied placeholder
 *    running beams share the same prefix and cache contents;
 *  - the -inf candidates of a forced step (forced BOS / EOS leave one finite score per beam): they only fill ranks >= nb,
 *    which neither become running beams nor finish.
 *
 * b2p_beam_topk (HF step b + the per-row part of c): per row, log_softmax of logits[r][0..V) in fp32, then the processors on
 * the log-probs in HF order -- no_repeat_ngram bans -> -inf (the ban scan is greedy_pick's), forced BOS / EOS: -inf except the
 * forced token's 0 (the logits are then not read) -- plus bscore[r]; writes the row's best 2 nb as cand_score / cand_idx
 * [B][2 nb] (flat index beam * V + token), best first.  The crop's top 2 nb lies in the union of its rows' top 2 nb.  Rows of
 * crops with done[crop] set are skipped (done may be null).  Refused before any launch: B < 0, nb outside [1, 16],
 * B % nb != 0, V < 2 nb, ld < V, ngram < 0, max_len outside [2, 8192], seq_ld < max_len, forced ids >= V.  B == 0 launches
 * nothing. */
int b2p_beam_topk(const float* logits, long long ld, int V, int B, int nb, const int* seq, int seq_ld, const int* step,
                  int ngram, int forced_bos, int forced_eos, int max_len, const float* bscore, const int* done,
                  float* cand_score, int* cand_idx, b2p_stream_t stream);
/* b2p_beam_update (HF steps c-g; one CTA per crop, crops with done[k] set are left untouched -- their hypotheses can no
 * longer change): merges the rows' candidates to the crop's top 2 nb; flags EOS / max-length hits; picks the running beams
 * (score + hit * -1e9, best nb: _get_running_beams_for_next_iteration :2995-3016); merges finished hypotheses
 * (_update_finished_beams :3018-3072: / L^lp, the "batch full" and heuristic -1e9 terms, top-nb mask, in fp32 and in HF's
 * order); updates the early-stop heuristic (_check_early_stop_heuristic :2876-2925; early_stopping 0 = False, 1 = True,
 * 2 = "never", only the sign of length_penalty is used); then writes the new tokens and parent-gathered prefixes into seq,
 * bscore, parent[r] (beam index, may be null) and the cache ancestor table src[r][0..t] (src'[r][j] = src[parent][j] for j < t,
 * src'[r][t] = the parent's row), and, when the crop stops (_beam_search_has_unfinished_sequences :2927-2949 for the crop),
 * sets done[k] and decrements *n_open.  lp_pow[L] = float(L ** length_penalty) computed in double (torch divides fp32 by the
 * Python float).  Finished hypotheses: hyp_seq [K * nb][seq_ld] (pad-filled), hyp_score / hyp_len (generated tokens incl.
 * EOS) / hyp_fin [K * nb], best first.  Initial state: bscore [0, -1e9, ...] per crop, hyp_score -1e9, hyp_fin 0, hyp_seq pad,
 * heur 1.  The crop's seq and src rows are staged in shared memory, so nb * max_len is limited to 16384.  Refused before any
 * launch: K < 0, nb outside [1, 16], V < 2 nb, max_len outside [2, 8192], seq_ld < max_len, tmax < max_len - 1,
 * nb * max_len > 16384, early_stopping outside {0, 1, 2}, lp_pow null.  K == 0 launches nothing. */
int b2p_beam_update(const float* cand_score, const int* cand_idx, int V, int K, int nb, int* seq, int seq_ld, int* src,
                    int tmax, const int* step, int eos, int pad, int max_len, int early_stopping, float length_penalty,
                    const float* lp_pow, float* bscore, int* parent, int* hyp_seq, float* hyp_score, int* hyp_len,
                    int* hyp_fin, int* heur, int* done, int* n_open, b2p_stream_t stream);
/* b2p_mha_cached with a beam-indexed cache instead of HF's reorder_cache (hf:generation/utils.py:3340-3346): row r's entry for
 * position j < *step is read from physical row src[r][j] ([B][tmax]); this step's k / v are appended at (r, *step). */
int b2p_mha_cached_beam(const float* q, long long ldq, const float* knew, const float* vnew, long long ldnew, float* kcache,
                        float* vcache, int tmax, const int* step, const int* src, int B, int heads, void* out, long long ldo,
                        int split, b2p_stream_t stream);
/* b2p_mha where query row b reads K / V batch b / rows_per_kv (the crop's cross-attention K / V, shared by its beams). */
int b2p_mha_grouped(const float* q, long long ldq, const float* k, const float* v, long long ldk, int B, int Lq, int Lk,
                    int heads, int rows_per_kv, void* out, long long ldo, int split, b2p_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200PARSE_H */
