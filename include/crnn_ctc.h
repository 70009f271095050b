/*
 * crnn_ctc.h -- C ABI of libcrnnctc.so: the H100 (sm_90a) CRNN+CTC hot path that stands
 * behind the model/solver API of ilovin/lstm_ctc_ocr.
 *
 * The reference has no C ABI of its own (it is pure Python on TensorFlow 1.0.1 + the
 * warp-ctc TF binding).  Each entry point below names the reference call site it replaces
 * (paths relative to the reference checkout).  Conventions follow warp-ctc's ctc.h:
 * status-code returns, no exceptions across the ABI, caller-owned device buffers and
 * workspace (size queried first), every call asynchronous on the caller's stream, no
 * hidden host synchronisation.  All pointers are DEVICE pointers unless marked host.
 * One host thread per handle (thread-compatible, not thread-safe).
 * These calls can be captured into a CUDA graph once the same call has run at the same shape, on a single-device model:
 * crnn_forward / _u8, crnn_forward_lines, crnn_forward_host (every compute_dtype; copy_stream joins the capture through the
 * events of its copy handshake), crnn_forward + crnn_backward in training mode, the three crnn_clip_*_step solvers (the step
 * number is baked into the graph), crnn_ctc_loss (shared-memory and workspace kernels), crnn_ctc_greedy, crnn_ctc_align,
 * crnn_lexicon_candidates and crnn_ctc_lexicon_score.
 */
#ifndef CRNN_CTC_H_
#define CRNN_CTC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* crnn_stream_t;   /* == cudaStream_t */
typedef struct crnn_model crnn_model;

enum crnn_status {
  CRNN_OK = 0,
  CRNN_INVALID_VALUE = 1,     /* bad shape / length / null pointer */
  CRNN_CUDA_ERROR = 2,        /* a CUDA runtime/driver call failed; see crnn_last_error() */
  CRNN_NOT_BOUND = 3,         /* model used before crnn_model_bind() */
  CRNN_UNSUPPORTED = 4,       /* shape outside what the sm_90a kernels implement */
  CRNN_WORKSPACE_TOO_SMALL = 5
};

int         crnn_version(void);
const char* crnn_status_string(int status);
const char* crnn_last_error(void);           /* host string, valid until the next failing call */

/* ------------------------------------------------------------------------------------------
 * CTC operator boundary.
 * Replaces warpctc_tensorflow.ctc(activations, flat_labels, label_lengths, input_lengths)
 * at lib/networks/network.py:653-654 (warp-ctc compute_ctc_loss semantics: softmax inside,
 * blank label 0 by default, cost = -log p(l|x), zero gradient for frames >= input_length,
 * infeasible alignment -> cost 0 and zero gradient).
 *   logits      [T,N,C] f32, unnormalised, time-major (lib/networks/network.py:126-128)
 *   grad        [T,N,C] f32 or NULL; receives grad_scale * d costs[n] / d logits
 *   flat_labels [sum(label_len)] i32, label_len [N] i32, input_len [N] i32
 *   costs       [N] f32
 * max_label_len is a host-side upper bound on label_len[] (chooses the states-per-lane
 * variant; labels longer than it make that sample's cost NaN).  C must be 64.
 * Validation (SURVEY 8(b)): a sample whose labels contain an id outside [0,C) or equal to `blank`, or whose label_len is
 * negative or above max_label_len, gets cost NaN and an all-zero gradient -- the kernels never index with such an id.
 * input_len is clamped to [0,T].  flat_labels MUST hold sum(label_len) entries (its length is not passed and cannot be
 * checked on the device; the Python wrappers check it).
 * Frame limits and the workspace.  Without a workspace alpha / beta live in shared memory (at most 200 KB per utterance),
 * so T is bounded per max_label_len:
 *   max_label_len <= 15: T <= 256 tensor-map kernel (CRNN_CTC_KERNEL=tma), T <= floor(51200 / (70 + 2*AS + ES)) fast
 *                        kernel (AS = (2*max_label_len+1)|1, ES = max_label_len|1: 348 at 15, 550 at 4), beyond that
 *                        the generic kernel to T <= 517; the largest supported T is the larger of 517 and the fast limit
 *   max_label_len 16..31: T <= 259;   32..63: T <= 130
 * Logits or a gradient not 16-byte aligned (4-byte alignment is enough) take the generic kernel (T <= 517 / 259 / 130).
 * Beyond these limits -- max_label_len up to 639 (S = 2L+1 <= 1279 states) and any T -- the workspace kernel runs, as
 * warp-ctc's GPU path does: crnn_ctc_workspace_size returns 0 where a shared-memory kernel serves the shape at any
 * alignment (max_label_len <= 63 and T <= 517 / 259 / 130), else 4 * N * T * (64 + S_pad) + 256 bytes (S_pad = 2L+1
 * rounded up to a multiple of 4: the log-softmax and alpha tables; any alignment); CRNN_UNSUPPORTED above max_label_len
 * 639 or when the per-utterance float count overflows an int or the total a size_t.  A call gets the kernel it gets with
 * no workspace, with the same bits, wherever that succeeds; otherwise the workspace kernel when workspace_bytes is at
 * least the size.  Its results are the same bits from run to run (no float atomics).  With neither, the call returns
 * CRNN_UNSUPPORTED without touching costs or grad; crnn_last_error() names T and the shared memory it needed (or
 * max_label_len above 63) and, when in range, the workspace bytes that would run it.  CRNN_CTC_KERNEL=long runs the
 * workspace kernel at every shape (the size query then returns its size everywhere).
 * ---------------------------------------------------------------------------------------- */
int crnn_ctc_workspace_size(int T, int N, int C, int max_label_len, size_t* bytes);
int crnn_ctc_loss(const float* logits, float* grad, const int* flat_labels, const int* label_len,
                  const int* input_len, int T, int N, int C, int blank, int max_label_len,
                  float grad_scale, float* costs, void* workspace, size_t workspace_bytes,
                  crnn_stream_t stream);

/* CTC forced alignment: the best path (Viterbi, max-plus form of the alpha recursion above) of a GIVEN labelling, where each
 * label sits in it and how sure the model is of each label.  Per utterance n, with y_t = softmax(logits[t,n,:]) (max
 * subtracted), the extended labelling l' = (blank, l_1, blank, ..., l_L, blank) of S = 2L+1 states and e_t(s) = log y_t(l'_s):
 *   v_0(0) = e_0(0), v_0(1) = e_0(1), every other state -inf;  v_t(s) = e_t(s) + max over P(s) of v_{t-1},
 *   P(s) = {s, s-1}, plus s-2 when l'_s != blank and l'_s != l'_{s-2} (the transitions of crnn_ctc_loss).
 * Ties: among predecessors s beats s-1, which beats s-2; at the end state S-1 beats S-2.  Natural log, f32 arithmetic
 * (lse_t = m + log(sum exp(x - m)) per frame, e = x - lse_t).
 *   logits        [T,N,C] f32, unnormalised, time-major; 4-byte alignment is enough
 *   labels        label_stride == 0: flat [sum(label_len)] i32, utterance n at offset sum(label_len[0..n)) (crnn_ctc_loss's layout);
 *                 label_stride > 0: dense rows [N, label_stride] i32 (the decoders' layout), row n holds its label_len[n] ids
 *   label_len [N], input_len [N] i32 (input_len clamped to [0,T] = T_n); blank in [0,C) (class 0 is what warp-ctc trains as blank)
 *   start, end    i32 and peak f32, indexed like `labels`: the best path is in label k's state 2k+1 during frames
 *                 [start[k], end[k]) -- at least one frame, spans ordered and disjoint, a blank frame between equal neighbours;
 *                 peak[k] = max over the span of y_t(l_k), the per-label confidence.  Dense rows are written in full: entries
 *                 past label_len[n] get -1 / -1 / 0.
 *   path_logprob  [N] f32: sum over t < T_n of e_t(pi_t) along the best path (log p of the best alignment, not of the labelling).
 * Edge cases: L = 0 -> the all-blank path, no spans (path_logprob 0 when T_n = 0).  Infeasible labelling (T_n < L + number of
 * adjacent equal pairs) -> path_logprob -inf, spans -1, peaks 0.  Invalid utterance, as in crnn_ctc_loss (an id outside [0,C)
 * or equal to `blank`, label_len negative, above max_label_len or, dense, above label_stride) -> path_logprob NaN, spans -1,
 * peaks 0; no invalid id is used as an index.
 * Frames to pixels: frame t is conv5 output t, which reads pooled columns t and t+1, so the span [s, e) covers input columns
 * [4s, 4e+4) of the line (3x3 halos aside).
 * Supported: C = 64 and max_label_len <= 639 (S <= 1279), any T; otherwise CRNN_UNSUPPORTED.  The workspace (any alignment; size
 * from crnn_ctc_align_workspace_size, no CUDA call) holds T * (8 + S_pad) bytes per utterance (S_pad = 2*max_label_len+1 rounded
 * up to 4) plus 256.  Every pointer is a device pointer; the call is asynchronous on `stream` and allocates nothing.  A short
 * workspace returns CRNN_WORKSPACE_TOO_SMALL, a null pointer CRNN_INVALID_VALUE; the outputs are then untouched.  The outputs do
 * not depend on what the outputs or the workspace held before, and a run gives the same bits every time (no float atomics). */
int crnn_ctc_align_workspace_size(int T, int N, int C, int max_label_len, size_t* bytes);
int crnn_ctc_align(const float* logits, const int* labels, int label_stride, const int* label_len, const int* input_len, int T, int N,
                   int C, int blank, int max_label_len, int* start, int* end, float* peak, float* path_logprob, void* workspace,
                   size_t workspace_bytes, crnn_stream_t stream);

/* Lexicon-based reading (CRNN's lexicon transcription, Shi, Bai & Yao, §2.3.2): for each line the lexicon entry l* that
 * maximises p(l | y), searched among the entries within edit distance max_edit of the lexicon-free read.  Two calls: the
 * candidates by edit distance, then their CTC scores.  The lexicon is caller-owned device CSR:
 *   lex_ids  i32, the entries' class ids concatenated;  lex_off [K+1] i32, entry k is lex_ids[lex_off[k] .. lex_off[k+1])
 *   max_entry_len  a host-side bound on every entry's length, at most 63 (else CRNN_UNSUPPORTED).  An entry longer than it (or
 *                  with lex_off decreasing) is never a candidate, and scores NaN.
 *
 * crnn_lexicon_candidates: reads [N, read_stride] i32 and read_len [N] i32 in the decoders' dense layout (engine.dense_decoded;
 * read_len clamped to [0, read_stride]).  d = the Levenshtein distance (unit insert, delete, substitute) between the read and an
 * entry, compared id for id; an id outside [0,64), in a read or an entry, matches nothing (not even itself) and is never used as
 * an index.  The candidates are the entries with d <= max_edit (max_edit < 0: no threshold), ordered by (d, lexicon index); the
 * first max_candidates (1 .. 256) are kept:
 *   cand [N, max_candidates] i32       the lexicon index, -1 past the count
 *   cand_dist [N, max_candidates] i32  d, -1 past the count
 *   cand_total [N] i32                 how many entries have d <= max_edit (all well-formed entries when max_edit < 0), so a
 *                                      truncated list is visible
 * Ties at the last kept distance go to the lower lexicon indices.  The outputs are the same bits run to run and do not depend
 * on what they held before (integer arithmetic, a fixed order; no workspace).  Supported: read_stride <= 1024 (the read is the
 * pattern of a bit-parallel Levenshtein kernel, 16 words of 64 rows), else CRNN_UNSUPPORTED.
 *
 * crnn_ctc_lexicon_score: score[n, j] = ln p(lex[cand[n, j]] | y_n), the sum over the CTC lattice of crnn_ctc_loss (same
 * transitions and `blank`; mathematically -cost of crnn_ctc_loss on that labelling), f32 in log2 arithmetic as crnn_ctc_loss
 * computes it (log2-softmax with the row maximum subtracted), returned in natural log.
 *   logits [T,N,C] f32, input_len [N] i32 (clamped to [0,T] = T_n); blank in [0,C) (0 is the blank warp-ctc trains);
 *   cand [N, max_candidates] i32 as crnn_lexicon_candidates writes it (any value below 0 is an empty slot; an index must be < K).
 *   score [N, max_candidates] f32;  best [N] i32: the lexicon index of the highest finite score, ties to the lowest slot (the
 *   nearer distance, then the lower index), -1 when no slot has a finite score;  best_score [N] f32: its score, or -inf.
 * Special values: an empty slot -> -inf; an infeasible labelling (T_n < L + number of adjacent equal pairs) -> -inf; L = 0 is the
 * all-blank path (0 when T_n = 0); an invalid entry (an id outside [0,C) or equal to `blank`, or longer than max_entry_len) ->
 * NaN.  No float atomics: the same bits run to run.
 * Supported: C = 64 and T <= 768 (the line's log2-softmax, 256 B per frame, is kept in shared memory and shared by all of its
 * candidates), otherwise CRNN_UNSUPPORTED with crnn_last_error() naming T or the entry length.
 * Both calls: every pointer a device pointer, asynchronous on `stream`, no allocation; a null pointer returns
 * CRNN_INVALID_VALUE and every status other than CRNN_OK leaves the outputs untouched. */
int crnn_lexicon_candidates(const int* reads, int read_stride, const int* read_len, int N, const int* lex_ids, const int* lex_off,
                            int K, int max_entry_len, int max_edit, int max_candidates, int* cand, int* cand_dist, int* cand_total,
                            crnn_stream_t stream);
int crnn_ctc_lexicon_score(const float* logits, const int* input_len, int T, int N, int C, int blank, const int* lex_ids,
                           const int* lex_off, int max_entry_len, const int* cand, int max_candidates, float* score, int* best,
                           float* best_score, crnn_stream_t stream);

/* Resize native-size 8-bit gray text lines to the network's 32 rows and pack them into the batch crnn_forward_lines_u8 takes.
 * Replaces the host step of lib/lstm/test.py (Image.resize((nw, 32), BILINEAR) per line, then pad and transpose): the result
 * is byte for byte Pillow's 8-bit BILINEAR on mode "L" -- the horizontal pass (src_w -> out_w) first, then the vertical pass
 * (src_h -> 32) on its u8 result, each skipped when its size is unchanged, integer taps of 22 fractional bits; a source more
 * than 100 times taller than wide takes the vertical pass first, as Pillow (12.2) does.
 *   src         u8; line i is src_h[i] x src_w[i] bytes, row-major, at src + src_offset[i] (any alignment)
 *   src_offset  [N] i64;  src_h, src_w, out_w [N] i32
 *   out         [N, W, 32] u8, 4-byte aligned: out[i, x, y] = resized line i at row y, column x for x < out_w[i]; every column
 *               from out_w[i] to W is written as zero, so `out` needs no clearing.
 * max_h is a host-side bound on every src_h[i] and sizes the launch: at most 1024 (CRNN_INVALID_VALUE outside [1, 1024]).
 * The per-line values are preconditions the call cannot check without a host sync: 1 <= src_h[i] <= max_h, src_w[i] >= 1,
 * 1 <= out_w[i] <= W, src_w[i] / out_w[i] <= max_h / 16 + 1 (the size rule below keeps it under src_h[i] / 16), and the bytes
 * of line i inside `src`.  A line whose height, widths or ratio break them gets an all-zero slot and is not read.
 * The size rule of the evaluation path (lib/lstm/test.py line_size): out_w = src_w if src_h == 32 else
 * max(1, (int)(32.0 / src_h * src_w)) in double arithmetic, computed on the host; the line's padded width is
 * max(8, ceil(out_w / 4) * 4) and its time_step_len max(out_w / 4 - 1, 0).
 * CRNN_INVALID_VALUE for a null pointer, N <= 0, W < 8, W % 4 != 0 or a misaligned `out`; CRNN_UNSUPPORTED for W above
 * 2 097 120.  Every pointer is a device pointer; asynchronous on `stream`, no allocation, the same bits on every run. */
int crnn_resize_lines_u8(const uint8_t* src, const int64_t* src_offset, const int* src_h, const int* src_w, const int* out_w, int N,
                         int W, int max_h, uint8_t* out, crnn_stream_t stream);

/* PNG files decoded to 8-bit gray on the device, byte for byte what the host reader of lib/lstm/test.py load_line_image gives:
 *   rule 0  cv2.imread(path, 0) (OpenCV 4.13 on libpng 1.6): colour (9797 R + 19234 G + 3737 B) >> 15 at 8 bits,
 *           ((9797 R + 19234 G + 3737 B + 16384) >> 15) >> 8 at 16 bits; 16-bit gray the high byte
 *   rule 1  Pillow 12.2 Image.convert("L"): colour (19595 R + 38470 G + 7471 B + 0x8000) >> 16 on the high bytes; 16-bit gray
 *           clipped to 255
 * Under both, alpha is dropped, gray below 8 bits is scaled by 255 / (2^d - 1), palette entries go through the colour formula
 * and 16-bit gray+alpha gives its high byte.  Every colour type, bit depth, Adam7 and DEFLATE block kind is read.
 *
 * The decoder is at least as strict as both readers: a file it accepts reads the same on the host.  Any irregularity, and any
 * chunk that makes a host reader compute something else, gives the file a non-zero status and an all-zero slot:
 *   CRNN_PNG_BAD_HEADER     no PNG signature, IHDR missing, invalid or unlike h[i] x w[i], more than 1024 rows, more than
 *                           1 000 000 columns or 178 956 970 pixels (beyond Pillow's decompression-bomb limit)
 *   CRNN_PNG_BAD_CHUNK      truncated chunk, bad length or type, unknown critical chunk, PLTE missing / misplaced / invalid,
 *                           IDAT not consecutive, IEND missing or bytes after it, an ancillary chunk of the wrong size or place
 *   CRNN_PNG_BAD_CRC        a chunk CRC (ancillary or critical)
 *   CRNN_PNG_BAD_ZLIB       zlib header (method, window, check bits, preset dictionary), Adler-32, bytes after the stream
 *   CRNN_PNG_BAD_DEFLATE    block type 3, a bad stored length, over-subscribed or incomplete codes, a code or distance out of
 *                           range, a distance past the window or the output, the stream ending early
 *   CRNN_PNG_BAD_SIZE       more or less image data than IHDR implies
 *   CRNN_PNG_BAD_DATA       a filter type above 4, a palette index at or beyond the PLTE length
 *   CRNN_PNG_HOST_DIFFERS   a chunk a host reader acts on: any ancillary chunk but cHRM, pHYs, tIME, sBIT, tRNS, bKGD, tEXt,
 *                           zTXt, iTXt, gAMA, sRGB and iCCP (so acTL / APNG and eXIf orientation among them); under rule 0
 *                           gAMA, sRGB or iCCP on a colour or palette file (libpng then gamma-corrects its gray conversion,
 *                           palette entries included); under rule 1 a zTXt, compressed iTXt or iCCP payload above 1016 bytes
 *                           (it may inflate past the 1 MiB Pillow refuses) or text chunks that may hold more than Pillow's
 *                           64 MiB in all
 *   CRNN_PNG_WORKSPACE      the file's workspace region is smaller than its plan or lies beyond `bytes`
 *
 * crnn_png_plan (host only) lays out the workspace: file i owns bytes [ws_offset[i], ws_offset[i+1]) of it, first its zlib
 * stream (the IDAT payloads gathered in order; file_len[i] rounded up to 16 bytes of room) and then its inflated scanlines (a
 * filter byte and the packed samples of every row of every non-empty Adam7 pass, in pass order; room rounded up to 16), whose
 * rows the call unfilters in place: after a successful call each row holds its samples, its filter byte unchanged.  A file whose 13 IHDR bytes are invalid gets an empty region.  ihdr is [N][13] (bytes 16 .. 28 of each
 * file), file_len [N], ws_offset [N + 1]; *workspace_bytes = ws_offset[N].  CRNN_INVALID_VALUE for a null pointer or N <= 0.
 *
 * crnn_png_decode_gray_u8: file i is file_len[i] bytes at files + file_offset[i]; its gray image, h[i] x w[i] bytes row-major,
 * goes to out + out_offset[i] (the src / src_offset / src_h / src_w layout crnn_resize_lines_u8 reads) and its status to
 * status[i].  ws_offset [N + 1] is crnn_png_plan's, on the device; `bytes` is the workspace's size.  One warp per file: chunk
 * walk with warp-wide CRC-32, inflate with warp-wide copies and Adler-32, unfilter, expand, convert and the Adam7 scatter.
 * file_offset, file_len, out_offset and ws_offset must be 8-byte aligned, h, w and status 4-byte aligned; files, out and the
 * workspace take any alignment.  CRNN_INVALID_VALUE for a null pointer, N <= 0, rule outside {0, 1} or a misaligned pointer,
 * and then nothing is written.  Every pointer but the host-side plan's is a device pointer; asynchronous on `stream`, no
 * allocation, the same bits on every run. */
enum crnn_png_status {
  CRNN_PNG_OK = 0,
  CRNN_PNG_BAD_HEADER = 1,
  CRNN_PNG_BAD_CHUNK = 2,
  CRNN_PNG_BAD_CRC = 3,
  CRNN_PNG_BAD_ZLIB = 4,
  CRNN_PNG_BAD_DEFLATE = 5,
  CRNN_PNG_BAD_SIZE = 6,
  CRNN_PNG_BAD_DATA = 7,
  CRNN_PNG_HOST_DIFFERS = 8,
  CRNN_PNG_WORKSPACE = 9
};
int crnn_png_plan(const uint8_t* ihdr, const int64_t* file_len, int N, int64_t* ws_offset, size_t* workspace_bytes);
int crnn_png_decode_gray_u8(const uint8_t* files, const int64_t* file_offset, const int64_t* file_len, int N, const int* h,
                            const int* w, const int64_t* out_offset, int rule, uint8_t* out, int* status, void* workspace,
                            const int64_t* ws_offset, size_t bytes, crnn_stream_t stream);

/* JPEG files decoded to 8-bit gray on the device, byte for byte what the host reader of lib/lstm/test.py load_line_image gives
 * (libjpeg-turbo 3.1, ISLOW IDCT):
 *   rule 0  cv2.imread(path, 0) (OpenCV 4.13): libjpeg's JCS_GRAYSCALE output, the Y plane; the chroma is entropy-decoded only
 *   rule 1  Pillow 12.2 Image.convert("L"): a 1-component file its Y plane; a colour file libjpeg-turbo's RGB decode (fancy
 *           upsampling, jdcolor.c's table-driven YCbCr -> RGB), then (19595 R + 38470 G + 7471 B + 0x8000) >> 16
 * Read: baseline and extended-sequential Huffman files (SOF0, SOF1), 8-bit, one scan holding every component, 1 component or 3
 * taken as YCbCr (a JFIF APP0, an Adobe APP14 with transform 1, or neither with component ids other than 'R', 'G', 'B'),
 * 1 .. 1024 rows, 1 .. 65535 columns, any restart interval, fill bytes, bytes after EOI (ignored).  Under rule 0 every sampling
 * is read whose Y carries the largest factors; under rule 1 every component's factors must divide the largest by 1 or 2.
 *
 * The decoder is at least as strict as both readers: a file it accepts reads the same on the host.  libjpeg-turbo warns and
 * goes on over much of what is refused here.  A refused file gets a non-zero status and an all-zero slot:
 *   CRNN_JPEG_BAD_HEADER    no SOI, SOS before SOF, an invalid SOF (length, sampling factors, component ids, quantisation table
 *                           index, more than 10 blocks per MCU), a size unlike h[i] x w[i] or beyond 1024 rows
 *   CRNN_JPEG_UNSUPPORTED   progressive, lossless, hierarchical or arithmetic-coded frames, precision other than 8, 2 or 4
 *                           components, RGB colour (Adobe transform 0, any other Adobe transform, or ids 'R', 'G', 'B'), the
 *                           components in several scans, a second scan, DNL or a zero height
 *   CRNN_JPEG_BAD_MARKER    a bad marker or segment length, a truncated or malformed DQT, DHT, DRI or SOS (spectral selection
 *                           and approximation other than 0, 63, 0), a table the scan needs missing, RSTn before the scan, a
 *                           marker after the scan other than RSTn and EOI, no EOI
 *   CRNN_JPEG_BAD_HUFFMAN   a DHT class above 1 or index above 3, more than 256 symbols, an over-subscribed code or an all-ones
 *                           code (libjpeg's jpeg_make_d_derived_tbl checks), a DC symbol above 15
 *   CRNN_JPEG_BAD_DATA      an invalid code, a coefficient index past 63, a DC category above 11 or an AC category above 10, a
 *                           segment that ends before its MCUs or holds bytes after them
 *   CRNN_JPEG_BAD_RESTART   an RSTn out of order, missing or beyond the last interval
 *   CRNN_JPEG_HOST_DIFFERS  rule 0: an Exif APP1 whose IFD0 orientation is not 1 or cannot be read (OpenCV turns the image), a
 *                           colour file whose Y lacks the largest sampling factors; rule 1: a sampling ratio other than 1 or 2;
 *                           both: a block outside the range where jidctint.c and libjpeg-turbo's SIMD IDCT (which the host
 *                           readers run) agree -- a dequantised coefficient or first-pass output beyond +-16383, or an output sum
 *                           outside [-512, 511], where jidctint.c's range-limit table wraps and the SIMD code saturates
 *   CRNN_JPEG_WORKSPACE     the file's workspace region is smaller than its plan, lies beyond `bytes` or starts off a 16-byte
 *                           boundary
 *
 * crnn_jpeg_plan (host only) lays out the workspace: file i owns bytes [ws_offset[i], ws_offset[i+1]) of it: a 512-byte record
 * (what the IDCT reads: block grids, quantisation tables), the restart segment table (8 bytes per MCU, plus 8), the int16
 * coefficients of each stored component (Y, or under rule 1 all three of a colour file; 64 per block in natural order, the block
 * grid padded to whole MCUs, a 1-component file's grid ceil(w / 8) x ceil(h / 8)), then under rule 1 a colour file's three
 * component planes (8 x 8 bytes per block).  Every size is a multiple of 16.  sof is [N][16]: each file's SOF payload after its
 * length field (precision, height, width, Nf, then id, sampling factors and table index per component), zero-filled to 16
 * bytes; a record the decoder cannot lay out gets an empty region.  file_len [N], ws_offset [N + 1]; *workspace_bytes =
 * ws_offset[N].  CRNN_INVALID_VALUE for a null pointer, N <= 0 or rule outside {0, 1}.
 *
 * crnn_jpeg_decode_gray_u8: file i is file_len[i] bytes at files + file_offset[i]; its gray image, h[i] x w[i] bytes row-major,
 * goes to out + out_offset[i] (the src / src_offset / src_h / src_w layout crnn_resize_lines_u8 reads) and its status to
 * status[i].  ws_offset [N + 1] is crnn_jpeg_plan's for the same rule, on the device; `bytes` is the workspace's size.  Three
 * kernels: jpeg_entropy_kernel (one warp per file: marker walk, Huffman tables, RSTn scan, one restart segment per lane),
 * jpeg_idct_kernel (ISLOW, 8 threads per block), jpeg_finish_kernel (zero slots of refused files; rule 1 colour conversion).
 * file_offset, file_len, out_offset and ws_offset must be 8-byte aligned, h, w and status 4-byte aligned, the workspace 16-byte
 * aligned; files and out take any alignment.  CRNN_INVALID_VALUE for a null pointer, N <= 0, rule outside {0, 1} or a
 * misaligned pointer, and then nothing is written.  Every pointer but the host-side plan's is a device pointer; asynchronous on
 * `stream`, no allocation, the same bits on every run. */
enum crnn_jpeg_status {
  CRNN_JPEG_OK = 0,
  CRNN_JPEG_BAD_HEADER = 1,
  CRNN_JPEG_UNSUPPORTED = 2,
  CRNN_JPEG_BAD_MARKER = 3,
  CRNN_JPEG_BAD_HUFFMAN = 4,
  CRNN_JPEG_BAD_DATA = 5,
  CRNN_JPEG_BAD_RESTART = 6,
  CRNN_JPEG_HOST_DIFFERS = 7,
  CRNN_JPEG_WORKSPACE = 8
};
int crnn_jpeg_plan(const uint8_t* sof, const int64_t* file_len, int N, int rule, int64_t* ws_offset, size_t* workspace_bytes);
int crnn_jpeg_decode_gray_u8(const uint8_t* files, const int64_t* file_offset, const int64_t* file_len, int N, const int* h,
                             const int* w, const int64_t* out_offset, int rule, uint8_t* out, int* status, void* workspace,
                             const int64_t* ws_offset, size_t bytes, crnn_stream_t stream);

/* Training lines rendered on the device.  Replaces the host generator (lib/lstm/utils/gen.py render_line + groupBatch, the
 * reference's gen.py:31-110): a batch's random layout, its glyphs composited with Pillow's blend arithmetic into 60-row
 * canvases, and the Pillow BILINEAR resize of crnn_resize_lines_u8 into the [N, W, 32] uint8 batch groupBatch(..., uint8)
 * builds.  Every pixel equals what Pillow draws (ImageDraw's draw_bitmap of each glyph mask) and resizes for the layout the
 * call reports.
 *
 * Glyph atlas (built on the host from one PIL font, lstm_ctc_ocr_b200.engine.GlyphAtlas): glyphs [nglyphs][8] i32 rows
 *   (advance int(getlength), mask width w, mask height h, offset ox, offset oy, byte offset of the mask in `masks`, 0, 0);
 *   masks: each glyph's w x h anti-aliased mask (getmask2(ch, "L", anchor="la")), row-major.  Charset index c is label id c + 1.
 *
 * crnn_render_layout: the layouts of lines 0 .. N-1 of the stream `seed`, from Philox4x64-10 with key (seed, 0x43524e4e52454e44)
 * and counter (line, attempt, block, 0).  An integer in [a, b] is a + ((u * (b - a + 1)) >> 64) of one 64-bit word u; its bias
 * is below 2^-57.  Words: block 0 gives the length U[min_len, max_len] (w0), the background U[180, 255] (w1) and x0 U[2, 12]
 * (w2); block 1 + j gives glyph j's charset index U[0, nglyphs-1] (w0), y U[0, 10] (w1), fill U[0, 90] (w2) and advance
 * jitter dx U[-2, 3] (w3).  Glyph j is drawn at x_j (x_0 = x0, x_{j+1} = x_j + advance_j + dx_j), y_j on a canvas of 60 rows and
 * sum(advance) + 28 columns; nw = (int)(32.0 / 60 * canvas_w) in double, time_step = nw / 4 - 1.  nw_hi > 0 makes the stream
 * bucketed: line i is redrawn with attempt + 1 until nw_lo < nw <= nw_hi, at most 256 attempts; nw_hi = 0: no bucket.
 *   layout  [N][8 + 4 * max_len] i32: length, background, x0, canvas width, nw, time_step, flat label offset, attempt, then
 *           label ids [max_len], x [max_len], y [max_len], fill [max_len] (entries past the length are unspecified)
 *   feeds   [4 + 2N + N * max_len] i32: [0] lines that found no width in the bucket within 256 attempts (0 = every line fits),
 *           [1] max nw, [2] labels in total, [3] padded width (nw_hi, else max(8, max nw rounded up to 4)), then label_len [N],
 *           time_step [N] and the flat labels (label ids 1 .. nglyphs).  One copy of it gives every integer feed of the batch.
 * CRNN_INVALID_VALUE for a null pointer, N <= 0, min_len < 1 or max_len < min_len, nglyphs outside [1, 62], or a bucket with
 * nw_hi < 8, nw_hi % 4 != 0 or nw_lo outside [0, nw_hi); CRNN_UNSUPPORTED for max_len > 256.
 *
 * crnn_render_lines_u8: the batch of `layout` (crnn_render_layout's output for N lines of max_len): each canvas filled with its
 * background, then glyph j's mask blended in draw order at (x_j + ox, y_j + oy), clipped to the canvas on every side, as Pillow's
 * fill_mask_L does: out = DIV255(out * (255 - m) + fill * m), DIV255(v) = (((v + 128) >> 8) + v + 128) >> 8.  The canvases are
 * then resized to nw x 32 and written to out [N, W, 32] u8 (4-byte aligned) exactly as crnn_resize_lines_u8 writes, columns nw
 * .. W-1 zero.  W: the padded width (feeds[3]), a multiple of 4 and >= 8.  max_adv bounds every advance of the atlas and sizes
 * the canvases: workspace (256-byte aligned) of crnn_render_workspace_size(N, max_len, max_adv) bytes.  A record whose canvas
 * does not fit that bound gets an all-zero slot.
 * CRNN_INVALID_VALUE for a null pointer, N <= 0, max_len < 1, max_adv < 1, a bad W or a misaligned out / workspace;
 * CRNN_UNSUPPORTED for max_len > 256 or widths beyond the launch grid; CRNN_WORKSPACE_TOO_SMALL.  Every pointer is a device
 * pointer; asynchronous on `stream`, no allocation, the same bits on every run; a failing call leaves the outputs untouched. */
int crnn_render_layout(int64_t seed, int N, int min_len, int max_len, int nw_lo, int nw_hi, const int* glyphs, int nglyphs,
                       int* layout, int* feeds, crnn_stream_t stream);
int crnn_render_workspace_size(int N, int max_len, int max_adv, size_t* bytes);
int crnn_render_lines_u8(const int* layout, int N, int max_len, const int* glyphs, const uint8_t* masks, int max_adv, int W,
                         void* workspace, size_t workspace_bytes, uint8_t* out, crnn_stream_t stream);

/* Greedy decode.  Replaces tf.nn.ctc_*_decoder(merge_repeated=True) + sparse_tensor_to_dense
 * at lib/networks/network.py:656-657 and the zero stripping of lib/lstm/utils/training.py:32:
 * per frame argmax (lowest index on ties) for t < input_len; emit iff != tf_blank and != the
 * previous raw argmax; drop `strip`.  out [N,T] i32 zero padded, out_len [N] i32.  logits need 4-byte alignment only. */
int crnn_ctc_greedy(const float* logits, const int* input_len, int T, int N, int C, int tf_blank,
                    int strip, int* out, int* out_len, crnn_stream_t stream);

/* Beam-search decode on the HOST.  Replaces tf.nn.ctc_beam_search_decoder(logits, seq_len, merge_repeated=True)
 * (beam_width 100, top_paths 1, blank = C-1) + sparse_tensor_to_dense(default 0) at lib/networks/network.py:656-657 and
 * lib/lstm/test.py:30-31.  The reference's op is a CPU-only TensorFlow kernel used at validation / evaluation time; so is
 * this one: ALL pointers are HOST pointers (copy the logits back once), utterances are spread over `num_threads` host
 * threads (0 = hardware concurrency).  logits [T,N,C] f32 unnormalised; out [N,T] i32 zero padded (labels equal to `strip`
 * dropped, lib/lstm/utils/training.py:32); out_len [N]; neg_log_prob [N] or NULL (-log P of the best prefix). */
int crnn_ctc_beam_search(const float* logits_host, const int* input_len_host, int T, int N, int C, int beam_width,
                         int merge_repeated, int strip, int* out_host, int* out_len_host, float* neg_log_prob_host,
                         int num_threads);

/* The same beam-search decode on the DEVICE: labellings identical to crnn_ctc_beam_search on the same logits (the
 * algorithm, its visit order and its tie rules are those of the host decoder; the double exp / log are the device's).  Same
 * layouts and meanings, but every pointer is a DEVICE pointer: logits [T,N,C] f32, input_len [N] i32, out [N,T] i32 zero
 * padded, out_len [N] i32, neg_log_prob [N] f32 or NULL.  Asynchronous on `stream`; no host synchronisation and no
 * allocation inside the call.  input_len is clamped to [0,T] (it cannot be checked without a sync): a negative length
 * decodes as 0 frames, one above T as T frames.  Supported: 2 <= C <= 64, 1 <= beam_width <= 128, else CRNN_UNSUPPORTED.
 * The workspace (16-byte aligned, size from crnn_ctc_beam_workspace_size, CRNN_WORKSPACE_TOO_SMALL when short) holds each
 * utterance's prefix tree: 64 bytes per entry, 1 + beam_width*(T+C) entries per utterance, a bound that depends on the
 * shapes alone (about 0.83 GB at T = 63, N = 1024, C = 64, width 100). */
int crnn_ctc_beam_workspace_size(int T, int N, int C, int beam_width, size_t* bytes);
int crnn_ctc_beam_search_device(const float* logits, const int* input_len, int T, int N, int C, int beam_width,
                                int merge_repeated, int strip, int* out, int* out_len, float* neg_log_prob,
                                void* workspace, size_t workspace_bytes, crnn_stream_t stream);

/* The n best labellings of each utterance: tf.nn.ctc_beam_search_decoder's top_paths, on the host (crnn_ctc_beam_search's
 * pointers and threads) and on the device (crnn_ctc_beam_search_device's pointers, limits, workspace and stream rules).  The
 * beam runs exactly as in the single-best decoders; after the last frame the entries it lists (at most beam_width, the empty
 * prefix and entries of total -inf included) are ranked by total, highest first, exact ties broken by insertion order,
 * earliest first (TensorFlow leaves the order of exact ties undefined).  Path 0 is therefore the single-best decoders' output,
 * bit for bit.  Path i is entry i's labels, consecutive equal labels merged when merge_repeated is set, `strip` dropped, zero
 * padded to T: two different prefixes can give the same labels ("a a" and "a" with merge_repeated), and both are returned.
 * out [N, top_paths, T] i32; out_len [N, top_paths] i32; log_prob [N, top_paths] f32 or NULL: the entry's total, log P <= 0
 * (TensorFlow's log_probability; note the sign is that of neither neg_log_prob above); num_paths [N] i32 or NULL: the paths
 * that are real, min(top_paths, listed entries).  Paths past num_paths have length 0 and log_prob -inf (where TensorFlow fails
 * the op).  1 <= top_paths <= beam_width, else CRNN_INVALID_VALUE. */
int crnn_ctc_beam_search_topk(const float* logits_host, const int* input_len_host, int T, int N, int C, int beam_width,
                              int top_paths, int merge_repeated, int strip, int* out_host, int* out_len_host,
                              float* log_prob_host, int* num_paths_host, int num_threads);
int crnn_ctc_beam_search_topk_device(const float* logits, const int* input_len, int T, int N, int C, int beam_width,
                                     int top_paths, int merge_repeated, int strip, int* out, int* out_len, float* log_prob,
                                     int* num_paths, void* workspace, size_t workspace_bytes, crnn_stream_t stream);

/* 1 when `host_ptr` lies in page-locked (cudaHostAlloc / cudaHostRegister) memory, else 0.  The Python feed path uses it to
 * decide whether a fed numpy batch can be DMA'd in place (crnn_forward_host) or has to be staged. */
int crnn_host_is_pinned(const void* host_ptr);

/* ------------------------------------------------------------------------------------------
 * Model boundary.  Replaces the graph built by lib/networks/LSTM_train.py:22-38 through
 * lib/networks/network.py (conv_single :160-191, max_pool :343-350, reshape_squeeze_layer
 * :361-368, bi_lstm :97-129) and executed by sess.run at lib/lstm/train.py:129-130.
 * ---------------------------------------------------------------------------------------- */
typedef struct crnn_config {
  int   img_height;     /* cfg.IMG_HEIGHT = 32        (lib/lstm/config.py:19) */
  int   nclasses;       /* cfg.NCLASSES   = 64        (lib/lstm/config.py:23) */
  int   num_hid;        /* cfg.TRAIN.NUM_HID = 512    (lib/lstm/config.py:48) */
  float bn_eps;         /* 1e-3  tf.contrib.layers.batch_norm default */
  float weight_decay;   /* cfg.TRAIN.WEIGHT_DECAY (lstm/lstm.yml:13 -> 1e-5) */
  int   compute_dtype;  /* 1 = bf16 operands / f32 accumulate (wgmma bf16): the throughput path, forward + backward.
                         * 2 = f32-class: every operand split into bf16 hi + bf16 lo, three bf16 products per term, f32
                         *     accumulate and f32 elementwise math (the reference computes in fp32, LSTM_train.py:10);
                         *     forward + CTC only (BASELINE configs[1])
                         * 3 = tf32: the same forward-only orchestration on tf32 wgmma operands (f32 tensors, rounded to
                         *     nearest tf32 where produced; 10-bit mantissa, one pass over K at half the bf16 rate)
                         * 4 = fp8, inference only: conv3_1, conv3_2, conv4_1, conv4_2 and conv5 run on e4m3 wgmma operands
                         *     (twice the bf16 tensor rate); everything else is the bf16 path.  Weights get one scale per
                         *     output channel (amax / 448); each of the five activation operands one power-of-two scale that
                         *     crnn_model_calibrate_fp8 or crnn_model_set_fp8_scales provides (see below) */
} crnn_config;

/* Not on the hot path: an fp8 model's creation synchronises the device after zeroing its e4m3 weight and scale block, so that
 * work on any stream afterwards (a non-blocking one included) sees the block zeroed before it writes it. */
int     crnn_model_create(const crnn_config* cfg, crnn_model** out);
int     crnn_model_destroy(crnn_model* m);

/* Trainable tensors, addressable by TF variable name and laid out exactly as the reference
 * checkpoint has them (HWIO conv kernels, [768,1024] LSTM matrices with gate order i,j,f,o;
 * SURVEY §8(a)).  All live in ONE flat f32 buffer owned by the caller. */
int     crnn_num_tensors(const crnn_model* m);
int64_t crnn_param_count(const crnn_model* m);
int     crnn_param_info(const crnn_model* m, int index, const char** tf_name, int64_t* offset,
                        int64_t shape[4], int* ndim);
/* Bind caller-owned flat buffers (each crnn_param_count() f32).  grads/adam_* may be NULL
 * for inference.  Marks the derived bf16 operand copies dirty.  Each non-null pointer must be 16-byte aligned (bias rows and the
 * solver steps read them as float4): otherwise CRNN_INVALID_VALUE and the previous binding stays. */
int     crnn_model_bind(crnn_model* m, float* params, float* grads, float* adam_m, float* adam_v);
int     crnn_model_params_changed(crnn_model* m);   /* caller wrote params in place */

/* The workspace is scratch, as in warp-ctc: its contents before a forward (crnn_forward*, crnn_forward_lines,
 * crnn_model_calibrate_fp8) do not matter, so a caller may use the same memory for anything else between calls, at the same
 * (N, W, pointer) too.  One exception: between a training forward and its crnn_backward the workspace holds what the
 * backward reads and must not be touched. */
int     crnn_model_workspace_size(const crnn_model* m, int N, int W, int train, size_t* bytes);

/* data [N,W,32] f32 (width-major rows, lib/lstm/utils/gen.py:62-64), time_step_len [N] i32
 * (nw//4-1, gen.py:54) -> logits_out [T=W/4-1, N, 64] f32.  workspace 1024-byte aligned.
 * Alignment (every forward entry point, crnn_model_calibrate_fp8 and crnn_backward): the f32 `data` / `data_staging` the kernels
 * read and `logits_out` must be 16-byte aligned (float4 loads and stores); otherwise CRNN_INVALID_VALUE, checked on the host
 * before anything is enqueued, and the outputs are untouched.  Host pointers (host_data, pageable_data, pinned_staging) may
 * have any alignment. */
int     crnn_forward(crnn_model* m, const float* data, const int* time_step_len, int N, int W,
                     float* logits_out, void* workspace, size_t workspace_bytes,
                     crnn_stream_t stream);

/* Same forward, fed from PAGE-LOCKED HOST memory (the reference feeds host numpy arrays through feed_dict every iteration,
 * lib/lstm/train.py:121-130).  The batch is copied in `chunks` image ranges on `copy_stream` into the caller-owned device
 * tensor `data_staging` [N,W,32] while the batch-independent front end (conv1 .. conv3_2) of the previous range runs on
 * `stream`; from the first batch-statistics BatchNorm on the batch is processed whole.  chunks <= 1 (or a batch that does not
 * split on tile boundaries) degenerates to copy-then-compute.  `data_staging` holds the whole batch on return order of
 * `stream` (crnn_backward reads it).  Whatever the compute_dtype, every copy out of `host_data` runs on `copy_stream`
 * (after the work queued earlier on `stream`): the caller may rewrite `host_data` once the work queued on `copy_stream`
 * has completed. */
int     crnn_forward_host(crnn_model* m, const float* host_data, float* data_staging, const int* time_step_len,
                          int N, int W, float* logits_out, void* workspace, size_t workspace_bytes, int chunks,
                          crnn_stream_t stream, crnn_stream_t copy_stream);

/* Same forward, fed from ORDINARY (pageable) host memory -- the reference's solver builds a fresh np.array(...) batch every
 * iteration (lib/lstm/train.py:119-125).  Every image range is first moved into the caller's page-locked `pinned_staging`
 * [N,W,32] by `host_threads` host threads (a persistent pool inside the library), then DMA'd and processed as in
 * crnn_forward_host; the host moves range c+1 while the GPU copies / computes range c.  The caller must not touch
 * `pinned_staging` until the copies issued on `copy_stream` have completed; whatever the compute_dtype, every copy out of it
 * runs there, so `pinned_staging` may be reused once the work queued on `copy_stream` has completed. */
int     crnn_forward_pageable(crnn_model* m, const float* pageable_data, float* pinned_staging, float* data_staging,
                              const int* time_step_len, int N, int W, float* logits_out, void* workspace,
                              size_t workspace_bytes, int chunks, int host_threads, crnn_stream_t stream,
                              crnn_stream_t copy_stream);

/* Packed evaluation: N text lines of different widths in one call, each computed as if it were fed alone to crnn_forward as
 * [1, W_i, 32].  data [N,W,32] f32: line i in columns [0, W_i) of its slot (columns past W_i are ignored); line_width [N] i32 =
 * W_i, clamped on the device to [8, W] and rounded down to a multiple of 4; time_step_len [N] i32 -> logits_out [W/4-1, N, 64].
 * Every SAME convolution sees zero padding at the line's own right edge, and conv4_1 / conv4_2 normalise with the line's own
 * batch statistics (count W_i, like the reference's one-line-per-run evaluation, lib/lstm/test.py).  Only frames t < W_i/4 - 1
 * are defined: time_step_len[i] must be <= W_i/4 - 1; like input_len elsewhere it cannot be checked without a sync.
 * All pointers are device pointers; asynchronous on `stream`, no allocation.  The workspace (crnn_lines_workspace_size) is
 * the inference plan's plus the per-line statistics and coefficients (about 33 MB more at N = 1024).
 * CRNN_INVALID_VALUE for a model in training mode (training uses whole-batch statistics) and the shape errors of
 * crnn_forward; CRNN_UNSUPPORTED for compute_dtype 2 or 3.  crnn_debug_tap / _raw read this forward afterwards. */
int     crnn_lines_workspace_size(const crnn_model* m, int N, int W, size_t* bytes);
int     crnn_forward_lines(crnn_model* m, const float* data, const int* line_width, const int* time_step_len, int N, int W,
                           float* logits_out, void* workspace, size_t workspace_bytes, crnn_stream_t stream);

/* fp8 models (compute_dtype 4).  The scales of the five e4m3 activation operands -- conv2's pooled output a2, conv3_1's a3,
 * conv3_2's pooled a3p and the BatchNorm + ReLU outputs a4a (conv4_1) and a4b (conv4_2, pooled) -- are
 *   s = 2^max(-126, ceil(log2(amax / 448)))   (the f32 quotient; 1 when amax is 0 or not finite)
 * so that dividing by them is exact; values above the calibrated range saturate to +-448.
 * crnn_model_calibrate_fp8 runs the bf16 forward's front end (conv1 .. conv4_2's BatchNorm) on a caller-supplied batch (the
 * layouts of crnn_forward; the workspace of crnn_model_workspace_size(train = 0)) and reduces the five amaxes on the device:
 * asynchronous, no host sync, no allocation (an fp8 model allocates its e4m3 weights and scales in crnn_model_create),
 * deterministic.  Any parameter change (crnn_model_bind, crnn_model_params_changed)
 * invalidates the scales; an fp8 forward without valid scales returns CRNN_INVALID_VALUE ("calibration is missing") and leaves
 * its outputs untouched.  get and set (host arrays of 5 floats; set refuses anything but powers of two in [2^-126, 2^127] with
 * CRNN_INVALID_VALUE) restate them; both synchronise the device, set before and after its write, so that a forward on any
 * stream afterwards reads the new scales.  On a model of another compute_dtype all three return CRNN_UNSUPPORTED.
 * crnn_forward, _host and _pageable (copy, then compute) and crnn_forward_lines run the fp8 path on an fp8 model;
 * crnn_model_set_training(m, 1) and a training workspace return CRNN_UNSUPPORTED. */
int     crnn_model_calibrate_fp8(crnn_model* m, const float* data, const int* time_step_len, int N, int W, void* workspace,
                                 size_t workspace_bytes, crnn_stream_t stream);
int     crnn_model_get_fp8_scales(crnn_model* m, float* scales_host);
int     crnn_model_set_fp8_scales(crnn_model* m, const float* scales_host);

/* Moving BatchNorm statistics of conv4_1 / conv4_2 -- the moving_mean / moving_variance that tf.contrib.layers.batch_norm creates
 * next to gamma / beta (the reference's conv_single, lib/networks/network.py:176-178, trains and evaluates with is_training=True and
 * never updates them).  `moving` is a caller-owned device buffer f32 [2 layers][mean, variance][512]; TF initialises it to mean 0,
 * variance 1.  Once bound (NULL unbinds), every crnn_backward updates it once, before anything else, from the f64 sums its training
 * forward normalised with (over the global batch when data parallel, so every rank computes the same bits), per channel:
 *   moving -= (moving - batch value) * (1 - decay)      (TF's assign_moving_average without zero-debias)
 * with the batch mean and the population (biased) variance, every operation in f64 from the stored f32 value, rounded once to f32;
 * 1 - decay is taken in f64 from the f32 decay (0.999f: 1 - decay is 1.3e-5 below TF's f32 1e-3).
 * Forwards never update it: training forwards that no crnn_backward follows (validation), evaluation and fp8 calibration.
 * crnn_model_set_bn_statistics(m, 1) makes evaluation forwards normalise with it:  y = relu(gamma * (conv(x) + b - mean) /
 * sqrt(var + bn_eps) + beta).  The BatchNorm folds into the conv: s = gamma / sqrt(var + eps) in f64, W' = bf16(W * s) per output
 * channel and b' = f32((b - mean) * s + beta), each rounded once; conv4_1 then runs as conv3_1's ReLU GEMM and conv4_2 as
 * conv3_2's ReLU + pool GEMM, with no batch statistics, finalize or apply pass.  Each image's (and, in crnn_forward_lines, each
 * line's) logits no longer depend on the rest of the batch.  fp8 models fold s into conv4_x's column scales (colscale x s, f64
 * product rounded once) and the same b'; the e4m3 weights stay.  The folded operands are kept apart from the batch-mode ones and
 * are re-derived on the next moving-mode forward after a parameter change, a bind, a backward or a mode change; a caller that
 * writes `moving` in place calls crnn_model_params_changed.  0 (the default, the reference's behaviour) = batch statistics.
 * Training forwards always use batch statistics.  Errors: set_bn_statistics(m, 1) on a model in training mode
 * CRNN_INVALID_VALUE; a moving-mode forward with no buffer bound CRNN_NOT_BOUND; compute_dtype 2 or 3 CRNN_UNSUPPORTED (both
 * calls); decay outside [0, 1] CRNN_INVALID_VALUE.  Binding a buffer and changing the mode invalidate an fp8 model's activation
 * scales, as a parameter change does: calibrate again in the mode that will be evaluated (crnn_model_calibrate_fp8 runs the
 * mode's own conv4_x).  After a moving-mode forward the taps "a4a_pre", "a4b_pre", "bn" and "stats" return CRNN_INVALID_VALUE;
 * crnn_debug_tap_raw adds "moving_w_conv4_1" / "moving_w_conv4_2" (bf16 W' [512][K], K = 2304 / 4608 in (kh, kw, ci) order) and
 * "moving_bias" (f32 b' [2][512]), and on fp8 models "fp8_colscale_moving" (f32 [2][512]).  crnn_lines_workspace_size depends
 * on the mode: with moving statistics it holds no per-line statistics.  `moving` must be 4-byte aligned (CRNN_INVALID_VALUE
 * otherwise, the previous binding stays). */
int     crnn_model_bind_bn_moving(crnn_model* m, float* moving, float decay);
int     crnn_model_set_bn_statistics(crnn_model* m, int moving);   /* 0 = batch statistics (default, the reference), 1 = moving */

/* The host-side copy crnn_forward_pageable uses, on its own: `bytes` from `src` to `dst` (plain host pointers, non-overlapping) split
 * over `threads` threads of the library's persistent pool (the caller's thread included).  No CUDA call is made. */
int     crnn_host_copy(void* dst, const void* src, size_t bytes, int threads);

/* loss = mean_n(costs) + weight_decay * 0.5 * sum(w^2) over conv kernels + logits matrix
 * (lib/networks/network.py:655,660-662).  loss_out: 1 f32 on device. */
int     crnn_total_loss(crnn_model* m, const float* costs, int N, float* loss_out,
                        crnn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * uint8 feed.  Every text line starts as an 8-bit gray image (the reference reads cv2.imread(..., 0) and resizes it with PIL,
 * still uint8); these twins take those bytes instead of the f32 `data`, a quarter of the host memory traffic, PCIe and device
 * bytes.  u [N,W,32] uint8 has the layout of the f32 data (width-major rows, lib/lstm/utils/gen.py:62-64), and the input value
 * of a byte is
 *     x = (float)u / 255.0f      (IEEE round-to-nearest division; numpy: u.astype(np.float32) / np.float32(255))
 * -- the value the f32 data tensor holds for that pixel, so conv1 gets the same operands and everything downstream is the same
 * computation on the same values (a reciprocal multiply would differ on 126 of the 256 bytes).  Each twin takes the arguments
 * and returns the status codes of its f32 entry point; only data, host_data and the staging buffers are uint8_t (the staging
 * buffers of _host_u8 / _pageable_u8 hold N*W*32 bytes).  Copies are sized by the byte count; the chunking rule is unchanged.
 * The device pointer the kernels read (data, data_staging) must be 4-byte aligned: otherwise CRNN_INVALID_VALUE and the
 * outputs are untouched.  _lines_u8 ignores the bytes past each line's width, as crnn_forward_lines ignores those columns.
 * ---------------------------------------------------------------------------------------- */
int     crnn_forward_u8(crnn_model* m, const uint8_t* data, const int* time_step_len, int N, int W, float* logits_out,
                        void* workspace, size_t workspace_bytes, crnn_stream_t stream);
int     crnn_forward_host_u8(crnn_model* m, const uint8_t* host_data, uint8_t* data_staging, const int* time_step_len, int N, int W,
                             float* logits_out, void* workspace, size_t workspace_bytes, int chunks, crnn_stream_t stream,
                             crnn_stream_t copy_stream);
int     crnn_forward_pageable_u8(crnn_model* m, const uint8_t* pageable_data, uint8_t* pinned_staging, uint8_t* data_staging,
                                 const int* time_step_len, int N, int W, float* logits_out, void* workspace, size_t workspace_bytes,
                                 int chunks, int host_threads, crnn_stream_t stream, crnn_stream_t copy_stream);
int     crnn_forward_lines_u8(crnn_model* m, const uint8_t* data, const int* line_width, const int* time_step_len, int N, int W,
                              float* logits_out, void* workspace, size_t workspace_bytes, crnn_stream_t stream);
int     crnn_model_calibrate_fp8_u8(crnn_model* m, const uint8_t* data, const int* time_step_len, int N, int W, void* workspace,
                                    size_t workspace_bytes, crnn_stream_t stream);
int     crnn_backward_u8(crnn_model* m, const uint8_t* data, const int* time_step_len, const float* dlogits, int N, int W,
                         void* workspace, size_t workspace_bytes, crnn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Training.  Replaces tf.gradients + tf.clip_by_global_norm(., 10.0) + {Adam, RMSProp, Momentum}Optimizer.apply_gradients
 * (lib/lstm/train.py:73-83).  Protocol per step:
 *   crnn_model_set_training(m, 1) once; crnn_forward (saves what the backward needs in the workspace);
 *   crnn_ctc_loss with grad != NULL and grad_scale = 1/N  -> dlogits;  crnn_backward -> flat `grads` buffer;
 *   [data parallel: all-reduce(SUM) `grads` across ranks];  crnn_clip_adam_step (or _momentum_step / _rmsprop_step).
 * ---------------------------------------------------------------------------------------- */
int     crnn_model_set_training(crnn_model* m, int flag);
/* dlogits [T,N,64] f32, 16-byte aligned (read as float4); f32 data 16-byte aligned as in crnn_forward: otherwise
 * CRNN_INVALID_VALUE and `grads` is untouched. */
int     crnn_backward(crnn_model* m, const float* data, const int* time_step_len, const float* dlogits,
                      int N, int W, void* workspace, size_t workspace_bytes, crnn_stream_t stream);
/* grads += weight_decay*wd_mul*w on the L2-regularised tensors (network.py:660-662); g *= grad_mul;
 * g *= clip/max(||g||, clip); TF Adam: lr_t = lr*sqrt(1-b2^step)/(1-b1^step), theta -= lr_t*m/(sqrt(v)+1e-8).
 * Single GPU: grad_mul = wd_mul = 1.  Data parallel after a SUM all-reduce: grad_mul = 1/world, wd_mul = world. */
int     crnn_clip_adam_step(crnn_model* m, float lr, float clip, int step, float grad_mul, float wd_mul,
                            crnn_stream_t stream);
/* The reference's other two solvers (cfg.TRAIN.SOLVER, lib/lstm/train.py:73-76), with the same gradient finish, averaging and
 * global-norm clip as crnn_clip_adam_step (same grad_mul / wd_mul meaning); g below is the clipped gradient.  Their state lives
 * in the two slot buffers bound through crnn_model_bind:
 *   Momentum (TF MomentumOptimizer, no Nesterov): adam_m holds accum (initialise to 0; adam_v is not used and may be NULL).
 *     accum = accum*momentum + g;  theta -= lr*accum.
 *   RMSProp (TF RMSPropOptimizer, not centred; TF's defaults decay 0.9, momentum 0, epsilon 1e-10): adam_m holds mom
 *     (initialise to 0), adam_v holds ms, which THE CALLER MUST INITIALISE TO 1.0 as TF does.
 *     ms += (g*g - ms)*(1 - decay);  mom = mom*momentum + lr*g/sqrt(ms + epsilon);  theta -= mom.
 * CRNN_NOT_BOUND when params, grads or a slot the solver uses is not bound; CRNN_INVALID_VALUE for momentum < 0, decay outside
 * [0, 1], epsilon < 0, or no prior crnn_model_set_training(m, 1).  crnn_last_grad_norm reports the norm of either step. */
int     crnn_clip_momentum_step(crnn_model* m, float lr, float momentum, float clip, float grad_mul, float wd_mul,
                                crnn_stream_t stream);
int     crnn_clip_rmsprop_step(crnn_model* m, float lr, float decay, float momentum, float epsilon, float clip,
                               float grad_mul, float wd_mul, crnn_stream_t stream);
int     crnn_last_grad_norm(crnn_model* m, float grad_mul, float* out_host, crnn_stream_t stream);   /* syncs */

/* ------------------------------------------------------------------------------------------
 * Data parallelism (one process per GPU; SURVEY 8(e)).  The reference is single-device: its BatchNorm sees the whole batch
 * (lib/networks/network.py:177-178) and its optimizer the whole-batch gradient (lib/lstm/train.py:81-83).  With the batch
 * sharded over `world` ranks the same function needs (1) the BN sums of conv4_1 / conv4_2 -- forward [sum x, sum x^2] and
 * backward [sum dy, sum dy*xhat], 2 x 512 f64 each -- summed over ranks, and (2) the SUM of the flat gradient buffers before
 * crnn_clip_adam_step(grad_mul = 1/world, wd_mul = world).
 *
 * (1) crnn_model_set_data_parallel switches the BN layers to global-batch statistics.  The exchange runs INSIDE the BN
 *     finalize kernel over NVLink peer memory when crnn_model_set_peers was called (every rank stores its 8 KB of sums into
 *     every peer's inbox, release/acquire flags at system scope, fixed-order f64 summation: bit-identical on all ranks, no
 *     NCCL launch on the forward path); otherwise through `allreduce` (e.g. an NCCL all-reduce issued by the caller).
 * (2) crnn_model_set_grad_ready_callback: crnn_backward calls `fn(user, offset, count, stream)` as soon as the gradients of a
 *     contiguous range [offset, offset+count) of the flat buffer are final (LSTM+logits first, conv1+conv2 last, 7 ranges
 *     covering the buffer exactly once), so the caller can all-reduce each range on a side stream while the rest of the
 *     backward pass still runs.
 * ---------------------------------------------------------------------------------------- */
typedef int  (*crnn_allreduce_fn)(void* user, void* dev_ptr, size_t count, int is_f64, crnn_stream_t stream);   /* in-place SUM */
typedef void (*crnn_grad_ready_fn)(void* user, int64_t offset, int64_t count, crnn_stream_t stream);
int     crnn_model_set_data_parallel(crnn_model* m, int rank, int world, crnn_allreduce_fn allreduce, void* user);
int     crnn_model_set_grad_ready_callback(crnn_model* m, crnn_grad_ready_fn fn, void* user);
/* Leave `sms` SMs free in the persistent kernels of crnn_backward (their grids are num_sms - sms CTAs), so that the collective
 * kernels the caller launches from the grad-ready callback find free SMs instead of delaying the tail of a full-GPU grid. */
int     crnn_model_set_backward_sm_reserve(crnn_model* m, int sms);
/* Peer-memory inboxes (cudaMalloc + CUDA IPC): create one per rank, exchange the 64-byte handles through the host language
 * (e.g. torch.distributed.all_gather_object), open the peers', hand all `world` pointers (own at [rank]) to the model.
 * crnn_peer_inbox_create and crnn_model_set_peers synchronise the device after writing device memory (the zeroed inbox, the
 * peer table), so that exchanges on any stream afterwards read what they wrote.  Neither is on the hot path. */
size_t  crnn_peer_inbox_bytes(void);
int     crnn_peer_inbox_create(void** dev_ptr, unsigned char handle[64]);
int     crnn_peer_inbox_open(const unsigned char handle[64], void** dev_ptr);
int     crnn_peer_inbox_close(void* dev_ptr);      /* a pointer obtained from crnn_peer_inbox_open */
int     crnn_peer_inbox_destroy(void* dev_ptr);    /* a pointer obtained from crnn_peer_inbox_create */
int     crnn_model_set_peers(crnn_model* m, int rank, int world, void* const* inbox_ptrs_host);
int     crnn_peer_error(crnn_model* m, int* err_host);   /* 1 if an exchange timed out waiting for a peer (syncs the device) */

/* Debug/parity taps: copy a named intermediate of the last crnn_forward() as f32 into dst.
 * names: "conv1" "conv2" "conv3_1" "conv3_2" "conv4_1" "conv4_2" "conv5" "lstm_out"
 * (pooled / post-activation, NHWC, as the reference's layers dict holds them), "xproj" (input projection,
 * permuted gate columns, backward-direction rows reversed by length), "a4a_pre" "a4b_pre" (conv4_x before BatchNorm).
 * Training-mode plans only (CRNN_INVALID_VALUE otherwise): "gates" (saved post-activation gates, layout of
 * lstm_gate_off) and the backward buffers "dl_rows" "d_lstm_out" "dz_all" "d_a5" "d_a4b" "d_pre4b" "d_pre4a"
 * "d_a3p" "d_pre32" "d_pre31" "d_a2" "d_pre2" "d_a1" of the last crnn_backward().
 * f32-class models (compute_dtype 2, 3): the eight activation names (split mode: the f32 sum hi + lo) and "xproj", which
 * there is f32 [N, H2, 2048]: both directions' x W_x in natural [i|j|f|o] column order, WITHOUT bias and with the rows
 * of the backward direction NOT reversed (the cell adds the bias and indexes frame len-1-step).  Other names fail with
 * CRNN_INVALID_VALUE. */
int     crnn_debug_tap(crnn_model* m, const char* name, float* dst, size_t dst_elems,
                       void* workspace, crnn_stream_t stream);
/* Same for the buffers that are not bf16, copied byte for byte: "bn" (f32 [2 layers][scale, shift, mean, invstd][512]),
 * "stats" (f64 [2 layers][sum, sum of squares][512]); after crnn_forward_lines per line: "bn" f32 [2 layers][N][4][512], "stats"
 * f64 [2 layers][N][2][512].  And, training-mode plans only, "am1" "am2" "am3" (u8 pool
 * window index dy*2+dx per pooled element) and "csave" (f32 saved cell state, layout of lstm_c_off).
 * f32-class models: "bn" and "stats" (same layouts), "cst" (f32 final cell state [2 dirs][Npad][256]) and the
 * activation buffers as stored under their tap names "conv1" .. "conv5", "lstm_out": split mode (2) bf16 rows
 * [hi(G*C) | lo(G*C)] of G consecutive positions (G = 2 for "conv4_2", else 1), tf32 mode (3) f32 [positions][C]
 * rounded to tf32.  Other names (am1..3, csave, the backward buffers) fail with CRNN_INVALID_VALUE.
 * fp8 models (compute_dtype 4): crnn_debug_tap returns "conv2" "conv3_1" "conv3_2" "conv4_1" "conv4_2" dequantised (e4m3 value
 * x its scale), the other names as on the bf16 path; crnn_debug_tap_raw returns those five as the raw e4m3 bytes (same NHWC
 * shapes), "fp8_scales" (f32 [5]: a2, a3, a3p, a4a, a4b), "fp8_wscale" and "fp8_colscale" (f32 [5 layers][512]: per output
 * channel weight scale and activation x weight scale of conv3_1, conv3_2, conv4_1, conv4_2, conv5; conv3_x fill 256 columns),
 * "fp8_w_conv3_1" .. "fp8_w_conv5" (u8 e4m3 weights [Cout][K], K in (kh, kw, ci) order), and "bn" / "stats" as above. */
int     crnn_debug_tap_raw(crnn_model* m, const char* name, void* dst, size_t dst_bytes,
                           void* workspace, crnn_stream_t stream);

/* Per-stage timing of crnn_forward with CUDA events recorded on the caller's stream (bench.py's roofline line).
 * crnn_profile_begin arms the next `max_forwards` forward calls; crnn_profile_read synchronises on the events and
 * returns ms_out[forwards][crnn_profile_num_stages()]. */
int         crnn_profile_begin(crnn_model* m, int max_forwards);
int         crnn_profile_num_stages(void);
const char* crnn_profile_stage_name(int stage);
int         crnn_profile_read(crnn_model* m, float* ms_out, int* forwards);
/* same for crnn_backward (armed by the same crnn_profile_begin) */
int         crnn_profile_bwd_num_stages(void);
const char* crnn_profile_bwd_stage_name(int stage);
int         crnn_profile_bwd_read(crnn_model* m, float* ms_out, int* backwards);

/* Stand-alone bf16 GEMM test entry (tests only): D[M,Nc] f32 = A[M,K] * B[Nc,K]^T, bf16 in. */
int     crnn_test_gemm_bf16(const void* A, const void* B, float* D, int M, int Nc, int K,
                            int block_n, crnn_stream_t stream);

/* MN-major ("TN") GEMM test entry (tests only): D[M,N] f32 (caller-zeroed) += A[K,M]^T * B[K,N], bf16 in. */
int     crnn_test_gemm_tn_bf16(const void* A, const void* B, float* D, int M, int N, int K, int block_n,
                               int k_splits, crnn_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif  /* CRNN_CTC_H_ */
