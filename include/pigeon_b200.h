/*
 * pigeon_b200 — C ABI of the H100-native (sm_90a) PIGEON inference hot path.
 *
 * The reference (LukasHaas/PIGEON) has no FFI: its hot path sits behind Python nn.Module calls.  This header
 * is the seam a maintainer binds underneath those modules (ctypes stub in INTEGRATION.md); every entry point
 * names the reference code it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host; the caller owns every buffer;
 *   - no hidden device allocations: scratch comes from the caller (`*_workspace_bytes` tells how much);
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*) and returns immediately;
 *   - return value 0 = success, non-zero = failure with a message in pg_last_error() (thread-local);
 *     no exceptions cross the boundary; there is NO CPU fallback anywhere behind this ABI;
 *   - fp16 means IEEE binary16 (`__half`), "f32"/"f64" IEEE float/double, i64 = int64_t.
 */
#ifndef PIGEON_B200_H_
#define PIGEON_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PG_ABI_VERSION 4

/* ---------------------------------------------------------------------------------------------------
 * Library
 * ------------------------------------------------------------------------------------------------- */
int pg_abi_version(void);
/* Message of the last failing call on this thread ("" if none). */
const char* pg_last_error(void);
/* Number of SMs of the current device (grid sizing); < 0 on failure. */
int pg_device_sm_count(void);

/* ---------------------------------------------------------------------------------------------------
 * CLIP ViT vision tower  (HF CLIPVisionTransformer as driven by reference
 * models/clip_embedder.py:58-65 and models/super_guessr.py:386-398)
 * ------------------------------------------------------------------------------------------------- */
typedef struct pg_vit_config {
  int32_t image_size;   /* 336 */
  int32_t patch_size;   /* 14  */
  int32_t hidden;       /* 1024, multiple of 256 */
  int32_t heads;        /* 16, hidden / heads must be 64 */
  int32_t intermediate; /* 4096, multiple of 256 */
  int32_t layers;       /* 24 */
  float ln_eps;         /* 1e-5 */
  int32_t patch_k_pad;  /* padded im2col K: multiple of 64, >= 3*patch*patch (640 for 14x14) */
} pg_vit_config;

/* One encoder block (HF CLIPEncoderLayer).  Matrices are fp16 in nn.Linear layout [out, in]. */
typedef struct pg_vit_layer {
  const float* ln1_g; const float* ln1_b;       /* layer_norm1 [hidden] */
  const void* w_qkv; const float* b_qkv;        /* [3*hidden, hidden] = [Wq; Wk; Wv], bias [3*hidden] */
  const void* w_o; const float* b_o;            /* out_proj [hidden, hidden] */
  const float* ln2_g; const float* ln2_b;       /* layer_norm2 [hidden] */
  const void* w_fc1; const float* b_fc1;        /* mlp.fc1 [intermediate, hidden] */
  const void* w_fc2; const float* b_fc2;        /* mlp.fc2 [hidden, intermediate] */
  /* Optional (all six or none; NULL = pg_vit_forward runs the LayerNorm kernels): LayerNorm folded into the GEMM after it.
   *   w_*_ln   fp16 = W * gamma (column-wise), same shape as W;   cs_* f32 [out] = row sums of the fp16 values of w_*_ln;
   *   b_*_ln   f32 [out] = b + W beta.
   * With them the forward feeds the RAW fp16 residual row to the tensor cores and applies
   * rstd * (acc - mu * cs) + b_ln in the epilogue; (mu, rstd) come from moments the previous epilogue left behind. */
  const void* w_qkv_ln; const float* b_qkv_ln; const float* cs_qkv;
  const void* w_fc1_ln; const float* b_fc1_ln; const float* cs_fc1;
} pg_vit_layer;

typedef struct pg_vit_weights {
  const void* patch_w;      /* fp16 [hidden, patch_k_pad]: Conv2d weight flattened (c, ky, kx), zero padded */
  const float* class_emb;   /* [hidden] */
  const float* pos_emb;     /* [tokens, hidden], tokens = (image/patch)^2 + 1 */
  const float* pre_ln_g; const float* pre_ln_b; /* pre_layrnorm [hidden] */
  const pg_vit_layer* layers_host;              /* HOST array of `layers` entries (device pointers inside) */
} pg_vit_weights;

typedef struct pg_vit pg_vit;

/* Copies the config and the pointer tables (not the weights).  Replaces CLIPVisionModel construction at
 * reference models/clip_embedder.py:26 / evaluation/evaluate.py:36 for the forward path. */
int pg_vit_create(const pg_vit_config* cfg, const pg_vit_weights* w, pg_vit** out);
void pg_vit_destroy(pg_vit* h);
/* Scratch needed by pg_vit_forward for `n_views` images. */
size_t pg_vit_workspace_bytes(const pg_vit* h, int32_t n_views);
/* pixels [n_views, 3, image, image] (fp32 if pixels_f16 == 0 else fp16), NCHW contiguous
 *   -> emb_out f32 [n_views, hidden] = mean over all tokens of last_hidden_state (pre post_layernorm),
 *      i.e. reference models/clip_embedder.py:63-65 / models/super_guessr.py:395-398;
 *   -> hidden_out (optional, may be NULL) f32 [n_views, tokens, hidden] = last_hidden_state. */
int pg_vit_forward(pg_vit* h, const void* pixels, int32_t pixels_f16, int32_t n_views, void* workspace,
                   size_t workspace_bytes, float* emb_out, float* hidden_out, void* stream);
/* pg_vit_forward plus cls_out f32 [n_views, hidden] = last_hidden_state[:, 0], the CLS rows that HF
 * CLIPVisionTransformer pools into post_layernorm (transformers 4.23.1 modeling_clip.py, `pooled_output =
 * last_hidden_state[:, 0, :]`) and CLIPModel.get_image_features projects — without writing the whole hidden_out.
 * hidden_out may still be given (or NULL). */
int pg_vit_forward_cls(pg_vit* h, const void* pixels, int32_t pixels_f16, int32_t n_views, void* workspace,
                       size_t workspace_bytes, float* emb_out, float* hidden_out, float* cls_out, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * CLIP text tower and image-text logits (HF CLIPModel, transformers 4.23.1 modeling_clip.py, the dual encoder that
 * reference training/train_modes.py:30-64 pretrains and dataset_creation/pretrain/pretrain_dataset.py:299-330 scores:
 * `model(**clip_processor(text=captions, images=images), return_loss=True).logits_per_image.softmax(1).argmax(1)`).
 * ------------------------------------------------------------------------------------------------- */
typedef struct pg_text_config {
  int32_t vocab;          /* 49408 */
  int32_t max_positions;  /* 77 */
  int32_t hidden;         /* 768, multiple of 256 */
  int32_t heads;          /* 12, hidden / heads must be 64 */
  int32_t intermediate;   /* 3072, multiple of 256 */
  int32_t layers;         /* 12 */
  float ln_eps;           /* 1e-5 */
} pg_text_config;

/* HF CLIPTextTransformer weights.  The encoder layers are the vision tower's pg_vit_layer (same pre-LN CLIPEncoderLayer)
 * with the LayerNorm-fold fields NULL: the text tower runs the LayerNorm kernels. */
typedef struct pg_text_weights {
  const float* token_emb;        /* f32 [vocab, hidden]          embeddings.token_embedding.weight */
  const float* pos_emb;          /* f32 [max_positions, hidden]  embeddings.position_embedding.weight */
  const pg_vit_layer* layers_host;  /* HOST array of `layers` entries (device pointers inside) */
  const float* final_ln_g; const float* final_ln_b;   /* final_layer_norm [hidden] */
} pg_text_weights;

typedef struct pg_text pg_text;

int pg_text_create(const pg_text_config* cfg, const pg_text_weights* w, pg_text** out);
void pg_text_destroy(pg_text* h);
/* Scratch needed by pg_text_forward for n captions of S tokens. */
size_t pg_text_workspace_bytes(const pg_text* h, int32_t n, int32_t S);
/* HF CLIPTextTransformer.forward (4.23.1): input_ids i64 [n, S] (1 <= S <= max_positions), attention_mask i64 [n, S] or
 * NULL (all ones; 0 excludes that key, on top of the causal mask; attention_mask[:, 0] must be 1, as CLIP's BOS is)
 *   -> pooled_out f32 [n, hidden] = final_layer_norm(x)[b, argmax_t input_ids[b, t]] (first index of the largest id);
 *   -> hidden_out (optional) f32 [n, S, hidden] = last_hidden_state (after final_layer_norm). */
int pg_text_forward(pg_text* h, const int64_t* input_ids, const int64_t* attention_mask, int32_t n, int32_t S,
                    void* workspace, size_t workspace_bytes, float* pooled_out, float* hidden_out, void* stream);

/* visual_projection / text_projection (nn.Linear, no bias) at fp32-faithful accuracy: x f32 [n, D], optional LayerNorm
 * (ln_g and ln_b both NULL = none; CLIPModel.get_image_features applies post_layernorm here), then the error-compensated
 * split GEMM of the geocell head: w3 = pg_head_pack_weight(W f32 [P, D]) fp16 [P, 3 D]  ->  out f32 [n, P] = LN(x) W^T. */
size_t pg_clip_project_workspace_bytes(int32_t n, int32_t D);
int pg_clip_project(const float* x, int32_t n, int32_t D, const float* ln_g, const float* ln_b, float ln_eps, const void* w3,
                    int32_t P, void* workspace, size_t workspace_bytes, float* out, void* stream);
/* CLIPModel.forward after the projections: img f32 [Ni, P], txt f32 [Nt, P] (not normalised)
 *   -> logits_per_image f32 [Ni, Nt] = (img / |img|) (txt / |txt|)^T * exp(logit_scale);
 *   -> optional (NULL = not written): logits_per_text f32 [Nt, Ni] (the transpose), probs f32 [Ni, Nt] (softmax over the
 *      captions), pred i64 [Ni] (first argmax), loss f32 [1] = clip_loss (mean of the two cross-entropies against arange;
 *      needs Ni == Nt). */
int pg_clip_logits(const float* img, int32_t Ni, const float* txt, int32_t Nt, int32_t P, float logit_scale,
                   float* logits_per_image, float* logits_per_text, float* probs, int64_t* pred, float* loss, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Geocell head (reference models/super_guessr.py:437-459: view mean, cell_layer, softmax, argmax, top-k)
 * ------------------------------------------------------------------------------------------------- */
/* One-off: cell_layer.weight f32 [C, D] -> packed fp16 [C, 3*D] = [Whi | Whi | Wlo] (error-compensated split). */
int pg_head_pack_weight(const float* w, void* w3_out, int32_t C, int32_t D, void* stream);
size_t pg_head_workspace_bytes(int32_t B, int32_t D);
/* emb f32 [B, V, D] (V = 4 for panoramas, 1 otherwise)
 *   -> pooled f32 [B, D]; logits f32 [B, C]; probs f32 [B, C]; pred_cell i64 [B];
 *      pred_lnglat f64 [B, 2] = centroids[pred_cell] (lng, lat);
 *      topk_val f32 [B, k] (descending), topk_idx i64 [B, k]. */
int pg_head_forward(const float* emb, int32_t B, int32_t V, int32_t D, const void* w3, const float* bias,
                    const double* centroids, int32_t C, int32_t k, void* workspace, size_t workspace_bytes,
                    float* pooled, float* logits, float* probs, int64_t* pred_cell, double* pred_lnglat,
                    float* topk_val, int64_t* topk_idx, void* stream);
/* Measurement / deployment switch of pg_head_forward for this process: 0 (default) = three kernels (view mean + split,
 * wgmma GEMM + bias, softmax / arg-max / top-k); 1 = ONE kernel doing all of it (D % 64 == 0 and C <= 6144, otherwise the
 * three-kernel sequence runs): the view mean and the hi/lo split happen in the GEMM's A-operand producer warps and the CTA
 * that completes a block of 128 samples last normalises its rows.  Same results to fp32 summation order. */
int pg_head_set_fused(int32_t on);

/* Classification loss of reference models/super_guessr.py:468-474 (CrossEntropyLoss, mean over the batch).
 *   mode 0: labels_idx i64 [B] class indices;  mode 1: soft f32 [B, C] target probabilities;
 *   mode 2: haversine-smoothed targets from labels_lnglat f64 [B, 2] and centroids f64 [C, 2]
 *           (preprocessing/geo_utils.py:58-74 + preprocessing/utils.py:7-19, smoothing_km = 65).
 * per_sample f64 [B] is scratch/out; loss_out f64 [1].
 * mode 0 labels outside [0, C) are never used as an index: that sample's loss and the batch mean become NaN (and, in
 * pg_head_loss_grad, its gradient row zero).  torch's ignore_index = -100 is not implemented — the reference's labels on this
 * path are geocell indices and never negative. */
int pg_head_loss(const float* logits, int32_t B, int32_t C, int32_t mode, const int64_t* labels_idx,
                 const float* soft, const double* labels_lnglat, const double* centroids, double smoothing_km,
                 double* per_sample, double* loss_out, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Image pre-processing ("next" row N2): what `CLIPProcessor.from_pretrained(CLIP_MODEL)(images=...)` does on the
 * CPU per item in reference dataset_creation/finetune/embed_dataset.py:17-22, preprocessing/dataset_preprocessing.py:
 * 182-204, dataset_creation/benchmark/benchmark_dataset.py:100-104 (transformers 4.23.1 CLIPFeatureExtractor over
 * Pillow): resize shortest edge to `size` (BICUBIC) -> center crop -> /255 -> (x - mean) / std, channel first.
 * Bit-exact with Pillow's fixed-point resampler (uint8 stage) and with numpy float32 (normalisation).
 * ------------------------------------------------------------------------------------------------- */
typedef struct pg_image {
  const uint8_t* data;  /* DEVICE pointer, RGB interleaved (H x W x 3) */
  int32_t height, width;
  int64_t row_stride;   /* bytes between rows, >= 3 * width */
} pg_image;
/* `images` is a HOST array of n descriptors.  0 on error (see pg_last_error). */
size_t pg_preprocess_workspace_bytes(const pg_image* images, int32_t n, int32_t size);
/* out: [n, 3, size, size] f32 (out_f16 = 0) or f16 (out_f16 = 1, round-to-nearest of the f32 value); mean/std: host float[3]. */
int pg_preprocess_clip(const pg_image* images, int32_t n, int32_t size, const float* mean, const float* std,
                       void* workspace, size_t workspace_bytes, void* out, int32_t out_f16, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Baseline JPEG decoding (csrc/jpeg.cu): what `PIL.Image.open(f).convert('RGB')` does on the CPU before every
 * CLIPProcessor call in reference dataset_creation/finetune/embed_dataset.py:17-22 (through the HF Image() column of
 * finetune_dataset.py:86-90), dataset_creation/benchmark/benchmark_dataset.py:66-79 and pretrain_dataset.py:109-161.
 * Byte-identical to Pillow over libjpeg-turbo with its defaults (ISLOW IDCT, fancy upsampling) for the files it
 * decodes: sequential Huffman (SOF0 / SOF1), 8-bit, one scan, grayscale or YCbCr 4:4:4 / 4:2:2 / 4:2:0, with or
 * without restart markers; through pg_jpeg_parse_multiscan also progressive (SOF2) and multi-scan sequential files of
 * the same kinds.  Everything else is refused with a status and a reason (DESIGN.md §1).
 * ------------------------------------------------------------------------------------------------- */
#define PG_JPEG_OK 0
#define PG_JPEG_UNSUPPORTED 1       /* a valid file outside the decoded subset: progressive, 12-bit, CMYK, RGB, ... */
#define PG_JPEG_BAD_HEADER 2        /* truncated or inconsistent marker segments, or not a JPEG */
#define PG_JPEG_BAD_CODE 3          /* entropy data: a code missing from its table, or a run past coefficient 63 */
#define PG_JPEG_OVERRUN 4           /* entropy data: a segment ends before its MCUs do */
#define PG_JPEG_UNEXPECTED_MARKER 5 /* entropy data: a marker where data should be */
#define PG_JPEG_BAD_RST 6           /* entropy data: wrong restart marker number or count */
#define PG_JPEG_NO_EOI 7            /* entropy data: the file ends without EOI */

typedef struct pg_jpeg_info {
  int32_t status;                 /* PG_JPEG_* */
  int32_t sof;                    /* frame marker (0xC0 .. 0xCF), 0 before one is seen */
  int32_t precision, height, width, components;
  int32_t component_id[3], h_samp[3], v_samp[3], quant_table[3], dc_table[3], ac_table[3];
  int32_t restart_interval;       /* MCUs per restart interval, 0 without DRI */
  int32_t num_segments;           /* entropy-coded segments: restart intervals, or 1 */
  int32_t table_mask;             /* bit t: DQT t defined; bit 4 + t: DC DHT t; bit 8 + t: AC DHT t;
                                     PG_JPEG_MULTISCAN and bits 16+ for multi-scan files (below) */
  int64_t scan_offset, scan_bytes; /* entropy-coded data, from the end of the SOS segment to the marker after it */
  uint16_t qt[4][64];             /* quantisation tables in zig-zag order, as stored */
  uint8_t dc_bits[4][16], ac_bits[4][16];
  uint8_t dc_vals[4][256], ac_vals[4][256];
} pg_jpeg_info;

/* Host-only marker walk of one file (data_host: `bytes` bytes).  Returns info_out->status; when it is not PG_JPEG_OK,
 * pg_last_error() names the reason.  Validates the restart-marker sequence and the EOI. */
int pg_jpeg_parse(const uint8_t* data_host, int64_t bytes, pg_jpeg_info* info_out);

/* Multi-scan files: progressive Huffman (SOF2, 8-bit) and sequential SOF0 / SOF1 files of more than one scan, with the
 * components and sampling layouts above.  pg_jpeg_parse_multiscan returns, for every file pg_jpeg_parse accepts, the
 * identical info; it also accepts these files, marking them with PG_JPEG_MULTISCAN in table_mask.  For such an info:
 * num_segments counts the entropy-coded segments of all scans, scan_offset / scan_bytes span the data from the first
 * scan to the EOI, restart_interval is that of the first scan, and table_mask >> 16 is the number of Huffman table
 * selections over all scans (it bounds the workspace).  The per-scan tables are found again from the file's bytes by
 * pg_jpeg_decode.  libjpeg's JERR_BAD_PROGRESSION cases are PG_JPEG_BAD_HEADER; sequences libjpeg only warns about
 * (JWRN_BOGUS_PROGRESSION), a coefficient sent twice, more than PG_JPEG_MAX_SCANS scans and a progression that leaves
 * any coefficient unsent or not refined to bit 0 (libjpeg then smooths between blocks) are PG_JPEG_UNSUPPORTED. */
#define PG_JPEG_MULTISCAN (1 << 12)
#define PG_JPEG_MAX_SCANS 256
int pg_jpeg_parse_multiscan(const uint8_t* data_host, int64_t bytes, pg_jpeg_info* info_out);

typedef struct pg_jpeg_scan {
  int32_t components;             /* in this scan: 1, or the interleaved components of a sequential or DC scan */
  int32_t component[3];           /* frame component indices (0 .. components of the frame - 1), in scan order */
  int32_t ss, se, ah, al;         /* spectral band and successive-approximation bits (0, 63, 0, 0 when sequential) */
  int32_t restart_interval;       /* MCUs per restart interval (single blocks in a one-component scan), 0 without DRI */
  int32_t num_segments;           /* entropy-coded segments of this scan */
  int32_t level;                  /* 1 + the highest level of earlier scans sharing a component and a coefficient */
} pg_jpeg_scan;
/* Host-only: the scans of a file pg_jpeg_parse_multiscan accepts (one for a single-scan file), the first min(count,
 * cap) written to out.  Returns their count, or -1 (pg_last_error() names the reason) for a refused file. */
int pg_jpeg_scans(const uint8_t* data_host, int64_t bytes, pg_jpeg_scan* out, int32_t cap);

/* Workspace of pg_jpeg_decode for n parsed files packed into packed_bytes bytes.  0 on error. */
size_t pg_jpeg_workspace_bytes(const pg_jpeg_info* infos_host, int32_t n, int64_t packed_bytes);
/* Decodes the files whose info status is PG_JPEG_OK: file i is packed_host[offsets_host[i] .. offsets_host[i+1]) (one
 * host-to-device copy of offsets_host[n] bytes; pinned memory makes it asynchronous), infos_host[i] its pg_jpeg_parse
 * or pg_jpeg_parse_multiscan result, dst_host[i] a descriptor of its height x width x 3 uint8 RGB destination
 * (written; the same descriptors feed pg_preprocess_clip).  status_out: device i32 [n], the parse status of a skipped
 * file, else PG_JPEG_OK or the entropy-data error of that file (whose destination is then left unwritten).  A batch of
 * single-scan files takes three or four launches: the Huffman decode of short entropy-coded segments (restart
 * intervals, small files) with one thread each and of long ones (a photo without restart markers) with one CTA each,
 * chunked and self-synchronising, then the IDCT and the colour conversion.  A batch with multi-scan files also zeroes
 * their coefficients and decodes their scans in one launch per dependency level (pg_jpeg_scan.level), all in stream
 * order. */
int pg_jpeg_decode(const uint8_t* packed_host, const int64_t* offsets_host, const pg_jpeg_info* infos_host, int32_t n,
                   const pg_image* dst_host, void* workspace, size_t workspace_bytes, int32_t* status_out, void* stream);
/* Huffman decode of single-scan segments in pg_jpeg_decode, process-wide: 0 = automatic (default; segments of at least
 * 32768 compressed bytes take the chunked kernel, shorter ones one thread each), 1 = one thread per segment, 2 = the
 * chunked kernel for every segment.  chunk_bytes > 0 forces the chunk size in de-stuffed bytes (raised where a segment
 * would need more than 1024 chunks); 0 sizes chunks automatically.  All give the same bytes and statuses; the switch
 * exists for tests and A/B benchmarks, not for tuning.  Returns 1 for a mode outside {0, 1, 2} or chunk_bytes < 0. */
int pg_jpeg_set_schedule(int32_t mode, int32_t chunk_bytes);
/* Host-only test entry: the entropy decode of pg_jpeg_decode on the CPU, for single-scan files (a multi-scan info is an
 * error).  chunk_bytes = 0 runs the one-thread-per-segment decoder; > 0 runs the chunked decoder's functions, in its
 * order of rounds, at that chunk size; < 0 at the automatic size.  coef_out (NULL: not returned) receives the int16
 * blocks, 64 in natural order each, of every image with an OK info in batch order, its components in order, each
 * component's grid padded to whole MCUs row by row; blocks of a failed image are unspecified.  status_out[n] as
 * pg_jpeg_decode's; rounds_out[n] (optional) the most synchronisation rounds any segment of the image took (0 for the
 * one-thread decoder).  Returns the number of blocks, or -1 (pg_last_error() names the reason). */
int64_t pg_jpeg_entropy_host(const uint8_t* packed_host, const int64_t* offsets_host, const pg_jpeg_info* infos_host,
                             int32_t n, int32_t chunk_bytes, int16_t* coef_out, int32_t* status_out, int32_t* rounds_out);

/* ---------------------------------------------------------------------------------------------------
 * PNG decoding (csrc/png.cu): the same `PIL.Image.open(f).convert('RGB')` for PNG files.  Byte-identical to Pillow
 * for the files it decodes: non-interlaced PNGs of every colour type and bit depth, with or without tRNS.  Alpha is
 * dropped, 16-bit samples keep their high byte (16-bit grey clips to 255, as Pillow's I;16 -> RGB does), 1/2/4-bit grey
 * scales to 0..255, and a palette index past PLTE (or a palette image without PLTE) is black.  Interlaced files, APNG,
 * IDAT chunks that are not consecutive, CRC errors before the first IDAT and text above Pillow's limits are refused
 * with a status and a reason (DESIGN.md §1).
 * ------------------------------------------------------------------------------------------------- */
#define PG_PNG_OK 0
#define PG_PNG_UNSUPPORTED 1        /* a file outside the decoded subset: interlaced, APNG, split IDAT runs, ... */
#define PG_PNG_BAD_HEADER 2         /* not a PNG, no or bad IHDR, no IDAT, a CRC error before the first IDAT */
#define PG_PNG_BAD_ZLIB 3           /* the zlib header or Adler-32 is wrong, or bytes follow the stream */
#define PG_PNG_BAD_DEFLATE 4        /* an invalid block type, code set, code or distance */
#define PG_PNG_TRUNCATED 5          /* the stream ends early, or yields fewer bytes than the rows need */
#define PG_PNG_TOO_LONG 6           /* more than 4096 decompressed bytes after the rows */
#define PG_PNG_BAD_FILTER 7         /* a row filter type above 4 */

typedef struct pg_png_info {
  int32_t status;                 /* PG_PNG_OK, PG_PNG_UNSUPPORTED or PG_PNG_BAD_HEADER */
  int32_t width, height, bit_depth, color_type;   /* IHDR */
  int32_t channels;               /* samples per pixel: 1 (grey, palette), 2 (grey + alpha), 3 (RGB) or 4 (RGBA) */
  int32_t bpp;                    /* filter distance in bytes: max(1, channels * bit_depth / 8) */
  int32_t palette_entries;        /* PLTE entries of a palette image, 0 without PLTE */
  int32_t idat_chunks;            /* chunks in the run of consecutive IDATs */
  int64_t row_bytes;              /* bytes per row, without the filter byte */
  int64_t idat_offset;            /* offset in the file of the first IDAT chunk (its length field) */
  int64_t zlib_bytes;             /* payload bytes of the IDAT run: the zlib stream */
  uint8_t palette[256][3];        /* PLTE, zero past palette_entries */
} pg_png_info;

/* Host-only chunk walk of one file.  Returns info_out->status; when it is not PG_PNG_OK, pg_last_error() names the
 * reason. */
int pg_png_parse(const uint8_t* data_host, int64_t bytes, pg_png_info* info_out);
/* Workspace of pg_png_decode for n parsed files packed into packed_bytes bytes.  0 on error. */
size_t pg_png_workspace_bytes(const pg_png_info* infos_host, int32_t n, int64_t packed_bytes);
/* Decodes the files whose info status is PG_PNG_OK, with the arguments of pg_jpeg_decode: one host-to-device copy of
 * the packed files and three launches (inflate, one warp per stream; unfiltering; RGB conversion into the dst_host
 * descriptors, which feed pg_preprocess_clip unchanged).  status_out: device i32 [n], the parse status of a skipped
 * file, else PG_PNG_OK or the stream / filter error of that file (whose destination is then left unwritten). */
int pg_png_decode(const uint8_t* packed_host, const int64_t* offsets_host, const pg_png_info* infos_host, int32_t n,
                  const pg_image* dst_host, void* workspace, size_t workspace_bytes, int32_t* status_out, void* stream);
/* Host-only test entry: pg_png_decode's inflate, unfilter and convert functions on the CPU.  rgb_out (NULL: not
 * returned) receives the height x width x 3 bytes of every image with an OK info, in batch order (a failed image's
 * bytes are unspecified); status_out[n] as pg_png_decode's.  Returns the bytes of rgb_out, or -1 (pg_last_error()). */
int64_t pg_png_decode_host(const uint8_t* packed_host, const int64_t* offsets_host, const pg_png_info* infos_host,
                           int32_t n, uint8_t* rgb_out, int32_t* status_out);

/* ---------------------------------------------------------------------------------------------------
 * Fine-tune step, head-only part ("next" row N1 with a frozen or absent base model): what loss.backward() and
 * torch.optim.AdamW.step() do for cell_layer in reference training/train_eval_loop.py:187,215-221.
 * ------------------------------------------------------------------------------------------------- */
/* pg_head_loss plus its gradient: dlogits f32 [B, C] = grad_scale / B * (softmax(logits) * sum_c(target) - target)
 * (the backward of CrossEntropyLoss(reduction='mean') at super_guessr.py:474 for index, soft or smoothed targets). */
int pg_head_loss_grad(const float* logits, int32_t B, int32_t C, int32_t mode, const int64_t* labels_idx,
                      const float* soft, const double* labels_lnglat, const double* centroids, double smoothing_km,
                      double grad_scale, double* per_sample, double* loss_out, float* dlogits, void* stream);
/* Backward of cell_layer (nn.Linear, super_guessr.py:447) in fp32:
 *   dw f32 [C, D] (+)= dlogits^T . pooled;  db f32 [C] (+)= column sums of dlogits;  dpooled f32 [B, D] = dlogits . w.
 * Any of dw / db / dpooled may be NULL; `accumulate` != 0 adds into dw/db (gradient accumulation, :218-221). */
int pg_head_backward(const float* dlogits, const float* pooled, const float* w, int32_t B, int32_t C, int32_t D,
                     int32_t accumulate, float* dw, float* db, float* dpooled, void* stream);
/* torch.optim.AdamW single-tensor update on a flat fp32 parameter (amsgrad = maximize = False), `step` counts from 1;
 * grad is read as grad * grad_scale (1/world_size after a summing all-reduce). */
int pg_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double lr,
                  double beta1, double beta2, double eps, double weight_decay, int64_t step, double grad_scale,
                  void* stream);

/* ---------------------------------------------------------------------------------------------------
 * CLIP pretraining optimizer step: what the HF Trainer (transformers 4.23.1, optim="adamw_hf") of reference
 * training/train_modes.py:30-64 runs after the accumulated micro-batches.
 * ------------------------------------------------------------------------------------------------- */
/* Bytes of workspace pg_grad_norm_clip needs for n gradient elements. */
size_t pg_grad_norm_clip_workspace_bytes(int64_t n);
/* torch.nn.utils.clip_grad_norm_(params, max_norm) over one flat fp32 gradient read as grad * grad_scale: writes the device
 * floats total_norm = ||grad * grad_scale||_2 and clip_coef = min(max_norm / (total_norm + 1e-6), 1); the gradient itself is
 * not modified (pg_adamw_hf_step applies clip_coef).  Deterministic: the same n and bits give the same result on every run.
 * A non-finite norm is not an error and the step is not skipped (as in torch with error_if_nonfinite=False): an inf norm
 * gives clip_coef 0 and a NaN norm a NaN clip_coef, so the parameters the next update touches become NaN. */
int pg_grad_norm_clip(const float* grad, int64_t n, double grad_scale, double max_norm, float* total_norm, float* clip_coef,
                      void* workspace, size_t workspace_bytes, void* stream);
/* transformers.optimization.AdamW.step (4.23.1, correct_bias = True) on a flat fp32 parameter, `step` counts from 1:
 *   g = grad * grad_scale * (*clip_coef);  m = m*beta1 + (1-beta1)*g;  v = v*beta2 + (1-beta2)*g*g;
 *   p -= lr * sqrt(1-beta2^t) / (1-beta1^t) * m / (sqrt(v) + eps);  then p += (-lr*weight_decay) * p if weight_decay > 0.
 * clip_coef is a device pointer (NULL = 1), so the step needs no host synchronisation. */
int pg_adamw_hf_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, double lr,
                     double beta1, double beta2, double eps, double weight_decay, int64_t step, double grad_scale,
                     const float* clip_coef, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Fine-tune step, vision tower ("next" row N1): the forward of pg_vit_forward with every activation the backward
 * needs kept in caller-provided buffers, and the backward itself — what autograd runs through HF
 * CLIPVisionTransformer for `accelerator.backward(output.loss)` in reference training/train_eval_loop.py:216.
 * Gradients flow in bf16 operands with fp32 accumulation; weight gradients accumulate in fp32.
 * rows = n_views * tokens.  All pointers are device pointers; the *_host arrays live on the host.
 * ------------------------------------------------------------------------------------------------- */
typedef struct pg_vit_saved_layer {
  float* x0;    /* f32 [rows, hidden]        residual stream entering the layer */
  void* xn1;    /* f16 [rows, hidden]        layer_norm1 output */
  void* qkv;    /* f16 [rows, 3*hidden]      q | k | v projections */
  float* lse2;  /* f32 [n_views*heads, tokens] log2-sum-exp of the scaled logits */
  void* ao;     /* f16 [rows, hidden]        attention output (input of out_proj) */
  float* x1;    /* f32 [rows, hidden]        residual stream after the attention block */
  void* xn2;    /* f16 [rows, hidden]        layer_norm2 output */
  void* u;      /* f16 [rows, intermediate]  fc1 pre-activation */
  void* h;      /* f16 [rows, intermediate]  quick_gelu(fc1) */
} pg_vit_saved_layer;

typedef struct pg_vit_saved {
  void* im2col;  /* f16 [n_views*patches, patch_k_pad] */
  float* e;      /* f32 [rows, hidden] class/patch + position embeddings (input of pre_layrnorm) */
  float* x_out;  /* f32 [rows, hidden] last_hidden_state */
  const pg_vit_saved_layer* layers_host;  /* [layers] */
} pg_vit_saved;

/* emb_out f32 [n_views, hidden] = token mean of last_hidden_state, as pg_vit_forward. */
int pg_vit_forward_train(pg_vit* h, const void* pixels, int32_t pixels_f16, int32_t n_views, const pg_vit_saved* saved,
                         float* emb_out, void* stream);

typedef struct pg_vit_layer_bwd {
  /* bf16 transposed weights for the data gradients: w_qkv_t [hidden, 3*hidden], w_o_t [hidden, hidden],
   * w_fc1_t [hidden, intermediate], w_fc2_t [intermediate, hidden] (row-major, = W^T of the [out, in] Linear weights) */
  const void *w_qkv_t, *w_o_t, *w_fc1_t, *w_fc2_t;
  /* f32 gradient accumulators (+=), same shapes as the parameters; all NULL = frozen layer
   * (reference freeze policy, models/super_guessr.py:159-160) */
  float *d_ln1_g, *d_ln1_b, *d_w_qkv, *d_b_qkv, *d_w_o, *d_b_o, *d_ln2_g, *d_ln2_b, *d_w_fc1, *d_b_fc1, *d_w_fc2, *d_b_fc2;
} pg_vit_layer_bwd;

typedef struct pg_vit_grads {
  /* embeddings + pre_layrnorm, f32 (+=); all NULL = frozen (the backward then stops at the lowest trainable layer) */
  float *d_patch_w;   /* [hidden, patch_k_pad] */
  float *d_class_emb; /* [hidden] */
  float *d_pos_emb;   /* [tokens, hidden] */
  float *d_pre_ln_g, *d_pre_ln_b;
  const pg_vit_layer_bwd* layers_host;  /* [layers] */
  /* Optional (may be NULL): layers + 1 cudaEvent_t handles.  pg_vit_backward records entry l on its stream as soon as the
   * weight gradients of encoder layer l are complete for this call, entry `layers` after the embedding gradients — so that
   * the caller can start the NCCL all-reduce of a layer's gradient bucket on a side stream while the layers below are
   * still in their backward (reference: DDP's bucketed overlap, training/train_eval_loop.py:192,216).  NULL entries skipped. */
  void* const* layer_done_events;
} pg_vit_grads;

size_t pg_vit_backward_workspace_bytes(const pg_vit* h, int32_t n_views);
/* d_emb f32 [n_views, hidden]: gradient of the loss with respect to the token-mean embedding of each view. */
int pg_vit_backward(pg_vit* h, const pg_vit_saved* saved, const float* d_emb, int32_t n_views, const pg_vit_grads* grads,
                    void* workspace, size_t workspace_bytes, void* stream);

/* As pg_vit_backward, but d_cls f32 [n_views, hidden] is the gradient of the CLS rows last_hidden_state[:, 0] (HF
 * CLIPVisionTransformer's pooled output, transformers 4.23.1 modeling_clip.py `pooled_output = last_hidden_state[:, 0, :]`,
 * which CLIPModel.get_image_features feeds to post_layernorm and visual_projection): the backward starts from d_cls at
 * token 0 of each view and zero elsewhere.  Same saved activations (x_out holds the CLS rows) and workspace. */
int pg_vit_backward_cls(pg_vit* h, const pg_vit_saved* saved, const float* d_cls, int32_t n_views, const pg_vit_grads* grads,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * CLIPModel contrastive training step: what autograd runs through HF CLIPModel (transformers 4.23.1 modeling_clip.py) for
 * `loss.backward()` under the HF Trainer of reference training/train_modes.py:30-64 (`return_loss=True`, nothing frozen).
 * The text tower reuses the vision tower's saved-activation layout and encoder-layer backward (causal + attention_mask
 * attention); the projections' backward is pg_head_backward with db = NULL, post_layernorm's pg_layernorm_f32 /
 * pg_layernorm_backward, the vision side pg_vit_forward_train + pg_vit_backward_cls.
 * ------------------------------------------------------------------------------------------------- */
typedef struct pg_text_saved {
  float* x_final;                         /* f32 [n*S, hidden] residual stream entering final_layer_norm */
  const pg_vit_saved_layer* layers_host;  /* [layers], rows = n*S (x0 of layer 0 = the embeddings; lse2 [n*heads, S]) */
} pg_text_saved;

typedef struct pg_text_grads {
  float* d_token_emb;    /* f32 [vocab, hidden]          (+=) embeddings.token_embedding.weight */
  float* d_pos_emb;      /* f32 [max_positions, hidden]  (+=) embeddings.position_embedding.weight (rows >= S untouched) */
  float* d_final_ln_g;   /* f32 [hidden] (+=) */
  float* d_final_ln_b;   /* f32 [hidden] (+=) */
  const pg_vit_layer_bwd* layers_host;  /* [layers]: every layer's gradients are required */
} pg_text_grads;

/* pg_text_forward with the activations the backward needs kept in `saved` (HF CLIPTextTransformer.forward):
 * pooled_out f32 [n, hidden] = final_layer_norm(x)[b, argmax_t input_ids[b, t]]. */
int pg_text_forward_train(pg_text* h, const int64_t* input_ids, const int64_t* attention_mask, int32_t n, int32_t S,
                          const pg_text_saved* saved, float* pooled_out, void* stream);
size_t pg_text_backward_workspace_bytes(const pg_text* h, int32_t n, int32_t S);
/* d_pooled f32 [n, hidden] (gradient of pooled_out) with the input_ids / attention_mask of the forward -> every text-tower
 * gradient (+=): final_layer_norm on the pooled rows, the encoder layers, d position_embedding[:S] = sums over captions,
 * d token_embedding = per-id sums over the n*S rows in a fixed order (deterministic; ids outside [0, vocab) skipped). */
int pg_text_backward(pg_text* h, const pg_text_saved* saved, const int64_t* input_ids, const int64_t* attention_mask,
                     const float* d_pooled, int32_t n, int32_t S, const pg_text_grads* grads, void* workspace,
                     size_t workspace_bytes, void* stream);

/* clip_loss of HF CLIPModel.forward (modeling_clip.py 4.23.1 `clip_loss(logits_per_text)`) and its gradient, for n images
 * and n captions: img, txt f32 [n, P] (projected, not normalised), logit_scale: DEVICE f32 scalar (the parameter; s = exp)
 *   -> loss f32 [1];  d_img, d_txt f32 [n, P] and d_logit_scale f32 [1] (overwritten, times grad_scale), with
 *      L = s T^ I^T, dL = (softmax_rows(L) - 1 + softmax_cols(L) - 1) / 2n, dT^ = s dL I^, dI^ = s dL^T T^,
 *      d logit_scale = sum dL o L, dT = (dT^ - T^ (T^ . dT^)) / |T| (and the same for I);
 *   -> optional (NULL = not written) logits_per_image / logits_per_text f32 [n, n].
 * Products and normalisation in fp32, sums and the softmax in fp64; deterministic. */
size_t pg_clip_loss_grad_workspace_bytes(int32_t n, int32_t P);
int pg_clip_loss_grad(const float* img, const float* txt, int32_t n, int32_t P, const float* logit_scale, double grad_scale,
                      void* workspace, size_t workspace_bytes, float* loss, float* d_img, float* d_txt, float* d_logit_scale,
                      float* logits_per_image, float* logits_per_text, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * ProtoRefiner (reference models/proto_refiner.py:121-255, 332-357; preprocessing/geo_utils.py:40-55)
 * ------------------------------------------------------------------------------------------------- */
typedef struct pg_refiner_bank {
  int32_t num_cells;           /* C */
  int32_t dim;                 /* D, multiple of 128, <= 1024 */
  const int64_t* cell_off;     /* [C+1] prototype range per geocell; empty range <=> protos[cell] is None */
  const float* proto_emb;      /* [P, D] */
  const float* proto_lnglat;   /* [P, 2] (lng, lat) */
  const int32_t* proto_count;  /* [P] */
  const int64_t* member_off;   /* [P+1] */
  const int64_t* member_idx;   /* [sum count] rows of data_emb/data_lnglat */
  const float* data_emb;       /* [Ntrain, D] */
  const float* data_lnglat;    /* [Ntrain, 2] */
  const float* proto_sqnorm;   /* [P] squared L2 norm of every prototype row (pg_refiner_bank_sqnorm), or NULL: the scans
                                  that need it (schedules 3, 4) are then replaced by the ones that do not */
  int64_t num_protos;          /* P = rows of proto_emb (bounds the TMA tensor map of schedule 4), or 0 */
  int32_t live_cells;          /* geocells with at least one prototype (a cell-sharded bank holds 1/N of them), or 0 = unknown:
                                  the automatic schedule sizes its work units by num_protos / live_cells */
} pg_refiner_bank;

/* |p|^2 of every row of proto_emb f32 [P, D] -> sqnorm_out f32 [P]; once per bank (the squared Euclidean distance of
 * reference models/proto_refiner.py:176-178 in the |p|^2 + |q|^2 - 2 p.q form torch.cdist itself uses). */
int pg_refiner_bank_sqnorm(const float* proto_emb, int64_t P, int32_t D, float* sqnorm_out, void* stream);

size_t pg_refiner_workspace_bytes(int64_t B, int32_t topk, int32_t D, int32_t num_cells);
/* The two stages of pg_refiner_forward as separate calls, for a CELL-SHARDED bank across GPUs (rank r holds the geocells with
 * cell % world == r, every other cell range empty): pg_refiner_scan on every rank over ALL queries -> per (query, candidate)
 * partials best_logit f32 [B, topk] (-100000 where this rank does not hold the cell), best_lnglat f32 [B, topk, 2],
 * best_proto i32 [B, topk]; the caller merges the ranks' partials by owner (one small all-gather), then pg_refiner_finalize
 * (temperature softmax x candidate probabilities, haversine gate, arg-max: reference models/proto_refiner.py:187-231). */
int pg_refiner_scan(const pg_refiner_bank* bank, const float* emb, int64_t B, int32_t V, const int64_t* cand_idx,
                    int32_t cand_stride, int32_t topk, void* workspace, size_t workspace_bytes, float* best_logit,
                    float* best_lnglat, int32_t* best_proto, void* stream);
int pg_refiner_finalize(const float* best_logit, const float* best_lnglat, const double* init_lnglat,
                        const int64_t* cand_idx, const float* cand_prob, int32_t cand_stride, int64_t B, int32_t topk,
                        float temperature, double max_refinement_km, float* out_lnglat, int64_t* out_cell, int32_t* choice,
                        void* stream);
/* Measurement aid: scan schedule of pg_refiner_forward for this process: 0 = automatic (cell-major when geocells are shared
 * by >= 2 (query, candidate) pairs on average; the slab scan when the bank carries proto_sqnorm / num_protos and its geocells
 * hold >= 256 prototypes on average over the non-empty ones), 1 = query-major, 2 = cell-major, 3 = tile scan, 4 = slab scan.  Same selections. */
int pg_refiner_set_schedule(int32_t mode);
/* emb f32 [B, V, D]; init_lnglat f64 [B, 2]; cand_idx i64 [B, cand_stride]; cand_prob f32 [B, cand_stride];
 * only the first `topk` candidates of each row are used (topk <= cand_stride).
 *   -> out_lnglat f32 [B, 2], out_cell i64 [B]   (ProtoRefiner.forward's preds_LLH, preds_geocell)
 *   -> optional debug outputs (may be NULL): best_logit f32 [B, topk] (negative Euclidean distance to the
 *      nearest prototype, -100000 for an empty cell), best_lnglat f32 [B, topk, 2], best_proto i32 [B, topk],
 *      choice i32 [B] (index into the candidate list that was emitted). */
int pg_refiner_forward(const pg_refiner_bank* bank, const float* emb, int64_t B, int32_t V,
                       const double* init_lnglat, const int64_t* cand_idx, const float* cand_prob,
                       int32_t cand_stride, int32_t topk, float temperature, double max_refinement_km,
                       void* workspace, size_t workspace_bytes, float* out_lnglat, int64_t* out_cell,
                       float* best_logit, float* best_lnglat, int32_t* best_proto, int32_t* choice, void* stream);

/* Prototype-bank builder (reference models/proto_refiner.py:359-378 `_compute_protos_for_cell`, the arithmetic of
 * `load_prototypes`): data_views f32 [N, V, D] training embeddings (V = 4 for panoramas, 1 otherwise)
 *   -> data_mean_out f32 [N, D]  (view mean, what `data_emb` of pg_refiner_bank holds)
 *   -> proto_emb_out f32 [P, D]  (mean over member_idx[member_off[p] .. member_off[p+1]) of data_mean rows). */
int pg_bank_build(const float* data_views, int64_t N, int32_t V, int32_t D, const int64_t* member_off,
                  const int64_t* member_idx, int64_t P, float* data_mean_out, float* proto_emb_out, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Per-launch device timing (measurement aid for bench.py; not part of the reference-facing surface).
 * begin: subsequent launches of this library are bracketed with CUDA events on their launch stream;
 * end: synchronises the device, stops recording and returns the number of kernel families seen;
 * read: fills `n` entries (family name, summed milliseconds, launch count).
 * ------------------------------------------------------------------------------------------------- */
void pg_profile_begin(void);
int pg_profile_end(void);
void pg_profile_read(const char** names, float* ms, int32_t* counts, int32_t n);

/* ---------------------------------------------------------------------------------------------------
 * Multi-GPU exchange (SURVEY.md 8e): the all-gather of per-rank results that the reference does with accelerate's
 * `gather` (preprocessing/embed.py:36-37; in evaluation the per-rank head outputs before the retrieval step).  One process
 * per GPU.  NCCL is resolved at run time by soname (libnccl.so.2): no link-time dependency, never loaded by single-GPU callers.
 * ------------------------------------------------------------------------------------------------- */
/* id128: HOST buffer of 128 bytes (ncclUniqueId).  Rank 0 creates it and hands it to the other ranks by any side channel. */
int pg_nccl_unique_id(void* id128);
/* Collective over the n_ranks processes (ncclCommInitRank on the current device).  *comm is an ncclComm_t. */
int pg_nccl_comm_create(const void* id128, int32_t n_ranks, int32_t rank, void** comm);
void pg_nccl_comm_destroy(void* comm);
/* recv[r * bytes_per_rank ...] = rank r's send[0 .. bytes_per_rank), for every r, enqueued on `stream` (ncclAllGather of
 * bytes: the caller packs whatever it exchanges - embeddings f32 [B, V, D], top-k candidates, predictions - into one
 * buffer, as pigeon_b200/dist.py does).  `comm` may also be a communicator the host created itself with NCCL. */
int pg_allgather_embeddings(void* comm, const void* send, void* recv, size_t bytes_per_rank, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Building blocks (exported for unit tests and for callers that fuse differently)
 * ------------------------------------------------------------------------------------------------- */
enum {
  PG_EPI_F16_BIAS = 0,       /* out fp16 = A W^T + bias                       (q/k/v projection) */
  PG_EPI_F16_BIAS_QGELU = 1, /* out fp16 = quick_gelu(A W^T + bias)            (mlp.fc1)          */
  PG_EPI_F32_BIAS_RESID = 2, /* out f32 += A W^T + bias                        (out_proj, mlp.fc2) */
  PG_EPI_F32_BIAS = 3,       /* out f32 = A W^T + bias (bias may be NULL)                          */
  /* the remaining epilogues are reached only through pg_gemm_problem_run (the towers use them internally) */
  PG_EPI_F32_ROWMAP = 4,     /* out f32 [mul * (r / div) + r % div + add] = A W^T + bias   (patch embedding -> token rows) */
  PG_EPI_BF16_DGELU = 5,     /* out bf16 = (A W^T) * quick_gelu'(aux fp16)                  (backward through mlp.fc1's activation) */
  PG_EPI_F16_BIAS_QGELU_SAVE = 6,  /* out fp16 = quick_gelu(A W^T + bias), aux fp16 = A W^T + bias  (training forward of mlp.fc1) */
  PG_EPI_F32_BIAS_RESID_STATS = 7, /* PG_EPI_F32_BIAS_RESID, aux fp16 = the new residual row, stats[r][c / 128] = (sum, sum of squares)
                                      of those fp16 values over 128 columns   (LayerNorm producer: out_proj, fc2) */
  PG_EPI_F16_LN_BIAS = 8,    /* out fp16 = rstd * (A W^T - mu * colsum) + bias, (mu, rstd) of row r of A from stats [M, K / 128]
                                (LayerNorm consumer: qkv; W = gamma-scaled weight, bias = b + W beta, colsum = row sums of W) */
  PG_EPI_F16_LN_BIAS_QGELU = 9     /* quick_gelu of the same                                    (LayerNorm consumer: fc1) */
};
/* D[M,N] = A[M,K] (fp16, row stride lda) * W[N,K]^T (fp16, row stride ldw), fp32 accumulate on wgmma. */
int pg_gemm_f16(const void* a, int32_t lda, const void* w, int32_t ldw, void* out, int32_t ldo, const float* bias,
                int32_t M, int32_t N, int32_t K, int32_t epilogue, void* stream);
/* Kernel of every K-major GEMM (pg_gemm_f16, pg_gemm_ex and the towers), process-wide: 0 = automatic (default; the 128 x 256
 * kernel for the fp16-output epilogues without side outputs and the fp32 residual epilogues when ldo % 8 == 0, else the
 * ping-pong kernel, whose epilogues overlap the next tile's MMAs), 1 = the single-warpgroup kernel, 2 = the ping-pong kernel.  All give the same bits; the
 * switch exists for tests and A/B benchmarks, not for tuning.  PG_GEMM_SCHEDULE=1 or 2 only sets the initial value, once. */
int pg_gemm_set_schedule(int32_t mode);
/* pg_gemm_f16 with bf16 operands (operand_bf16 != 0: BOTH a and w are bf16 — the tensor cores reject mixed pairs) and,
 * for PG_EPI_F32_BIAS_RESID, an out-of-place residual source
 * `resid` f32 [M, ldo] (NULL = update `out` in place). */
int pg_gemm_ex(const void* a, int32_t lda, const void* w, int32_t ldw, void* out, int32_t ldo, const float* bias,
               const float* resid, int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t operand_bf16, void* stream);
/* D[M, N] (+)= a^T w with BOTH operands stored contraction-major: a [K, lda] (M contiguous), w [K, ldw] (N contiguous) —
 * the weight-gradient form dW = dY^T X fed from row-major activations (MN-major wgmma operands, no transposes).
 * M > 128, N % 256 == 0, lda and ldw multiples of 8 (other shapes are rejected); epilogue PG_EPI_F32_BIAS (overwrite) or PG_EPI_F32_BIAS_RESID (accumulate in place). */
int pg_gemm_tn(const void* a, int32_t lda, const void* w, int32_t ldw, float* out, int32_t ldo, int32_t M, int32_t N,
               int32_t K, int32_t accumulate, int32_t operand_bf16, void* stream);
/* The whole GEMM problem, every epilogue (pg_gemm_f16 / pg_gemm_ex / pg_gemm_tn fill a subset of it).  Pointers as in
 * pg_gemm_ex; aux fp16 [M, ldo] for epilogues 5-7 (16-byte aligned); stats float2 (8-byte aligned) [M, N / 128] written by 7,
 * [M, K / 128] read by 8 and 9; colsum f32 [N] (16-byte aligned) and ln_eps for 8 and 9; rowmap_* for 4 (div <= 0 means 1);
 * mn_major != 0 selects pg_gemm_tn's operand layout (a [K, lda], w [K, ldw]).  Shapes an epilogue does not take are rejected
 * before anything is enqueued. */
typedef struct pg_gemm_problem {
  int32_t M, N, K;
  const void* a;
  int32_t lda;
  const void* w;
  int32_t ldw;
  void* out;
  int32_t ldo;
  const float* bias;
  int32_t epilogue;
  int32_t rowmap_div, rowmap_mul, rowmap_add;
  int32_t operand_bf16;
  const float* resid;
  void* aux;
  int32_t mn_major;
  float* stats;
  const float* colsum;
  float ln_eps;
} pg_gemm_problem;
int pg_gemm_problem_run(const pg_gemm_problem* p, void* stream);
/* LayerNorm over the last dim: x f32 [rows, hidden] -> y fp16 [rows, hidden]. */
int pg_layernorm_f16(const float* x, void* y, const float* gamma, const float* beta, int64_t rows, int32_t hidden,
                     float eps, void* stream);
/* softmax(q k^T / 8) v per (view, head); qkv fp16 [n_views*seq, 3*heads*64] -> out fp16 [n_views*seq, heads*64]. */
int pg_attention_f16(const void* qkv, void* out, int32_t n_views, int32_t seq, int32_t heads, void* stream);
/* The text tower's attention (HF CLIPTextTransformer: causal mask + expanded attention_mask, 4.23.1): key j is admissible
 * for query i only if (causal == 0 or j <= i) and (mask == NULL or mask[view, j] != 0); mask i64 [n_views, seq],
 * mask[:, 0] must be non-zero.  mask NULL and causal 0 is pg_attention_f16, bit for bit.  The models pass a 0/1 mask
 * (HF excludes every key whose attention_mask is not exactly 1; CLIPTextTower and the text trainer map it so on the host). */
int pg_attention_f16_masked(const void* qkv, void* out, const int64_t* mask, int32_t causal, int32_t n_views, int32_t seq,
                            int32_t heads, void* stream);
/* The same op with the optional lse2 side output (may be NULL).  `variant` (0..3) and `poly` selected among several forward
 * kernels in earlier versions of this ABI; the sm_90a library has one wgmma kernel, and every variant runs it. */
int pg_attention_f16_variant(const void* qkv, void* out, float* lse2, int32_t n_views, int32_t seq, int32_t heads,
                             int32_t variant, int32_t poly, void* stream);
/* Same, also writing lse2 f32 [n_views*heads, seq] (log2-sum-exp of the scaled logits) for the backward pass. */
int pg_attention_f16_lse(const void* qkv, void* out, float* lse2, int32_t n_views, int32_t seq, int32_t heads, void* stream);
/* Backward of the attention core: qkv f16 [n_views*seq, 3*heads*64], d_out f32 and out f16 [n_views*seq, heads*64],
 * lse2 from the forward -> dqkv bf16 [n_views*seq, 3*heads*64].  workspace: pg_attention_backward_workspace_bytes. */
size_t pg_attention_backward_workspace_bytes(int32_t n_views, int32_t seq, int32_t heads);
int pg_attention_backward(const void* qkv, const void* out, const float* d_out, const float* lse2, void* dqkv_bf16,
                          int32_t n_views, int32_t seq, int32_t heads, void* workspace, size_t workspace_bytes, void* stream);
/* pg_attention_f16_masked also writing lse2 f32 [n_views*heads, seq] over the admissible keys (the text tower's training
 * forward). */
int pg_attention_f16_masked_lse(const void* qkv, void* out, float* lse2, const int64_t* mask, int32_t causal, int32_t n_views,
                                int32_t seq, int32_t heads, void* stream);
/* pg_attention_backward of the masked attention (same admissibility as pg_attention_f16_masked; lse2 from
 * pg_attention_f16_masked_lse).  mask NULL and causal 0 is pg_attention_backward, bit for bit. */
int pg_attention_backward_masked(const void* qkv, const void* out, const float* d_out, const float* lse2, const int64_t* mask,
                                 int32_t causal, void* dqkv_bf16, int32_t n_views, int32_t seq, int32_t heads, void* workspace,
                                 size_t workspace_bytes, void* stream);
/* fp32 LayerNorm: x f32 [rows, hidden] -> y f32 [rows, hidden] (HF nn.LayerNorm in fp32; CLIPModel's post_layernorm input of
 * the visual_projection weight gradient). */
int pg_layernorm_f32(const float* x, float* y, const float* gamma, const float* beta, int64_t rows, int32_t hidden, float eps,
                     void* stream);
/* LayerNorm backward: dx (+)= dLN(x)/dx . dy;  dgamma / dbeta (both or neither NULL) += their gradients;
 * dx_bf16 (nullable): bf16 copy of the final dx, the operand of the next data-gradient GEMM. */
int pg_layernorm_backward(const float* dy, const float* x, const float* gamma, float* dx, int32_t accumulate, float* dgamma,
                          float* dbeta, void* dx_bf16, int64_t rows, int32_t hidden, float eps, void* stream);
/* du bf16 [n] = dh f32 [n] * quick_gelu'(u f16 [n]) */
int pg_dgelu_bf16(const float* dh, const void* u, void* du, int64_t n, void* stream);
/* out bf16 [cols, ldo] = transpose(src [rows, lds]); src_type 0 = f32, 1 = f16, 2 = bf16 */
int pg_transpose_to_bf16(const void* src, int32_t src_type, int64_t lds, void* out, int64_t ldo, int64_t rows, int32_t cols,
                         void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Prototype clustering: the per-geocell OPTICS-xi of reference dataset_creation/prototype/prototype.py:121-145
 * (`ProtoDataset._compute_distances`, `_compute_clusters`), i.e. for every cell
 *   sklearn.cluster.OPTICS(min_samples=m, xi=xi, metric='precomputed').fit_predict(D)
 * with D the fp64 haversine matrix of the cell in km (exact zeros read as 1e-5), restating scikit-learn's
 * compute_optics_graph (max_eps = inf), cluster_optics_xi (min_cluster_size = m, predecessor_correction = True),
 * _xi_cluster and _extract_xi_labels.  D is recomputed on the fly, never stored.
 * ------------------------------------------------------------------------------------------------- */
/* Bytes of workspace pg_optics_xi needs for N points in num_cells cells (about 90 bytes per point). */
size_t pg_optics_workspace_bytes(int64_t N, int32_t num_cells);
/* lnglat_deg f64 [N, 2] (lng, lat in degrees, finite) holds the points grouped by cell: cell c is rows
 * [cell_off[c], cell_off[c+1]) (cell_off i64 [num_cells + 1], cell_off[0] = 0, cell_off[num_cells] = N; empty cells allowed).
 * max_cell is the host-known largest cell size (it sizes shared memory only).  Writes labels_out i32 [N], the cell-local
 * OPTICS-xi label of every point (-1 = noise); a cell of fewer than min_samples points gets label 0 everywhere
 * (prototype.py:144-145).  The optional outputs (NULL = not written) are OPTICS' ordering_ (cell-local indices, at the
 * cell's rows), core_distances_, reachability_ and predecessor_ (cell-local, -1 = none) per point; for a cell below
 * min_samples they hold -1 / NaN / NaN / -1.  Deterministic; no host synchronisation.
 * Fails for min_samples < 2, xi outside (0, 1) or a workspace that is too small. */
int pg_optics_xi(const double* lnglat_deg, int64_t N, const int64_t* cell_off, int32_t num_cells, int64_t max_cell,
                 int32_t min_samples, double xi, void* workspace, size_t workspace_bytes, int32_t* labels_out,
                 int64_t* ordering_out, double* reach_out, double* core_out, int64_t* pred_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * GeoGuessr evaluation metrics (csrc/geo_metrics.cu): reference evaluation/metrics.py compute_geoguessr_metrics.
 *
 * Countries are Polygon / MultiPolygon geometries as CSR arrays, in feature order: verts f64 [num_verts, 2] (lng, lat,
 * finite); ring r is verts[ring_off[r] .. ring_off[r+1]) and is closed (last == first, at least 4 positions); part p
 * (one polygon: its shell, then its holes) is rings [part_ring_off[p], part_ring_off[p+1]); geometry q is parts
 * [geom_part_off[q], geom_part_off[q+1]).  Every offset array is i64, starts at 0 and ends at the next level's count.
 * The index (pg_country_index_bytes) holds bounding boxes and per-part latitude bands; `entries` (i32 [num_entries])
 * lists each band's edges.  Build: pg_country_index_build writes the entry count to *num_entries_out (device i64);
 * the caller allocates the entries and calls pg_country_index_fill.  Both are deterministic.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct {
  const double* verts;
  const int64_t* ring_off;
  const int64_t* part_ring_off;
  const int64_t* geom_part_off;
  int64_t num_verts, num_rings, num_parts, num_geoms;
  void* index;
  size_t index_bytes;
  int32_t* entries;
  int64_t num_entries;
} PgCountries;

#define PG_COUNTRY_NEAREST 1 /* flags: the label is covered by no geometry; its country is the nearest one */

size_t pg_country_index_bytes(int64_t num_verts, int64_t num_parts, int64_t num_geoms);
int pg_country_index_build(const PgCountries* countries, int64_t* num_entries_out, void* stream);
int pg_country_index_fill(const PgCountries* countries, void* stream);
/* Per sample n (label_lnglat, pred_lnglat f64 [N, 2]): country_out i32 = the lowest-index geometry that covers the label
 * (boundary included), else the nearest geometry by GEOS Distance::pointToSegment in degrees (lowest index on exact
 * ties) with PG_COUNTRY_NEAREST in flags_out u8; pred_inside_out u8 (optional) = that geometry contains the prediction
 * (interior only).  Exact orientation predicates, GEOS semantics (DESIGN.md §1).  No host synchronisation. */
int pg_country_locate(const PgCountries* countries, const double* label_lnglat, const double* pred_lnglat, int64_t N,
                      int32_t* country_out, uint8_t* flags_out, uint8_t* pred_inside_out, void* stream);

/* results_out f64 [PG_GEO_NUM_RESULTS] of pg_geo_metrics */
#define PG_GEO_MEAN_KM 0
#define PG_GEO_MEDIAN_KM 1
#define PG_GEO_UNDER_KM 2 /* 10 shares: distance < 1, 5, 10, 25, 50, 100, 200, 750, 1000, 2500 km */
#define PG_GEO_COUNTRY 12
#define PG_GEO_SCORE 13
#define PG_GEO_TOP1 14
#define PG_GEO_TOPK 15
#define PG_GEO_NUM_RESULTS 16
size_t pg_geo_metrics_workspace_bytes(int64_t N);
/* One pass over N >= 1 samples: pred_lnglat [N, 2] (f32 when pred_is_f32, else f64), label_lnglat f64 [N, 2],
 * cell_pred / cell_label i64 [N], topk i64 [N, k], pred_inside u8 [N] (pg_country_locate).  Writes dist_out f64 [N]
 * (haversine_np km, numpy 2 dtype rules) and results_out: mean and median (np.median) km, the Under_*_km shares, country
 * accuracy, mean GeoGuessr score, top-1 and top-k geocell accuracy.  Fixed-order reductions; no host synchronisation. */
int pg_geo_metrics(const void* pred_lnglat, int32_t pred_is_f32, const double* label_lnglat, int64_t N,
                   const int64_t* cell_pred, const int64_t* cell_label, const int64_t* topk, int32_t k,
                   const uint8_t* pred_inside, void* workspace, size_t workspace_bytes, double* dist_out,
                   double* results_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PIGEON_B200_H_ */
