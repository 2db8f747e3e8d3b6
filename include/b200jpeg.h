/*
 * b200jpeg.h -- C-ABI of the GPU-native (H100) JPEG encode hot path.
 *
 * Drop-in boundary for the encoder pipeline of mozilla/mozjpeg (libjpeg-turbo
 * 3.0.x + Mozilla encoder extensions).  Everything here is `extern "C"`, plain
 * pointers and sizes.  Each entry point names the reference interface it
 * replaces (file:line under the reference tree) so parity can be checked.
 *
 * Two groups:
 *   1. HOST-ONLY parameter logic (no GPU needed): mirrors the reference's
 *      jcparam.c / jcext.c / jcmaster.c decisions, because the output bytes
 *      depend on them (quant tables, sampling, scan script, pass plan).
 *   2. ENCODE entry points: stage pixels in HBM and run the sm_90a kernels
 *      (colour conversion + downsample, FDCT + quantize + deringing, trellis
 *      quantization, Huffman statistics / optimal tables / bit packing).
 *
 * There is NO CPU fallback: group 2 fails with B200JPEG_ERR_NO_DEVICE when no
 * CUDA device is usable.
 */
#ifndef B200JPEG_H
#define B200JPEG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200JPEG_MAX_COMPONENTS 4      /* subset of MAX_COMPONENTS (jmorecfg.h:33) we accept */
#define B200JPEG_NUM_QUANT_TBLS 4      /* NUM_QUANT_TBLS  jpeglib.h:50  */
#define B200JPEG_NUM_HUFF_TBLS  4      /* NUM_HUFF_TBLS   jpeglib.h:51  */
#define B200JPEG_MAX_SCANS      64     /* largest script the reference builds (jcparam.c:748-850) */
#define B200JPEG_DCTSIZE2       64

/* J_COLOR_SPACE subset (jpeglib.h:243-266), same numeric values. */
enum { B200JPEG_CS_UNKNOWN = 0, B200JPEG_CS_GRAYSCALE = 1, B200JPEG_CS_RGB = 2, B200JPEG_CS_YCbCr = 3,
       B200JPEG_CS_CMYK = 4, B200JPEG_CS_YCCK = 5,   /* 4 samples per pixel; CMYK -> YCCK as Adobe defines it (jccolor.c:395-441) */
       /* input pixel orders of the RGB family (in_color_space only; jccolor.c:253-291 dispatches them into jccolext.c:30-75):
        * 3 samples per pixel for EXT_RGB / EXT_BGR, 4 for the others (the filler / alpha sample is ignored) */
       B200JPEG_CS_EXT_RGB = 6, B200JPEG_CS_EXT_RGBX = 7, B200JPEG_CS_EXT_BGR = 8, B200JPEG_CS_EXT_BGRX = 9,
       B200JPEG_CS_EXT_XBGR = 10, B200JPEG_CS_EXT_XRGB = 11, B200JPEG_CS_EXT_RGBA = 12, B200JPEG_CS_EXT_BGRA = 13,
       B200JPEG_CS_EXT_ABGR = 14, B200JPEG_CS_EXT_ARGB = 15 };
/* RGB-family test and layout of an in_color_space value: samples per pixel, index of the first colour sample, blue-first */
#define B200JPEG_CS_IS_RGB(cs) ((cs) == B200JPEG_CS_RGB || ((cs) >= B200JPEG_CS_EXT_RGB && (cs) <= B200JPEG_CS_EXT_ARGB))
#define B200JPEG_CS_PIXELSIZE(cs) (((cs) == B200JPEG_CS_RGB || (cs) == B200JPEG_CS_EXT_RGB || (cs) == B200JPEG_CS_EXT_BGR) ? 3 : 4)
#define B200JPEG_CS_FIRST(cs) (((cs) == B200JPEG_CS_EXT_XBGR || (cs) == B200JPEG_CS_EXT_XRGB || (cs) == B200JPEG_CS_EXT_ABGR || (cs) == B200JPEG_CS_EXT_ARGB) ? 1 : 0)
#define B200JPEG_CS_BLUE_FIRST(cs) ((cs) == B200JPEG_CS_EXT_BGR || (cs) == B200JPEG_CS_EXT_BGRX || (cs) == B200JPEG_CS_EXT_XBGR || (cs) == B200JPEG_CS_EXT_BGRA || (cs) == B200JPEG_CS_EXT_ABGR)
/* J_DCT_METHOD (jpeglib.h:275-279); all three are on the device path, at 8 and at 12 bits. */
enum { B200JPEG_DCT_ISLOW = 0, B200JPEG_DCT_IFAST = 1, B200JPEG_DCT_FLOAT = 2 };
/* JINT_COMPRESS_PROFILE values (jpeglib.h:349-352). */
enum { B200JPEG_PROFILE_MAX_COMPRESSION = 0x5D083AAD, B200JPEG_PROFILE_FASTEST = 0x2AEA5CB4 };

/* Error codes (returned negative).  The reference reports errors through
 * err->error_exit (jerror.h); a libjpeg shim maps these to ERREXIT codes. */
enum {
  B200JPEG_OK = 0,
  B200JPEG_ERR_PARAM = -1,        /* ~ JERR_BAD_* parameter validation (jcmaster.c initial_setup) */
  B200JPEG_ERR_UNSUPPORTED = -2,  /* valid for the reference, not (yet) on the device path */
  B200JPEG_ERR_NO_DEVICE = -3,    /* no CUDA device / driver: there is no CPU fallback */
  B200JPEG_ERR_CUDA = -4,         /* a CUDA call failed (message via b200jpeg_last_error) */
  B200JPEG_ERR_BUFFER = -5,       /* output buffer too small */
  B200JPEG_ERR_BAD_DCT_COEF = -6, /* ~ JERR_BAD_DCT_COEF (jchuff.c:596-600) */
  B200JPEG_ERR_STATE = -7         /* ~ JERR_BAD_STATE: streaming calls out of order */
};

/* jpeg_scan_info (jpeglib.h:205-210) */
typedef struct {
  int comps_in_scan;
  int component_index[B200JPEG_MAX_COMPONENTS];
  int Ss, Se, Ah, Al;
} b200jpeg_scan_info;

/* the fields of jpeg_component_info the encoder reads (jpeglib.h:124-199) */
typedef struct {
  int component_id;
  int h_samp_factor, v_samp_factor;
  int quant_tbl_no, dc_tbl_no, ac_tbl_no;
} b200jpeg_component_info;

/* JHUFF_TBL (jpeglib.h:109-119) */
typedef struct {
  uint8_t bits[17];
  uint8_t huffval[256];
  int present;
} b200jpeg_huff_tbl;

/*
 * The encoder-relevant fields of jpeg_compress_struct (jpeglib.h:388-561) and of
 * the mozjpeg extension block jpeg_comp_master (jpegint.h:93-135), under the
 * reference's field names.
 */
typedef struct {
  /* source image (jpeglib.h:396-402) */
  int image_width, image_height;
  int input_components;
  int in_color_space;                     /* B200JPEG_CS_* (UNKNOWN: input_components samples, 1 to 4, passed through) */
  int data_precision;                     /* 8, or 12 (samples in uint16; trellis and deringing off, as the reference requires), or 16 (lossless only) */
  /* JPEG parameters */
  int jpeg_color_space;
  int num_components;
  b200jpeg_component_info comp_info[B200JPEG_MAX_COMPONENTS];
  uint16_t quant_tbl[B200JPEG_NUM_QUANT_TBLS][B200JPEG_DCTSIZE2];  /* natural order, like JQUANT_TBL.quantval */
  int quant_tbl_present[B200JPEG_NUM_QUANT_TBLS];
  b200jpeg_huff_tbl dc_huff_tbl[B200JPEG_NUM_HUFF_TBLS];
  b200jpeg_huff_tbl ac_huff_tbl[B200JPEG_NUM_HUFF_TBLS];
  int num_scans;                          /* 0 => one sequential scan of all components */
  b200jpeg_scan_info scan_info[B200JPEG_MAX_SCANS];
  int optimize_coding;
  int dct_method;
  int restart_interval;                   /* MCUs; 0 = none */
  int restart_in_rows;
  int smoothing_factor;                   /* 0..100 (jcsample.c:298-455; ignored for raw-data input) */
  int write_JFIF_header;
  int JFIF_major_version, JFIF_minor_version;
  int density_unit, X_density, Y_density;
  int write_Adobe_marker;
  /* mozjpeg extension parameters (jpegint.h:93-135, jcext.c) */
  int compress_profile;
  int optimize_scans;                     /* scan search over the jpeg_search_progression candidates (jcmaster.c:773-962) */
  int trellis_quant;
  int trellis_quant_dc;
  int trellis_eob_opt;                    /* block-level EOB-run optimisation along each block row (jcdctmgr.c:1224-1297) */
  int use_lambda_weight_tbl;              /* no effect in the reference (jcdctmgr.c:971,1017) */
  int use_scans_in_trellis;               /* trellis in two AC bands split at trellis_freq_split (jcmaster.c:451-467) */
  int trellis_q_opt;                      /* re-fit the quantization tables to the kept coefficients (jcmaster.c:1014-1030); per image */
  int overshoot_deringing;
  int trellis_freq_split;
  int trellis_num_loops;                  /* 1..16 rounds of statistics + trellis per component (jcmaster.c:453-465) */
  int quant_tbl_master_idx;               /* JINT_BASE_QUANT_TBL_IDX */
  int dc_scan_opt_mode;
  float lambda_log_scale1, lambda_log_scale2;
  float trellis_delta_dc_weight;          /* cjpeg -trellis-dc-ver-weight (jcdctmgr.c:1069-1086) */
  /* cjpeg keeps these outside cinfo (rdswitch.c:509): per-slot linear scale factors */
  int q_scale_factor[B200JPEG_NUM_QUANT_TBLS];
} b200jpeg_params;

/* ------------------------------------------------------------------ */
/* 1. Host-only parameter logic (mirrors of the reference's API).      */
/* ------------------------------------------------------------------ */

/* jpeg_CreateCompress + jpeg_set_defaults (jcapimin.c:34-110, jcparam.c:386-519).
 * `profile` is what JINT_COMPRESS_PROFILE would hold; in_color_space and
 * input_components must be set in *p before the call, like the reference. */
void b200jpeg_set_defaults(b200jpeg_params *p, int profile);
/* jpeg_default_colorspace / jpeg_set_colorspace (jcparam.c:526-652) */
int  b200jpeg_default_colorspace(b200jpeg_params *p);
int  b200jpeg_set_colorspace(b200jpeg_params *p, int colorspace);
/* jpeg_quality_scaling / jpeg_float_quality_scaling (jcparam.c:328-357) */
int   b200jpeg_quality_scaling(int quality);
float b200jpeg_float_quality_scaling(float quality);
/* jpeg_add_quant_table (jcparam.c:31-68) */
int  b200jpeg_add_quant_table(b200jpeg_params *p, int which_tbl, const unsigned int *basic_table,
                              int scale_factor, int force_baseline);
/* jpeg_set_linear_quality / jpeg_set_quality (jcparam.c:311-373) */
void b200jpeg_set_linear_quality(b200jpeg_params *p, int scale_factor, int force_baseline);
void b200jpeg_set_quality(b200jpeg_params *p, int quality, int force_baseline);
/* cjpeg's jpeg_default_qtables: per-slot q_scale_factor (rdswitch.c:509-521) */
void b200jpeg_default_qtables(b200jpeg_params *p, int force_baseline);
/* jpeg_simple_progression (jcparam.c:859-1004); with optimize_scans set it installs the candidate script of
 * jpeg_search_progression (jcparam.c:733-852: 64 scans, 23 for one component) like the reference. */
int  b200jpeg_simple_progression(b200jpeg_params *p);
/* jpeg_enable_lossless (jcparam.c:1015-1039): lossless (SOF3) coding with predictor psv (1..7) and point transform pt
 * (0..data_precision-1).  Lossless mode is a scan script whose first entry has Ss != 0, Se == 0, as the reference's
 * validate_script detects it (jcmaster.c:302-311).  Without a script (num_scans == 0) or over the one an earlier call
 * installed, this call installs one scan of all components in SOF order and turns the scan search off: it stands in for
 * the reference's scan_info == NULL, follows the component count jpeg_start_compress settles on, and is marked by
 * scan_info[1].comps_in_scan == -1.  A script of several lossless scans may be installed by hand instead.  Over any
 * other installed script the call changes nothing (the reference's validate_script then clears lossless mode), except
 * over the scan search's script, where the reference keeps lossless mode beside progressive mode: B200JPEG_ERR_PARAM
 * with trellis quantization on ("Bogus buffer control mode"), else B200JPEG_ERR_UNSUPPORTED.  Out-of-range values are
 * B200JPEG_ERR_PARAM.
 * At start the reference overrides (jcmaster.c:1072-1094): colour space from jpeg_default_colorspace (an RGB-family
 * input is coded as RGB), 1x1 sampling, no smoothing, optimal Huffman tables.  Precision 8, 12 or 16 (16 only here);
 * trellis quantization must be off; a restart interval must be a whole number of rows; pixels are uint16 at 12 and 16
 * bits and are not masked (12-bit samples are read as J12SAMPLE, i.e. signed short).  The raw-data and coefficient entry
 * points refuse lossless parameter blocks. */
int  b200jpeg_enable_lossless(b200jpeg_params *p, int psv, int pt);
/* std_huff_tables (jstdhuff.c) */
void b200jpeg_std_huff_tables(b200jpeg_params *p);
/* the base tables of jcparam.c:76-292, for inspection: 9 sets x {luma,chroma} */
const unsigned int *b200jpeg_std_quant_tbl(int set_idx, int chroma);

/* Parameter validation + derived geometry: jcmaster.c initial_setup (:118-249),
 * validate_script (:252-436) and per-scan setup.  Returns B200JPEG_OK, or an
 * error and a message retrievable with b200jpeg_last_error(). */
int  b200jpeg_validate(const b200jpeg_params *p);

/* total_passes as jinit_c_master_control computes it (jcmaster.c:1114-1139);
 * what a progress monitor would be told. */
int  b200jpeg_total_passes(const b200jpeg_params *p);

/* ------------------------------------------------------------------ */
/* 2. Encode entry points (device path).                               */
/* ------------------------------------------------------------------ */

typedef struct b200jpeg_encoder b200jpeg_encoder;

/* Create an encoder bound to CUDA device `device` (own stream, own HBM arenas). */
int  b200jpeg_encoder_create(b200jpeg_encoder **enc, int device);
void b200jpeg_encoder_destroy(b200jpeg_encoder *enc);
/* Run on a caller-owned CUDA stream (a cudaStream_t passed as void*; NULL = the
 * legacy default stream) instead of the encoder's own, so that the caller can
 * bracket the work with its own events. */
int  b200jpeg_encoder_set_stream(b200jpeg_encoder *enc, void *cuda_stream);

/* A batch is processed in chunks of images: the host->device staging of chunk
 * k+1 and the read-back of chunk k-1 overlap the kernels of chunk k, and the
 * intermediate HBM arenas are sized for one chunk.  0 = automatic (about 1.6 M
 * 8x8 blocks per chunk, i.e. 8 images of 3840x2160 4:2:0). */
int  b200jpeg_encoder_set_chunk_images(b200jpeg_encoder *enc, int images_per_chunk);
/* Images per chunk the last batch was processed with (= images per kernel launch). */
int  b200jpeg_last_chunk_images(const b200jpeg_encoder *enc);
/* Consecutive chunks rotate over `n_streams` (1 to 4, default 2; B200JPEG_STREAMS in the environment) compute
 * streams, each with its own intermediate arenas, so that one chunk's
 * latency-bound phases (serial Huffman table construction, trellis chains)
 * overlap the other's bandwidth-bound ones.  With 1 stream the per-stage times
 * of b200jpeg_last_stage_times() are those of kernels running alone. */
int  b200jpeg_encoder_set_streams(b200jpeg_encoder *enc, int n_streams);

/*
 * Encode a batch of `n_images` images that share one parameter set and one
 * geometry.  Replaces, per image, jpeg_start_compress (jcapistd.c:44-70) +
 * jpeg_write_scanlines (jcapistd.c:90-135) for all rows + jpeg_finish_compress
 * (jcapimin.c:176-229) with a memory destination (jdatadst.c:237-291).
 *
 * pixels      : first sample of image 0.  8-bit interleaved samples,
 *               input_components per pixel (RGB order for B200JPEG_CS_RGB).
 * pixels_on_device : 0 = host memory (staged with cudaMemcpyAsync inside the
 *               call; pinned memory recommended), 1 = device pointer (HBM).
 * row_pitch   : bytes between rows;  image_stride: bytes between images.
 * The finished JPEG files stay in the encoder (pinned host memory) until the
 * next encode call; read them with b200jpeg_get_output().
 */
int  b200jpeg_encode_batch(b200jpeg_encoder *enc, const b200jpeg_params *p,
                           const void *pixels, int pixels_on_device,
                           size_t row_pitch, size_t image_stride, int n_images);

/*
 * Raw-data variant: replaces jpeg_write_raw_data (jcapistd.c:145-195; the entry point under tj3CompressFromYUV*):
 * the caller supplies already converted and downsampled component planes, 8-bit samples.  planes[ci] points at
 * image 0's plane of component ci, which must hold at least height_in_blocks*8 rows of width_in_blocks*8 samples
 * (the library does no edge expansion on this path, exactly like the reference); row_pitch[ci] / image_stride[ci]
 * in bytes.  in_color_space / input_components of the parameter block are ignored.
 */
int  b200jpeg_encode_batch_raw(b200jpeg_encoder *enc, const b200jpeg_params *p,
                               const uint8_t *const *planes, int planes_on_device,
                               const size_t *row_pitch, const size_t *image_stride, int n_images);

/*
 * Coefficient-domain variant: replaces jpeg_write_coefficients + jpeg_finish_compress (jctrans.c:39-66, the encode
 * half of jpegtran): the caller supplies already QUANTIZED DCT coefficients and the path runs only its entropy-coding
 * stages (optimal tables, sequential / progressive scans, scan search, restarts).  planes[ci] points at image 0's
 * blocks of component ci in the libjpeg JBLOCK layout (64 int16 per block, natural order), height_in_blocks rows of
 * width_in_blocks blocks; row_pitch_blocks[ci] / image_stride_blocks[ci] in blocks.  Dummy blocks are generated like
 * compress_output does (jctrans.c:352-362).  The parameter block is what jpeg_copy_critical_parameters (jctrans.c:
 * 76-166) plus the caller's changes would hold: trellis_quant must be 0; in_color_space / input_components,
 * dct_method, smoothing and deringing have no meaning here.
 */
int  b200jpeg_encode_batch_coefs(b200jpeg_encoder *enc, const b200jpeg_params *p,
                                 const int16_t *const *planes, int planes_on_device,
                                 const size_t *row_pitch_blocks, const size_t *image_stride_blocks, int n_images);

/*
 * Per-image quantization tables: the three batch entry points above with one table set per image.  Image i is the
 * file the reference writes for it from a compress object holding `p` with quant_tbl replaced by image i's tables:
 * its DQT, its choice between SOF0 and SOF1 (a table entry above 255 makes it SOF1) and its quantization come from
 * them; everything else (geometry, sampling, scan script, trellis and Huffman options, markers, precision) is p's.
 *
 * qtables     : n_images x B200JPEG_NUM_QUANT_TBLS x 64 entries, natural order (like JQUANT_TBL.quantval); only the
 *               slots p->quant_tbl_present names are read.  Every entry read must lie in 1..32767 (the range
 *               jpeg_add_quant_table clamps to), else B200JPEG_ERR_PARAM naming the image and the slot.  With the
 *               trellis on, a table whose entries lie too far apart for the device divider returns
 *               B200JPEG_ERR_UNSUPPORTED naming the image.  A refused batch writes no file.
 * image_stride: may be 0 here (each image_stride[ci] on the raw and coefficient variants): every image then reads
 *               the same pixels, planes or blocks, e.g. one picture at several qualities.  Host input is staged once.
 * Images that share a table set share its device constants; a batch costs the same kernel launches as with one set.
 */
int  b200jpeg_encode_batch_qtables(b200jpeg_encoder *enc, const b200jpeg_params *p,
                                   const void *pixels, int pixels_on_device,
                                   size_t row_pitch, size_t image_stride,
                                   const uint16_t *qtables, int n_images);
int  b200jpeg_encode_batch_raw_qtables(b200jpeg_encoder *enc, const b200jpeg_params *p,
                                       const uint8_t *const *planes, int planes_on_device,
                                       const size_t *row_pitch, const size_t *image_stride,
                                       const uint16_t *qtables, int n_images);
int  b200jpeg_encode_batch_coefs_qtables(b200jpeg_encoder *enc, const b200jpeg_params *p,
                                         const int16_t *const *planes, int planes_on_device,
                                         const size_t *row_pitch_blocks, const size_t *image_stride_blocks,
                                         const uint16_t *qtables, int n_images);

/* b200jpeg_encode_batch, but stops after the entropy-coded bytes are in HBM: no device->host
 * copy, no host-side file assembly.  Used to time the device pipeline alone. */
int  b200jpeg_encode_batch_device_only(b200jpeg_encoder *enc, const b200jpeg_params *p,
                                       const void *pixels_device,
                                       size_t row_pitch, size_t image_stride, int n_images);

/* Size / pointer of finished JPEG file `i` of the last batch (host memory owned
 * by the encoder, valid until the next encode call). */
int  b200jpeg_get_output(b200jpeg_encoder *enc, int i, const uint8_t **data, size_t *size);
/* Total bytes of entropy-coded data produced by the last batch (all scans). */
size_t b200jpeg_last_scan_bytes(const b200jpeg_encoder *enc);
/* Number of kernels this library launched since the encoder was created. */
unsigned long long b200jpeg_kernel_launches(const b200jpeg_encoder *enc);
/* Milliseconds (CUDA events on the encoder's stream) spent in each pipeline
 * stage during the last batch, summed per stage name (one stage = one kernel,
 * except "h2d"); names[] are static strings. Returns the count. */
int  b200jpeg_last_stage_times(const b200jpeg_encoder *enc, const char **names, float *ms, int max);

/* Debug/parity taps: copy intermediate device state of image `i` of the last
 * batch to host (available for the images of the batch's LAST chunk only).  plane: 0 = quantized coefficients entering entropy coding
 * (after trellis, dummy blocks filled), 1 = raw DCT output (x8 scale),
 * 2 = plain-quantized coefficients (before trellis).  Blocks are returned in
 * the reference's layout: [height_in_blocks_padded][width_in_blocks_padded][64]
 * int16 in NATURAL order (JBLOCK, jpeglib.h).  Returns blocks written or <0.
 * Planes 0 and 2 need the encoder created with B200JPEG_KEEP_PLAIN=1 in the environment: without it the
 * pipeline keeps no copy of the plain-quantized plane and, for sequential scans behind the trellis, leaves the final
 * values in compact symbol records instead of writing the coefficient planes back (where the forward kernel also
 * counts the trellis statistics, the plain-quantized values never reach the planes at all). */
long b200jpeg_debug_get_coefs(b200jpeg_encoder *enc, int image, int component, int plane,
                              int16_t *dst, size_t dst_blocks, int *width_in_blocks, int *height_in_blocks);
/* Huffman tables actually written for scan `scan` of image `i` (as in the DHT). */
int  b200jpeg_debug_get_huff(b200jpeg_encoder *enc, int image, int scan, int is_ac, int tbl_no,
                             b200jpeg_huff_tbl *out);

/* Streaming shim in the shape of the libjpeg calls (one image):
 * jpeg_start_compress / jpeg_write_scanlines / jpeg_finish_compress. Rows are
 * copied into a pinned staging buffer during write_scanlines (the caller's
 * rows are not referenced afterwards, like jcapistd.c:90-135); all device work
 * runs in finish_compress. */
int  b200jpeg_start_compress(b200jpeg_encoder *enc, const b200jpeg_params *p);
int  b200jpeg_write_scanlines(b200jpeg_encoder *enc, const uint8_t *const *scanlines, int num_lines);
int  b200jpeg_finish_compress(b200jpeg_encoder *enc, const uint8_t **jpeg, size_t *size);

const char *b200jpeg_last_error(void);
const char *b200jpeg_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200JPEG_H */
