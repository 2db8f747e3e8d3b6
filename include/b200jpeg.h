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
  B200JPEG_ERR_STATE = -7,        /* ~ JERR_BAD_STATE: streaming calls out of order */
  B200JPEG_ERR_BAD_SOURCE = -8    /* a source JPEG file is malformed or its entropy-coded data is corrupt (the message names the image) */
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

/* Size of plane `ci` of the YUV image b200jpeg_encode_yuv_batch writes, as tj3EncodeYUVPlanes8 lays it out
 * (turbojpeg.c:1528-1578): pw0 = image_width padded to a multiple of the largest h_samp_factor, ph0 = image_height
 * padded to a multiple of the largest v_samp_factor; plane ci is pw0 * h_ci / hmax samples wide and
 * ph0 * v_ci / vmax rows high.  B200JPEG_ERR_PARAM for ci outside the components or non-positive sizes / factors. */
int  b200jpeg_yuv_plane_dims(const b200jpeg_params *p, int ci, int *width, int *height);

/* Source-file header parser: the marker segments of a JPEG file as jdmarker.c read_markers walks them (SOI, APPn,
 * DQT, SOF0/SOF1/SOF2, DHT, DRI, SOS, COM, DNL, EOI), for every scan.  Huffman table definitions are pooled in file
 * order; a scan names the definitions in force at its SOS.  In a sequential file, slots 0 and 1 still undefined at the
 * first SOS receive the standard tables, appended to the pool (std_huff_tables, jdhuff.c:819-823).  A component keeps the quantization table its slot held at
 * the component's first scan (latch_quant_tables, jdinput.c:257-283). */
#define B200JPEG_MAX_SOURCE_SCANS 128
#define B200JPEG_MAX_SOURCE_HUFF  64
typedef struct {
  int comps_in_scan;
  int component_index[B200JPEG_MAX_COMPONENTS];
  int dc_huff[B200JPEG_MAX_COMPONENTS], ac_huff[B200JPEG_MAX_COMPONENTS];   /* index into huff[], -1 when undefined */
  int dc_tbl_no[B200JPEG_MAX_COMPONENTS], ac_tbl_no[B200JPEG_MAX_COMPONENTS];
  int Ss, Se, Ah, Al;
  int restart_interval;                   /* DRI in force at this SOS */
  size_t data_offset, data_size;          /* entropy-coded bytes: the end of the SOS header up to the first marker that is
                                             neither RSTn nor a stuffed 0xFF00 (fill bytes before it excluded) */
} b200jpeg_source_scan;
typedef struct {
  int sof;                                /* 0xC0, 0xC1 or 0xC2 */
  int image_width, image_height, data_precision, num_components;
  int component_id[B200JPEG_MAX_COMPONENTS], h_samp_factor[B200JPEG_MAX_COMPONENTS], v_samp_factor[B200JPEG_MAX_COMPONENTS];
  int quant_tbl_no[B200JPEG_MAX_COMPONENTS];
  uint16_t quant_tbl[B200JPEG_NUM_QUANT_TBLS][B200JPEG_DCTSIZE2];   /* the slots as defined before the first SOS, natural order */
  int quant_tbl_present[B200JPEG_NUM_QUANT_TBLS];
  uint16_t comp_quant[B200JPEG_MAX_COMPONENTS][B200JPEG_DCTSIZE2];  /* latched at each component's first scan, natural order */
  int comp_quant_present[B200JPEG_MAX_COMPONENTS];
  int saw_JFIF, JFIF_major_version, JFIF_minor_version, density_unit, X_density, Y_density;
  int saw_Adobe, Adobe_transform;
  int jpeg_color_space;                   /* the guess of default_decompress_parms (jdapimin.c:111-213) */
  int has_extra_markers;                  /* COM, or APPn other than JFIF and Adobe */
  int num_huff;
  b200jpeg_huff_tbl huff[B200JPEG_MAX_SOURCE_HUFF];
  int huff_is_dc[B200JPEG_MAX_SOURCE_HUFF];
  int num_scans;
  b200jpeg_source_scan scans[B200JPEG_MAX_SOURCE_SCANS];
} b200jpeg_source_info;
/* B200JPEG_OK, or B200JPEG_ERR_PARAM for a file that is not a JPEG file or whose header is corrupt,
 * B200JPEG_ERR_UNSUPPORTED for lossless / hierarchical / arithmetic-coded files and component counts other than 1, 3
 * and 4, B200JPEG_ERR_BAD_SOURCE for a header the reference refuses (zero height, bad precision or sampling factors, a
 * Huffman table jpeg_make_d_derived_tbl refuses, a scan naming an undefined table or component, an unknown marker);
 * the message says which. */
int  b200jpeg_parse_source(const uint8_t *data, size_t size, b200jpeg_source_info *out);

/* Lossless transforms (jpegtran -rotate / -flip / -transpose / -transverse / -crop / -trim / -perfect / -grayscale):
 * the fields of jpeg_transform_info (transupp.h) that jpegtran's switches set, and what b200jpeg_transform_setup
 * derives from them.  Transform codes follow JXFORM_CODE, crop kinds JCROP_CODE. */
enum { B200JPEG_XFORM_NONE = 0, B200JPEG_XFORM_FLIP_H, B200JPEG_XFORM_FLIP_V, B200JPEG_XFORM_TRANSPOSE,
       B200JPEG_XFORM_TRANSVERSE, B200JPEG_XFORM_ROT_90, B200JPEG_XFORM_ROT_180, B200JPEG_XFORM_ROT_270 };
enum { B200JPEG_CROP_UNSET = 0, B200JPEG_CROP_POS, B200JPEG_CROP_NEG, B200JPEG_CROP_FORCE, B200JPEG_CROP_REFLECT };
typedef struct {
  /* set by the caller (jtransform_parse_crop_spec for the crop fields) */
  int transform, perfect, trim, force_grayscale;
  int crop;
  unsigned crop_width, crop_height, crop_xoffset, crop_yoffset;
  int crop_width_set, crop_height_set, crop_xoffset_set, crop_yoffset_set;
  /* filled by b200jpeg_transform_setup */
  int num_components;                       /* destination components (1 under -grayscale on a YCbCr source) */
  int output_width, output_height;          /* destination image size */
  int iMCU_sample_width, iMCU_sample_height;
  int x_crop_offset, y_crop_offset;         /* in iMCUs of the destination */
  /* the block mapping of the coefficient import, per destination component ci (source component ci): destination
   * block (row r, column c) reads, along each destination axis, a = c + x_crop_blocks (resp. r + y_crop_blocks),
   * mirrored to x_mirror - 1 - a when a < x_mirror (resp. y_mirror); with `transposed` the x axis indexes source
   * rows and the y axis source columns.  The block's coefficients are transposed with it, and a mirrored axis
   * negates its odd frequencies.  src_wib / src_hib: the source component's real blocks, the only ones read. */
  int transposed;
  int x_crop_blocks[B200JPEG_MAX_COMPONENTS], y_crop_blocks[B200JPEG_MAX_COMPONENTS];
  int x_mirror[B200JPEG_MAX_COMPONENTS], y_mirror[B200JPEG_MAX_COMPONENTS];
  int src_wib[B200JPEG_MAX_COMPONENTS], src_hib[B200JPEG_MAX_COMPONENTS];
} b200jpeg_transform_info;
/* jtransform_request_workspace + jtransform_adjust_parameters (transupp.c) as jpegtran calls them, for a source whose
 * header is `src`, on `p` as jpeg_copy_critical_parameters left it: p receives the destination size, 1x1 sampling for
 * a single component, -grayscale's colour space (component 0 keeps its table slot), and for transposing transforms
 * swapped sampling factors and transposed quantization tables; t receives the derived fields.  Errors (nothing is
 * changed): B200JPEG_ERR_PARAM with "transformation is not perfect" under -perfect, "Invalid crop request" for a crop
 * the reference refuses (JERR_BAD_CROP_SPEC), "Unsupported color conversion request" for -grayscale on a source that
 * is not YCbCr with 3 components or gray with luma at the largest factors (JERR_CONVERSION_NOTIMPL);
 * B200JPEG_ERR_UNSUPPORTED for a crop region larger than the image (crop extension). */
int  b200jpeg_transform_setup(const b200jpeg_source_info *src, b200jpeg_transform_info *t, b200jpeg_params *p);

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

/*
 * YUV encoding: replaces tj3EncodeYUVPlanes8 (turbojpeg.c:1467-1619), the colour conversion and downsampling of a
 * compress without the JPEG stages, for a batch of `n_images` images sharing `p` (what setCompDefaults builds for the
 * pixel format and TJSAMP_*).  Image i's plane ci (component ci of p) goes to planes[ci] + i * plane_stride[ci] as
 * b200jpeg_yuv_plane_dims rows of samples, plane_pitch[ci] bytes apart; bytes between pw and the pitch and between
 * images are not written.  Rows past image_height repeat the last row, columns past image_width the last column,
 * like the reference; the downsamplers are those jinit_downsampler picks without smoothing (jcsample.c:463-545).
 * pixels / pixels_on_device / row_pitch / image_stride as in b200jpeg_encode_batch; planes_on_device says where the
 * planes are.  Host input or output is processed in chunks on the encoder's streams (staging of chunk k+1 and
 * read-back of chunk k-1 overlap chunk k's kernel); with both sides on the device the call only enqueues the kernel
 * on the encoder's stream (b200jpeg_encoder_set_stream) and returns.
 * Besides b200jpeg_validate's checks: precision must be 8 and lossless parameter blocks are B200JPEG_ERR_PARAM, as is
 * a plane pitch below the plane's width or a plane stride below one plane; a smoothing factor, or a sampling layout
 * other than component 0 at the largest factors (1, 2 or 4 each way) with 1x1 components 1 and 2 (every TJSAMP_*),
 * is B200JPEG_ERR_UNSUPPORTED, as are 2 or 4 components.
 */
int  b200jpeg_encode_yuv_batch(b200jpeg_encoder *enc, const b200jpeg_params *p,
                               const void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride,
                               uint8_t *const *planes, int planes_on_device, const size_t *plane_pitch,
                               const size_t *plane_stride, int n_images);

/*
 * Device entropy decode of sequential Huffman JPEG files (SOF0 / SOF1, 8 and 12 bits; one interleaved scan or several
 * non-interleaved ones; restart intervals): replaces jpeg_read_coefficients (jdtrans.c:47-124) for a batch of files of
 * one geometry (size, precision, components and sampling); Huffman tables, quantization tables, restart interval and
 * scan layout may differ per file.  Progressive (SOF2) files are B200JPEG_ERR_UNSUPPORTED: pass their coefficients
 * to b200jpeg_encode_batch_coefs instead.  Corrupt entropy-coded data (an invalid code, too few bits for a segment's
 * MCUs, a wrong RSTn, an unexpected marker) is B200JPEG_ERR_BAD_SOURCE naming the first such image; the reference only
 * warns there and fills the gap.  Bytes after a segment's last MCU are ignored, like the reference does.
 *
 * b200jpeg_decode_coefs_batch writes the real blocks of image i's component ci, natural-order JBLOCKs, to planes[ci] +
 * i * image_stride_blocks[ci] blocks, height_in_blocks rows of width_in_blocks blocks row_pitch_blocks[ci] apart, in
 * host or device memory (planes_on_device).
 */
int  b200jpeg_decode_coefs_batch(b200jpeg_encoder *enc, const uint8_t *const *files, const size_t *sizes, int n_images,
                                 int16_t *const *planes, int planes_on_device, const size_t *row_pitch_blocks,
                                 const size_t *image_stride_blocks);
/* jpegtran from file bytes: the decode above feeding b200jpeg_encode_batch_coefs_qtables with `p` (what
 * jpeg_copy_critical_parameters and the switches leave, e.g. from the Python params_for_transcode) and, per image, the
 * quantization tables the file's components latched.  The finished files are read with b200jpeg_get_output. */
int  b200jpeg_transcode_batch(b200jpeg_encoder *enc, const b200jpeg_params *p, const uint8_t *const *files,
                              const size_t *sizes, int n_images);
/* The two routes above with a lossless transform applied while the coefficients are imported: `p` and `t` as
 * b200jpeg_transform_setup left them.  b200jpeg_transcode_batch_transform decodes the files on the device (sequential
 * sources only) and transposes each image's latched tables for transposing transforms.
 * b200jpeg_encode_batch_coefs_transform takes planes in the SOURCE geometry (t->src_wib / t->src_hib blocks per
 * component), e.g. any decoder's jpeg_read_coefficients output for progressive sources; qtables (or NULL for p's) are
 * the sources' tables, [n_images][4][64] natural order, transposed here like p's were. */
int  b200jpeg_transcode_batch_transform(b200jpeg_encoder *enc, const b200jpeg_params *p, const b200jpeg_transform_info *t,
                                        const uint8_t *const *files, const size_t *sizes, int n_images);
int  b200jpeg_encode_batch_coefs_transform(b200jpeg_encoder *enc, const b200jpeg_params *p, const b200jpeg_transform_info *t,
                                           const int16_t *const *planes, int planes_on_device,
                                           const size_t *row_pitch_blocks, const size_t *image_stride_blocks,
                                           const uint16_t *qtables, int n_images);
/* Synchronisation work of the last decode: the most rounds a CTA of the speculative decoder needed and the number of
 * subsequences the cross-CTA pass decoded again. */
int  b200jpeg_last_decode_sync(const b200jpeg_encoder *enc, int *max_cta_rounds, long long *resync_subsequences);

/*
 * Decompression to pixels on the device: replaces jpeg_read_header + jpeg_start_decompress + jpeg_read_scanlines of a
 * decompress object left at its defaults (JDCT_ISLOW, fancy upsampling, no scaling or colour quantization,
 * out_color_space as default_decompress_parms picks it: gray -> gray, YCbCr -> RGB, RGB -> RGB), sample for sample, for
 * a batch of sequential files of one geometry and colour space.  It is what the reference's cjpeg does with a JPEG
 * input file (rdjpeg.c).  The entropy decode is b200jpeg_decode_coefs_batch's, with its error reporting; dequantization
 * uses each file's own latched tables.
 *
 * Accepted: SOF0 / SOF1, 8 bits, one component, or three with component 0 at the largest sampling factors (1 or 2 each
 * way) over 1x1 chroma (4:4:4, 4:2:2, 4:4:0, 4:2:0).  12-bit, 4-component, progressive files and every other sampling
 * layout are B200JPEG_ERR_UNSUPPORTED naming the first such image, before any device work.
 *
 * b200jpeg_decompress_batch writes image i's rows (image_width * components bytes, see b200jpeg_decompress_output) to
 * pixels + i * image_stride, row_pitch bytes apart, in host or device memory (pixels_on_device).  The batch is
 * processed in chunks (b200jpeg_encoder_set_chunk_images): coefficient and sample planes are one chunk's.
 */
int  b200jpeg_decompress_batch(b200jpeg_encoder *enc, const uint8_t *const *files, const size_t *sizes, int n_images,
                               void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride);
/* cjpeg with JPEG input files: the decode above into device memory, then b200jpeg_encode_batch on the pixels where they
 * lie, so every encoder option applies.  p is the compress parameter block: image size, in_color_space,
 * input_components (and data_precision 8) must be what the sources decode to (b200jpeg_decompress_output), else
 * B200JPEG_ERR_PARAM.  Like cjpeg (cjpeg.c:960-990) each file receives, behind its JFIF / Adobe header, the COM and
 * APPn segments of its source in file order, except a JFIF APP0 when p->write_JFIF_header and an Adobe APP14 when
 * p->write_Adobe_marker.  The finished files are read with b200jpeg_get_output. */
int  b200jpeg_recompress_batch(b200jpeg_encoder *enc, const b200jpeg_params *p, const uint8_t *const *files,
                               const size_t *sizes, int n_images);
/* What rdjpeg.c's start_input_jpeg copies from the decompress object into the compress object: image size,
 * out_color_space (B200JPEG_CS_GRAYSCALE, _RGB, or _CMYK for 4-component files) and output_components. */
int  b200jpeg_decompress_output(const b200jpeg_source_info *src, int *width, int *height, int *color_space, int *components);

/*
 * Decompression with the decompress object's options (djpeg -scale, -dct, -nosmooth, -fast, -grayscale, -rgb and the
 * EXT_* output orders), sample for sample, on the sources b200jpeg_decompress_batch accepts (same checks, same
 * messages).
 *   scale_num / scale_denom: as jpeg_core_output_dimensions buckets them into a block size k (1/5 is k = 2); k must be
 *     1, 2, 4 or 8 (1/8, 1/4, 1/2, 1/1), other k are B200JPEG_ERR_UNSUPPORTED.  Output: ceil(W k / 8) x ceil(H k / 8).
 *   dct_method: B200JPEG_DCT_*, for components whose DCT_scaled_size is 8 (jddctmgr.c); smaller sizes use
 *     jidctred.c's IDCTs whatever the method.
 *   do_fancy_upsampling: 0 replicates chroma (and the merged upsampler, which gives the same pixels).
 *   out_color_space: -1 for what default_decompress_parms picks; else GRAYSCALE, RGB, EXT_*, or YCbCr from a YCbCr
 *     file.  Pairs the reference refuses are B200JPEG_ERR_PARAM "Unsupported color conversion request"; CMYK, YCCK
 *     and B200JPEG_CS_RGB565 output are B200JPEG_ERR_UNSUPPORTED.
 * The default options give b200jpeg_decompress_batch's and b200jpeg_recompress_batch's route and bytes.
 */
#define B200JPEG_CS_RGB565 16
typedef struct { int scale_num, scale_denom, dct_method, do_fancy_upsampling, out_color_space; } b200jpeg_decompress_options;
b200jpeg_decompress_options b200jpeg_default_decompress_options(void);
/* jpeg_calc_output_dimensions + out_color_components for these options: B200JPEG_ERR_* as the batch would refuse. */
int  b200jpeg_decompress_output_opts(const b200jpeg_source_info *src, const b200jpeg_decompress_options *opts,
                                     int *width, int *height, int *color_space, int *components);
int  b200jpeg_decompress_batch_opts(b200jpeg_encoder *enc, const b200jpeg_decompress_options *opts, const uint8_t *const *files,
                                    const size_t *sizes, int n_images, void *pixels, int pixels_on_device, size_t row_pitch,
                                    size_t image_stride);
/* b200jpeg_recompress_batch from the decode with opts: p must describe the decoded (scaled) pixels. */
int  b200jpeg_recompress_batch_opts(b200jpeg_encoder *enc, const b200jpeg_decompress_options *opts, const b200jpeg_params *p,
                                    const uint8_t *const *files, const size_t *sizes, int n_images);

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
