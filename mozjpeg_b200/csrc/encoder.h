// encoder.h -- the encoder object and the device / pinned buffers it owns, shared by the encode pipeline (encoder.cu)
// and the decompressor (decompress.cu), and the few functions one calls in the other (not installed).
#pragma once
#include "b200jpeg.h"
#include "internal.h"
#include "kernels.cuh"
#include <utility>
#include <vector>

namespace b200 {

#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); return B200JPEG_ERR_CUDA; } } while (0)

// a device (DevBuf) or pinned host (PinBuf) allocation that reserve() grows; freed by its destructor, so move-only
struct DevBuf {
  void *p = nullptr; size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  DevBuf &operator=(DevBuf &&o) noexcept { if (this != &o) { release(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); } return *this; }
  ~DevBuf() { release(); }
  int reserve(size_t n) {
    if (n <= cap) return B200JPEG_OK;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) { p = nullptr; set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e)); return B200JPEG_ERR_CUDA; }
    cap = want; return B200JPEG_OK;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <class T> T *as() { return static_cast<T *>(p); }
};
struct PinBuf {
  void *p = nullptr; size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf &) = delete;
  PinBuf &operator=(const PinBuf &) = delete;
  PinBuf(PinBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  PinBuf &operator=(PinBuf &&o) noexcept { if (this != &o) { release(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); } return *this; }
  ~PinBuf() { release(); }
  int reserve(size_t n) {
    if (n <= cap) return B200JPEG_OK;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 256;
    cudaError_t e = cudaMallocHost(&p, want);
    if (e != cudaSuccess) { p = nullptr; set_error("cudaMallocHost(%zu) failed: %s", want, cudaGetErrorString(e)); return B200JPEG_ERR_CUDA; }
    cap = want; return B200JPEG_OK;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
  template <class T> T *as() { return static_cast<T *>(p); }
};

struct Plan {                // everything derived from b200jpeg_params
  Geom g;
  std::vector<ScanDesc> scans;
  bool progressive = false, optimize = false, trellis = false, dering = false, restarts = false;
  bool lossless = false;         // SOF3: every scan is predicted and coded sample by sample (run_lossless)
  int smooth = 0;                // smoothing_factor: colour conversion + (smoothing) downsampling run as a pre-pass into planes
  // scan search (optimize_scans): the script of jpeg_search_progression (jcparam.c:733-852) and where its groups start
  bool search = false; int n_luma = 0, luma_split0 = 0, chroma_split0 = 0, chroma_al0 = 0;
  std::vector<int> order;        // scan ids in the order they are encoded; position in `order` = slot in out_pos
  RestartSpec rs = {0, 0};
  size_t coef_bytes[4] = {0, 0, 0, 0};
  long long max_scan_blocks = 0, max_real_blocks = 0, sum_real_blocks = 0;
};

}  // namespace b200

using namespace b200;

// intermediate HBM state of one chunk in flight
#define MAX_ARENAS 4
struct Arena {
  b200::DevBuf d_planes;             // input smoothing: the pre-pass's component planes
  b200::DevBuf d_coef[4], d_raw[4], d_plain[4], d_hist, d_tabs_trellis, d_rec, d_big, d_bigcnt, d_best_al, d_qimg, d_qsum, d_eo, d_es;
  b200::DevBuf d_slot, d_blk_aux, d_blk_run, d_blk_mask;
  b200::DevBuf d_stream;             // the scans' coded stream (ScanStream, kernels.cuh)
  b200::DevBuf d_sym, d_dcq;         // sequential scans after the trellis: symbol records + dense DC values (SymOut, kernels.cuh)
  b200::DevBuf d_diff;               // lossless scans: the differences of the scan being coded (launch_lossless_diff)
  b200::Geom g;                      // the plan's geometry with this arena's coefficient pointers
  b200::ScanStream ss;               // the buffers inside d_stream (status: the chunk's)
};

struct b200jpeg_encoder {
  int device = 0;
  int sms = 0;                       // SM count of `device`, read once at creation (sizes the AC trellis grid)
  cudaStream_t stream = nullptr;     // compute stream (caller-replaceable)
  cudaStream_t s_in = nullptr;       // host->device staging of the pixels
  cudaStream_t s_out = nullptr;      // device->host read-back of the entropy-coded bytes
  b200jpeg_params params;           // of the last batch
  Plan plan;
  int n = 0;                        // images of the last batch
  int chunk = 0;                    // images per chunk of the last batch
  int last_chunk_i0 = 0, last_chunk_n = 0, last_chunk_slot = 0;   // the chunk whose intermediates are still in the arenas
  int chunk_images_override = 0;    // 0 = automatic
  bool progressive_decode = false;  // decode SOF2 files too (b200jpeg_encoder_set_progressive_decode)
  bool keep_plain = false;
  // device arenas sized for ONE chunk; two of them so that consecutive chunks can run on two
  // streams and fill each other's latency-bound phases (serial table construction, trellis chains)
  Arena ar[MAX_ARENAS];
  cudaStream_t sc[MAX_ARENAS] = {nullptr, nullptr, nullptr, nullptr};   // sc[0] aliases `stream`
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  int n_streams = 2;
  // device buffers sized for the WHOLE batch
  DevBuf d_src, d_tabs_scan, d_tabs_fixed, d_status, d_out_pos, d_scan_size, d_out, d_qt, d_tc, d_best_al_all, d_qimg_all, d_qset;
  // quantization table sets of the last batch: the distinct [4][64] tables (natural order) its images use, and each
  // image's set; one set (the parameter block's) and no per-image index unless the caller passed per-image tables
  std::vector<uint16_t> qsets; std::vector<int> img_set; int nsets = 1;
  size_t bitbuf_words_per_image = 0, out_cap_per_image = 0;
  double cap_factor = 0.25;      // entropy-coded bytes the buffers hold per coefficient; grows on overflow, falls back after calm batches
  int calm_batches = 0;
  size_t max_image_scan_bytes = 0;   // largest entropy-coded size of one image in the last host-visible batch
  // pinned host mirrors
  PinBuf h_qt, h_tc, h_fixed, h_status, h_out_pos, h_scan_size, h_tabs, h_stage, h_best_al, h_qinit, h_qimg, h_qset;
  // finished files: bump-allocated from pinned arenas, valid until the next encode call
  std::vector<PinBuf> file_arenas; size_t arena_idx = 0, arena_off = 0;
  std::vector<std::pair<uint8_t *, size_t>> files;
  size_t last_file_bytes = 0;
  size_t last_scan_bytes = 0;
  unsigned long long launches_at_create = 0;
  // timing
  std::vector<cudaEvent_t> ev; std::vector<const char *> ev_names, stage_names; std::vector<float> stage_ms; std::vector<int> stage_calls;
  size_t pending_marks = 0;                     // device-resident YUV batch: timer events not yet summed into stage_ms
  DevBuf d_yuv;                                 // YUV planes bound for host memory, staged per chunk
  std::vector<cudaEvent_t> ev_in, ev_done;      // per chunk: pixels staged / pipeline + metadata read-back queued
  bool own_stream = true;
  // streaming shim state
  int st_state = 0, st_next_row = 0;
  b200jpeg_params st_params;
  // device entropy decode (b200jpeg_decode_coefs_batch / b200jpeg_transcode_batch): descriptors of the last batch, the
  // upload buffer of its unstuffed segments, and the decoded planes (per component, each image's [hib][wib][64] blocks
  // in turn, natural order)
  b200::DecBatch dec;
  PinBuf h_dec_words, h_dec_stat;
  DevBuf d_dec_words, d_dec_segs, d_dec_scans, d_dec_tabs, d_dec_out, d_dec_rec, d_dec_pre, d_dec_tsum, d_dec_dcd, d_dec_planes, d_dec_stat;
  size_t dec_plane_off[4] = {0, 0, 0, 0};
  cudaEvent_t dec_ev[9] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // [7], [8]: refinements
  int dec_rounds = 0; long long dec_redone = 0;
  bool dec_prog = false;            // the last decode had a progressive file: its stage times include the refinements
  bool dec_ms_prog = false;         // some chunk of the last decompress had one: dec_ms holds refinement times
  // decompression to pixels (b200jpeg_decompress_batch / b200jpeg_recompress_batch): one chunk's sample planes and
  // quantization tables, the whole batch's pixels where the caller gave no device buffer, the stage times summed over
  // the chunks, and per image the source's COM / APPn segments a recompress copies into its file
  DevBuf d_dec_samples, d_dec_quant, d_dec_pixels, d_dec_mtab;   // d_dec_mtab: ifast / float multiplier tables
  std::vector<cudaEvent_t> pix_ev;   // per pixel output of a chunk: before the IDCT, before the upsampling, after it
  float dec_ms[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // the six decode stages, idct, upsample_color, the two refinements
  std::vector<std::vector<uint8_t>> dec_markers;
  const std::vector<std::vector<uint8_t>> *copy_markers = nullptr;   // of the batch being encoded, or nullptr
  // renditions (b200jpeg_decompress_renditions / b200jpeg_recompress_renditions): the whole batch's pixels of each
  // distinct option set, and the files of every rung but the last (the next rung's encode reuses the file arenas)
  std::vector<DevBuf> d_rend_pixels;
  std::vector<uint8_t> rend_files;
  // batches of mixed geometry (b200jpeg_decompress_mixed / b200jpeg_recompress_mixed): one chunk's pixel-stage
  // descriptors and work tables (IdctImg, UpsImg)
  DevBuf d_mix_meta;
  CoefXform xform{};                            // the coefficient import's block mapping in the current batch (all zero: a copy)
};

// One chunk of a batch: images [i0, i0+n) and where their results go.
struct ChunkIO {
  int i0, n;
  int slot;                         // which arena / stream
  const uint8_t *src;               // first pixel of image i0 (device)
  const uint8_t *plane[4];          // raw-data input: image i0's component planes (device)
  uint8_t *out;                     // [n][out_cap_per_image]
  unsigned long long *out_pos;      // [nscans+1][n]: start of every scan's bytes inside out[img]; row nscans = total
  uint32_t *status;                 // [n]
  uint32_t *scan_size;              // [nscans][n]
  b200::DevHuff *tabs_scan;         // [n][nscans][8]
  int *best_al;                     // [2][n] scan search: best luma / chroma Al per image
  uint16_t *qimg;                   // [n][4][64] trellis_q_opt: the re-fitted quantization tables per image (natural order)
  const int *qset;                  // [n] each image's quantization table set (device), or nullptr: set 0
};

namespace b200 {

// defined in encoder.cu; the decompressor's recompress and transcode routes call them too
int div_up(long long a, long long b);
struct RawDesc;
int encode_common(b200jpeg_encoder *e, const b200jpeg_params *p, const void *pixels, int on_device,
                  size_t row_pitch, size_t image_stride, int n_images, bool device_only, const RawDesc *raw,
                  const uint16_t *qtables, const std::vector<std::vector<uint8_t>> *markers);
void transpose_qsets(uint16_t *q, int n);
int encode_coefs_xform(b200jpeg_encoder *enc, const b200jpeg_params *p, const b200jpeg_transform_info *t, const int16_t *const *planes, int planes_on_device,
                       const size_t *row_pitch_blocks, const size_t *image_stride_blocks, const uint16_t *qtables, int n_images);

}  // namespace b200
