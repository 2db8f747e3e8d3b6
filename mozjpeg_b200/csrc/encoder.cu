// encoder.cu -- host side of libb200jpeg: HBM arenas, the pass plan of
// jcmaster.c restated as batch-wide kernel launches, and the C-ABI entry points
// of include/b200jpeg.h.  One encoder = one CUDA device + one stream; every
// launch covers the whole batch, so the reference's per-image "passes"
// (jcmaster.c:612-715) become one launch per phase for all images.
#include "b200jpeg.h"
#include "internal.h"
#include "kernels.cuh"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace b200 {

#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); return B200JPEG_ERR_CUDA; } } while (0)

static const int kZigzag[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct DevBuf {
  void *p = nullptr; size_t cap = 0;
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

// host copy of a DHT payload (first 288 bytes of DevHuff)
struct HostHuff { uint8_t bits[17]; uint8_t huffval[256]; uint8_t nsym; uint8_t pad[12]; uint16_t nsym16; };
static_assert(sizeof(HostHuff) == 288, "HostHuff");

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
  b200::DevBuf d_coef[4], d_raw[4], d_plain[4], d_hist, d_tabs_trellis, d_rec, d_srec, d_splits, d_best_al, d_qimg, d_qsum, d_eo, d_es;
  b200::DevBuf d_blk_bits, d_tile_bits, d_tile_base, d_seg_corr, d_mark, d_stuff_lb, d_blk_aux, d_blk_run, d_blk_mask, d_total_bits, d_bitbuf;
  b200::DevBuf d_sym, d_dcq;         // sequential scans after the trellis: symbol records + dense DC values (SymOut, kernels.cuh)
  b200::DevBuf d_diff;               // lossless scans: the differences of the scan being coded (launch_lossless_diff)
  b200::Geom g;                      // the plan's geometry with this arena's coefficient pointers
  void release() {
    b200::DevBuf *db[] = {&d_planes, &d_hist, &d_tabs_trellis, &d_rec, &d_srec, &d_splits, &d_best_al, &d_qimg, &d_qsum, &d_eo, &d_es, &d_blk_bits, &d_tile_bits, &d_tile_base, &d_seg_corr, &d_mark, &d_stuff_lb, &d_blk_aux, &d_blk_run, &d_blk_mask, &d_total_bits, &d_bitbuf, &d_sym, &d_dcq, &d_diff};
    for (b200::DevBuf *b : db) b->release();
    for (int i = 0; i < 4; i++) { d_coef[i].release(); d_raw[i].release(); d_plain[i].release(); }
  }
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
  // upload buffer of its unstuffed segments, and the decoded planes ([n][hib][wib][64] per component, natural order)
  b200::DecBatch dec;
  PinBuf h_dec_words, h_dec_stat;
  DevBuf d_dec_words, d_dec_segs, d_dec_scans, d_dec_tabs, d_dec_out, d_dec_rec, d_dec_pre, d_dec_tsum, d_dec_dcd, d_dec_planes, d_dec_stat;
  size_t dec_plane_off[4] = {0, 0, 0, 0};
  cudaEvent_t dec_ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  int dec_rounds = 0; long long dec_redone = 0;
  // decompression to pixels (b200jpeg_decompress_batch / b200jpeg_recompress_batch): one chunk's sample planes and
  // quantization tables, the whole batch's pixels where the caller gave no device buffer, the stage times summed over
  // the chunks, and per image the source's COM / APPn segments a recompress copies into its file
  DevBuf d_dec_samples, d_dec_quant, d_dec_pixels, d_dec_mtab;   // d_dec_mtab: ifast / float multiplier tables
  cudaEvent_t pix_ev[3] = {nullptr, nullptr, nullptr};
  float dec_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  std::vector<std::vector<uint8_t>> dec_markers;
  const std::vector<std::vector<uint8_t>> *copy_markers = nullptr;   // of the batch being encoded, or nullptr
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

static int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Lossless mode (p after the start-time overrides, lossless_start): one data unit = one sample, every component 1x1,
// so a scan is W*H MCUs of one sample per scan component (per_scan_setup, jcmaster.c:518-601 with data_unit 1).
static void build_plan_lossless(const b200jpeg_params *p, Plan &pl)
{
  Geom &g = pl.g;
  g.mcus_per_row = g.W; g.mcu_rows = g.H;
  pl.max_real_blocks = pl.sum_real_blocks = 0;
  for (int ci = 0; ci < g.nc; ci++) {
    CompGeom &c = g.c[ci]; const b200jpeg_component_info &ic = p->comp_info[ci];
    c.h = c.v = c.hx = c.vx = 1;
    c.wib = c.wpad = g.W; c.hib = c.hpad = g.H; c.rows_avail = g.H;
    c.qt = ic.quant_tbl_no; c.dc_tbl = ic.dc_tbl_no; c.ac_tbl = ic.ac_tbl_no;
    c.blocks_per_image = (long long)g.W * g.H;
    pl.coef_bytes[ci] = 0;
  }
  pl.scans.clear();
  pl.max_scan_blocks = (long long)g.W * g.H;
  for (int si = 0; si < p->num_scans; si++) {
    const b200jpeg_scan_info &s = p->scan_info[si];
    ScanDesc sd; memset(&sd, 0, sizeof sd);
    sd.ncomps = s.comps_in_scan; for (int k = 0; k < 4; k++) sd.ci[k] = s.component_index[k];
    sd.Ss = s.Ss; sd.Se = s.Se; sd.Ah = s.Ah; sd.Al = s.Al;
    sd.bim = 1; sd.per_row = g.W; sd.rows = g.H; sd.nblocks = (long long)g.W * g.H;
    sd.ri = p->restart_in_rows > 0 ? (int)std::min((long long)p->restart_in_rows * g.W, 65535LL) : p->restart_interval;
    pl.scans.push_back(sd);
  }
  pl.lossless = true; pl.progressive = false; pl.optimize = true; pl.trellis = false; pl.dering = false; pl.smooth = 0; pl.search = false;
  pl.restarts = p->restart_interval != 0 || p->restart_in_rows > 0;
  pl.rs.interval = p->restart_interval; pl.rs.in_rows = p->restart_in_rows;
  pl.order.clear();
  for (int si = 0; si < p->num_scans; si++) pl.order.push_back(si);
}

static int build_plan(const b200jpeg_params *p, size_t row_pitch, size_t image_stride, Plan &pl)
{
  Geom &g = pl.g;
  memset(&g, 0, sizeof g);
  g.W = p->image_width; g.H = p->image_height; g.nc = p->num_components; g.in_comps = p->input_components;
  g.hmax = g.vmax = 1;
  for (int ci = 0; ci < g.nc; ci++) { g.hmax = std::max(g.hmax, p->comp_info[ci].h_samp_factor); g.vmax = std::max(g.vmax, p->comp_info[ci].v_samp_factor); }
  g.mcus_per_row = div_up(g.W, g.hmax * 8); g.mcu_rows = div_up(g.H, g.vmax * 8);
  g.row_pitch = row_pitch; g.image_stride = image_stride;
  g.max_coef_bits = p->data_precision + 2;
  const bool rgb_in = B200JPEG_CS_IS_RGB(p->in_color_space);
  if (rgb_in && p->jpeg_color_space == B200JPEG_CS_YCbCr) g.cs_mode = 0;
  else if (rgb_in && p->jpeg_color_space == B200JPEG_CS_GRAYSCALE) g.cs_mode = 1;
  else if (p->in_color_space == B200JPEG_CS_CMYK && p->jpeg_color_space == B200JPEG_CS_YCCK) g.cs_mode = 3;
  else g.cs_mode = 2;                               // RGB->RGB, gray, YCbCr->YCbCr/gray, CMYK, YCCK, UNKNOWN: null_convert
  g.px_first = rgb_in ? B200JPEG_CS_FIRST(p->in_color_space) : 0;             // jccolor.c:253-291 (JCS_EXT_* pixel orders)
  g.px_swap = rgb_in ? B200JPEG_CS_BLUE_FIRST(p->in_color_space) : 0;
  pl.lossless = false;
  if (is_lossless(p)) { build_plan_lossless(p, pl); return B200JPEG_OK; }
  pl.max_real_blocks = 0; pl.sum_real_blocks = 0;
  for (int ci = 0; ci < g.nc; ci++) {
    CompGeom &c = g.c[ci]; const b200jpeg_component_info &ic = p->comp_info[ci];
    c.h = ic.h_samp_factor; c.v = ic.v_samp_factor; c.hx = g.hmax / c.h; c.vx = g.vmax / c.v;
    c.wib = div_up((long long)g.W * c.h, g.hmax * 8); c.hib = div_up((long long)g.H * c.v, g.vmax * 8);   // jcmaster.c:221-226
    c.wpad = g.mcus_per_row * c.h; c.hpad = g.mcu_rows * c.v;
    c.qt = ic.quant_tbl_no; c.dc_tbl = ic.dc_tbl_no; c.ac_tbl = ic.ac_tbl_no;
    c.rows_avail = div_up(g.H, g.vmax) * c.v;
    c.blocks_per_image = (long long)c.wpad * c.hpad;
    pl.coef_bytes[ci] = (size_t)c.blocks_per_image * 128;
    pl.max_real_blocks = std::max(pl.max_real_blocks, (long long)c.wib * c.hib); pl.sum_real_blocks += (long long)c.wib * c.hib;
  }
  // scan list (select_scan_parameters jcmaster.c:443-515 + per_scan_setup :518-601)
  pl.scans.clear();
  int nscans = p->num_scans > 0 ? p->num_scans : 1;
  pl.max_scan_blocks = 0;
  for (int si = 0; si < nscans; si++) {
    ScanDesc sd; memset(&sd, 0, sizeof sd);
    if (p->num_scans > 0) {
      const b200jpeg_scan_info &s = p->scan_info[si];
      sd.ncomps = s.comps_in_scan; for (int k = 0; k < 4; k++) sd.ci[k] = s.component_index[k];
      sd.Ss = s.Ss; sd.Se = s.Se; sd.Ah = s.Ah; sd.Al = s.Al;
    } else { sd.ncomps = g.nc; for (int k = 0; k < 4; k++) sd.ci[k] = k; sd.Ss = 0; sd.Se = 63; }
    if (sd.ncomps == 1) {
      const CompGeom &c = g.c[sd.ci[0]];
      sd.bim = 1; sd.k_comp[0] = 0; sd.k_first[0] = 0; sd.k_count[0] = 1;
      sd.per_row = c.wib; sd.rows = c.hib;
    } else {
      int k = 0;
      for (int i = 0; i < sd.ncomps; i++) {
        const CompGeom &c = g.c[sd.ci[i]];
        sd.k_first[i] = k; sd.k_count[i] = c.h * c.v;
        for (int y = 0; y < c.v; y++) for (int x = 0; x < c.h; x++) { sd.k_comp[k] = i; sd.k_y[k] = y; sd.k_x[k] = x; k++; }
      }
      sd.bim = k; sd.per_row = g.mcus_per_row; sd.rows = g.mcu_rows;
    }
    sd.nblocks = (long long)sd.per_row * sd.rows * sd.bim;
    sd.ri = p->restart_in_rows > 0 ? (int)std::min((long long)p->restart_in_rows * sd.per_row, 65535LL) : p->restart_interval;   // jcmaster.c:594-599
    pl.max_scan_blocks = std::max(pl.max_scan_blocks, sd.nblocks);
    pl.scans.push_back(sd);
  }
  pl.progressive = p->num_scans > 0 && (p->scan_info[0].Ss != 0 || p->scan_info[0].Se != 63);
  pl.optimize = p->optimize_coding || pl.progressive || p->data_precision == 12;   // jcmaster.c:1091-1094, :1102-1105
  pl.trellis = p->trellis_quant != 0;
  pl.dering = p->overshoot_deringing != 0;
  pl.smooth = p->smoothing_factor;
  pl.search = p->optimize_scans && p->num_scans > 0;
  pl.restarts = p->restart_interval != 0 || p->restart_in_rows > 0;       // before the search guard below reads it
  pl.rs.interval = p->restart_interval; pl.rs.in_rows = p->restart_in_rows;
  if (pl.search) {
    // every candidate is buffered with its own scan header; a DRI marker opens it when its restart interval differs from
    // the previously coded scan's (write_scan_header).  Scans that the search may skip share their neighbours' interval
    // as long as Cb and Cr have the same geometry, so the flags do not depend on the search's course.
    int last = 0;
    for (size_t k = 0; k < pl.scans.size(); k++) { pl.scans[k].dri = pl.scans[k].ri != last; last = pl.scans[k].ri; }
    if (pl.restarts && g.nc == 3 && (g.c[1].wib != g.c[2].wib || g.c[1].hib != g.c[2].hib)) { set_error("scan search with restart intervals needs equal Cb/Cr geometry"); return B200JPEG_ERR_UNSUPPORTED; }
  }
  pl.order.clear();
  if (pl.search) {
    // jpeg_search_progression constants: num_scans_luma_dc 1, Al_max_luma 3, 5 frequency splits; chroma: 3 DC scans, Al_max 2
    pl.n_luma = 1 + (3 * 3 + 2) + (2 * 5 + 1);                  // 23
    pl.luma_split0 = 1 + 3 * 3 + 2;                             // 12: first luma frequency-split scan (coded at the best luma Al)
    pl.chroma_al0 = pl.n_luma + 3;                              // 26: first chroma Al-search scan
    pl.chroma_split0 = pl.n_luma + 3 + (6 * 2 + 4);             // 42
    const bool colour = nscans > pl.n_luma;
    if (nscans != (colour ? 64 : 23)) { set_error("optimize_scans needs the script of jpeg_search_progression (%d scans given)", nscans); return B200JPEG_ERR_PARAM; }
    // phase A: every scan whose parameters are fixed; phase B: the frequency-split scans, coded at the image's best Al
    for (int si = 0; si < pl.luma_split0; si++) pl.order.push_back(si);
    if (colour) for (int si = pl.n_luma; si < pl.chroma_split0; si++) pl.order.push_back(si);
    for (int si = pl.luma_split0; si < pl.n_luma; si++) pl.order.push_back(si);
    if (colour) for (int si = pl.chroma_split0; si < nscans; si++) pl.order.push_back(si);
  } else for (int si = 0; si < nscans; si++) pl.order.push_back(si);
  return B200JPEG_OK;
}

// exact floor((|x| + d/2) / d) for |x| + d/2 < 2^18 by multiply-shift:
// k = 18 + ceil(log2 d), m = ceil(2^k / d)  (Granlund-Montgomery round-up method)
static void make_quant_consts(const b200jpeg_params *p, QuantTables *qt)
{
  memset(qt, 0, sizeof *qt);
  for (int t = 0; t < 4; t++) {
    if (!p->quant_tbl_present[t]) continue;
    for (int i = 0; i < 64; i++) {
      unsigned d = 8u * p->quant_tbl[t][i];
      int l = 0; while ((1ull << l) < d) l++;
      int k = 18 + l;
      unsigned long long m = ((1ull << k) + d - 1) / d;
      QuantConst &q = qt->q[t][i];
      q.mul = (uint32_t)m; q.shift = (uint16_t)k; q.bias = d / 2; q.d = d; q.pad = 0;
    }
    // one shift for the whole table: L >= log2 of every divisor, mul2 = ceil(2^(18+L)/d) must fit 32 bits
    unsigned dmax = 1, dmin = ~0u;
    for (int i = 0; i < 64; i++) { unsigned d = 8u * p->quant_tbl[t][i]; dmax = std::max(dmax, d); dmin = std::min(dmin, d); }
    int L = 0; while ((1ull << L) < dmax) L++;
    qt->L[t] = L;
    qt->fast[t] = (((1ull << (18 + L)) + dmin - 1) / dmin) < (1ull << 32) ? 1 : 0;
    for (int i = 0; i < 64; i++) { unsigned d = qt->q[t][i].d; qt->q[t][i].mul2 = qt->fast[t] ? (uint32_t)(((1ull << (18 + L)) + d - 1) / d) : 0; }
    for (int i = 0; i < 64; i++) qt->qpack[t][i] = make_uint2(qt->q[t][i].mul2, qt->q[t][i].bias << 14);
    static const short aanscales[64] = {16384, 22725, 21407, 19266, 16384, 12873, 8867, 4520, 22725, 31521, 29692, 26722, 22725, 17855, 12299, 6270,
      21407, 29692, 27969, 25172, 21407, 16819, 11585, 5906, 19266, 26722, 25172, 22654, 19266, 15137, 10426, 5315,
      16384, 22725, 21407, 19266, 16384, 12873, 8867, 4520, 12873, 17855, 16819, 15137, 12873, 10114, 6967, 3552,
      8867, 12299, 11585, 10426, 8867, 6967, 4799, 2446, 4520, 6270, 5906, 5315, 4520, 3552, 2446, 1247};
    for (int i = 0; i < 64; i++) {                                 // jcdctmgr.c:290-339 + compute_reciprocal :181-230
      unsigned divisor = (unsigned)(unsigned short)(((long)p->quant_tbl[t][i] * aanscales[i] + (1L << 10)) >> 11);
      IfastConst &k = qt->ifast[t][i]; k.pad = 0;
      if (divisor == 1) { k.recip = 1; k.corr = 0; k.shift = -32; continue; }
      // the 16-bit divisor wraps to 0 for 14 table values (16384 at the 16384-scaled positions, ...); only the fast DCT
      // reads these constants, and the reference cannot quantize such a table with it either (compute_reciprocal
      // divides by the wrapped value), so leave them zero instead of dividing by zero for every DCT method
      if (divisor == 0) { k.recip = 0; k.corr = 0; k.shift = 0; continue; }
      int b = 0; for (unsigned v = divisor; v; v >>= 1) b++; b -= 1;
      int r = 32 + b;
      unsigned long long fq = (1ULL << r) / divisor, fr = (1ULL << r) % divisor; unsigned c = divisor / 2;
      if (fr == 0) { fq >>= 1; r--; } else if (fr <= (divisor / 2U)) c++; else fq++;
      k.recip = (unsigned)fq; k.corr = c; k.shift = r - 32;
    }
    static const double aan[8] = {1.0, 1.387039845, 1.306562965, 1.175875602, 1.0, 0.785694958, 0.541196100, 0.275899379};
    for (int i = 0; i < 64; i++) qt->fdiv[t][i] = (float)(1.0 / (((double)p->quant_tbl[t][i] * aan[i / 8] * aan[i % 8] * 8.0)));       // jcdctmgr.c:371-374
  }
}
static void make_trellis_consts(const b200jpeg_params *p, TrellisConsts *tc)
{
  memset(tc, 0, sizeof *tc);
  for (int t = 0; t < 4; t++) {
    if (!p->quant_tbl_present[t]) continue;
    for (int k = 0; k < 64; k++) {
      int q = p->quant_tbl[t][kZigzag[k]];
      tc->w_zz[t][k] = (float)(1.0 / (q * q));                       // jcdctmgr.c:1020 (double divide, float store)
      tc->q8_zz[t][k] = 8 * q;

    }
  }
  for (int t = 0; t < 4; t++) {
    if (!p->quant_tbl_present[t]) continue;
    unsigned dmax = 1; for (int k = 0; k < 64; k++) dmax = std::max(dmax, 8u * p->quant_tbl[t][k]);
    int L = 0; while ((1ull << L) < dmax) L++;
    tc->qL[t] = L;
    for (int k = 0; k < 64; k++) { unsigned d = 8u * p->quant_tbl[t][kZigzag[k]]; tc->qmul_zz[t][k] = (unsigned)std::min<unsigned long long>(((1ull << (18 + L)) + d - 1) / d, 0xFFFFFFFFull); }
    // the DC trellis' divider; its fast form needs 9 candidates (get_num_dc_trellis_candidates, jcdctmgr.c:929-933) and
    // no candidate that can reach the coefficient limit
    const unsigned d = 8u * p->quant_tbl[t][0];
    int l = 0; while ((1ull << l) < d) l++;
    tc->dc_shift[t] = 18 + l;
    tc->dc_mul[t] = (unsigned)(((1ull << tc->dc_shift[t]) + d - 1) / d);
    int ncand = (2 + 60 / (int)(d >> 3)) | 1; if (ncand > 9) ncand = 9;
    tc->dc_fast[t] = ncand == 9 && (int)((32768 + d / 2) / d) + 9 < (1 << (p->data_precision + 2)) - 1;
  }
  tc->use_norm = p->lambda_log_scale2 > 0.0f;
  tc->delta_dc_weight = p->trellis_delta_dc_weight;
  tc->p1 = pow(2.0, (double)p->lambda_log_scale1);
  tc->p2 = pow(2.0, (double)p->lambda_log_scale2);
  tc->lambda_const = (float)(pow(2.0, (double)p->lambda_log_scale1 - 12.0) * 1.0f);
  tc->max_coef_bits = p->data_precision + 2;
  tc->dc_trellis = p->trellis_quant_dc;
}
// jpeg_make_c_derived_tbl (jchuff.c:231-318) for caller-supplied tables
static int make_fixed_table(const b200jpeg_huff_tbl &t, bool is_dc, DevHuff *out)
{
  memset(out, 0, sizeof *out);
  if (!t.present) return 0;
  memcpy(out->bits, t.bits, 17); memcpy(out->huffval, t.huffval, 256);
  int n = 0; unsigned code = 0;
  for (int l = 1; l <= 16; l++) {
    for (int c = 0; c < t.bits[l]; c++) {
      if (n >= 256) return -1;
      int sym = t.huffval[n++];
      if ((is_dc && sym > 15) || out->size[sym]) return -1;
      out->code[sym] = (uint16_t)code; out->size[sym] = (uint8_t)l; code++;
    }
    if (code > (1u << l)) return -1;
    code <<= 1;
  }
  out->nsym16 = (uint16_t)n; out->nsym = (uint8_t)n;
  return 0;
}

struct Timer {
  b200jpeg_encoder *e; size_t idx = 0; cudaStream_t s = nullptr;
  void mark(const char *name) {
    if (idx >= e->ev.size()) { cudaEvent_t ev; cudaEventCreate(&ev); e->ev.push_back(ev); }
    cudaEventRecord(e->ev[idx], s ? s : e->stream);
    if (idx >= e->ev_names.size()) e->ev_names.push_back(name); else e->ev_names[idx] = name;
    idx++;
  }
};

// per-stage device times from the first `marks` timer events, summed by stage name over the chunks; an interval starts
// at every mark but "end" (with two streams the intervals of concurrent chunks overlap)
static void collect_stage_times(b200jpeg_encoder *e, size_t marks)
{
  e->pending_marks = 0;
  e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
  if (marks) cudaEventSynchronize(e->ev[marks - 1]);
  for (size_t i = 0; i + 1 < marks; i++) {
    if (!strcmp(e->ev_names[i], "end")) continue;
    float ms = 0.f; cudaEventElapsedTime(&ms, e->ev[i], e->ev[i + 1]);
    size_t k = 0;
    for (; k < e->stage_names.size(); k++) if (!strcmp(e->stage_names[k], e->ev_names[i])) break;
    if (k == e->stage_names.size()) { e->stage_names.push_back(e->ev_names[i]); e->stage_ms.push_back(0.f); e->stage_calls.push_back(0); }
    e->stage_ms[k] += ms; e->stage_calls[k]++;
  }
}

static uint32_t scan_slot_mask(const Plan &pl, const ScanDesc &sd)
{
  uint32_t m = 0;
  for (int i = 0; i < sd.ncomps; i++) {
    const CompGeom &c = pl.g.c[sd.ci[i]];
    bool want_dc = !pl.progressive || (sd.Ss == 0 && sd.Ah == 0);
    bool want_ac = !pl.progressive || (sd.Ss != 0);
    if (want_dc) m |= 1u << c.dc_tbl;
    if (want_ac) m |= 1u << (4 + c.ac_tbl);
  }
  return m;
}

// bytes per image of the smoothing pre-pass's planes (hib*8 rows of wib*8 samples per component, 256-byte aligned each)
static size_t smooth_plane_bytes(const Geom &g)
{
  const size_t sb = g.max_coef_bits == 14 ? 2 : 1; size_t t = 0;
  for (int ci = 0; ci < g.nc; ci++) t += ((size_t)g.c[ci].wib * 8 * sb * g.c[ci].hib * 8 + 255) & ~(size_t)255;
  return t;
}

// Sequential scans behind the default trellis (one round over 1..63 by k_trellis_ac3): the entropy stages read the symbol
// records the trellis back-track leaves instead of the coefficient planes.  B200JPEG_SYMREC=0 keeps them on the planes.
static bool use_symrec(const Plan &pl, const b200jpeg_params *p)
{
  static const bool off = getenv("B200JPEG_SYMREC") && getenv("B200JPEG_SYMREC")[0] == '0';
  const bool generic_rounds = p->use_scans_in_trellis || p->trellis_num_loops > 1 || p->trellis_q_opt || p->trellis_eob_opt;
  return !off && pl.trellis && !pl.progressive && !generic_rounds;
}

// Buffers and constants of one batch of n_total images processed in chunks of `chunk`.
static int prepare_batch(b200jpeg_encoder *e, int n_total, int chunk, bool host_pixels, size_t src_bytes, int n_arenas)
{
  Plan &pl = e->plan; const b200jpeg_params *p = &e->params; cudaStream_t s = e->stream;
  Geom &g = pl.g;
  const int nscans = (int)pl.scans.size();
  int rc;
  const int n = chunk;
  long long total_blocks = 0; for (int ci = 0; ci < g.nc; ci++) total_blocks += g.c[ci].blocks_per_image;
  if (pl.lossless) total_blocks = (total_blocks + 7) / 8;       // one sample per data unit: the buffers start at 2 bytes per sample
  size_t cap = (size_t)((double)total_blocks * 64 * e->cap_factor) + 65536;
  cap = (cap + 255) & ~(size_t)255;
  e->bitbuf_words_per_image = cap / 4; e->out_cap_per_image = (cap + cap / 64 + 4096) * (pl.search ? 6 : 1);   // scan search keeps all 64 candidate scans
  const size_t hist_bytes = (size_t)n * HIST_SLOTS * HIST_BINS * 4;
  const size_t tabset = sizeof(DevHuff) * HIST_SLOTS;
  for (int ai = 0; ai < n_arenas; ai++) {
    Arena &a = e->ar[ai];
    a.g = g;
    for (int ci = 0; ci < g.nc; ci++) {
      if ((rc = a.d_coef[ci].reserve(pl.coef_bytes[ci] * n))) return rc;
      if ((rc = a.d_raw[ci].reserve(pl.coef_bytes[ci] * n))) return rc;
      a.g.c[ci].coef = a.d_coef[ci].as<int16_t>(); a.g.c[ci].raw = a.d_raw[ci].as<int16_t>();
      if (e->keep_plain && pl.trellis) { if ((rc = a.d_plain[ci].reserve(pl.coef_bytes[ci] * n))) return rc; }
    }
    if (pl.smooth && !g.raw_in) { if ((rc = a.d_planes.reserve(smooth_plane_bytes(g) * n))) return rc; }
    if ((rc = a.d_hist.reserve(hist_bytes * g.nc))) return rc;
    if ((rc = a.d_tabs_trellis.reserve(tabset * 4 * n))) return rc;
    if ((rc = a.d_rec.reserve((size_t)n * pl.sum_real_blocks * sizeof(DcRec)))) return rc;
    if ((rc = a.d_srec.reserve((size_t)n * pl.sum_real_blocks * 16))) return rc;
    if ((rc = a.d_splits.reserve((size_t)n * 4 * (4 + 128) * 4))) return rc;      // class boundaries + the sort's counters
    if (use_symrec(pl, p)) {
      if ((rc = a.d_sym.reserve((size_t)n * pl.sum_real_blocks * SYMREC_BYTES))) return rc;
      if ((rc = a.d_dcq.reserve((size_t)n * pl.sum_real_blocks * 2))) return rc;
    }
    if ((rc = a.d_best_al.reserve((size_t)n * 2 * 4))) return rc;
    if (p->trellis_quant && p->trellis_q_opt) {
      if ((rc = a.d_qimg.reserve((size_t)n * 512))) return rc;
      if ((rc = a.d_qsum.reserve((size_t)n * 4 * 2 * 64 * 8))) return rc;
    }
    if (p->trellis_quant && p->trellis_eob_opt) {
      if ((rc = a.d_eo.reserve((size_t)n * pl.sum_real_blocks * 16))) return rc;
      if ((rc = a.d_es.reserve((size_t)n * pl.sum_real_blocks * 16))) return rc;
    }
    if (pl.lossless) { if ((rc = a.d_diff.reserve((size_t)n * pl.max_scan_blocks * g.nc * 2))) return rc; }
    if ((rc = a.d_blk_bits.reserve((size_t)n * pl.max_scan_blocks * 4))) return rc;
    if (pl.progressive) { if ((rc = a.d_blk_aux.reserve((size_t)n * pl.max_scan_blocks * 4))) return rc; if ((rc = a.d_blk_run.reserve((size_t)n * pl.max_scan_blocks * 4))) return rc; if ((rc = a.d_blk_mask.reserve((size_t)n * pl.max_scan_blocks * 24))) return rc; }
    if ((rc = a.d_total_bits.reserve((size_t)n * 8))) return rc;
    if ((rc = a.d_tile_bits.reserve((size_t)n * ((pl.max_scan_blocks + 255) / 256) * 4))) return rc;
    if ((rc = a.d_tile_base.reserve((size_t)n * ((pl.max_scan_blocks + 255) / 256) * 8))) return rc;
    if (pl.restarts) {
      if ((rc = a.d_seg_corr.reserve((size_t)n * pl.max_scan_blocks * 4))) return rc;       // worst case: one block per segment
      if ((rc = a.d_mark.reserve((size_t)n * (cap / 8 + 64)))) return rc;
    }
    if ((rc = a.d_bitbuf.reserve(cap * n))) return rc;
    if ((rc = a.d_stuff_lb.reserve(stuff_lookback_bytes(e->bitbuf_words_per_image, n)))) return rc;
  }
  // whole batch
  if (host_pixels) { if ((rc = e->d_src.reserve(src_bytes))) return rc; }
  if ((rc = e->d_tabs_scan.reserve(tabset * nscans * n_total))) return rc;
  if ((rc = e->d_tabs_fixed.reserve(tabset))) return rc;
  if ((rc = e->d_status.reserve((size_t)n_total * 4))) return rc;
  if ((rc = e->d_out_pos.reserve((size_t)n_total * (nscans + 1) * 8))) return rc;
  if ((rc = e->d_scan_size.reserve((size_t)n_total * nscans * 4))) return rc;
  if ((rc = e->d_best_al_all.reserve((size_t)n_total * 2 * 4))) return rc;
  const int ns = e->nsets;
  if (p->trellis_quant && p->trellis_q_opt) {
    if ((rc = e->d_qimg_all.reserve((size_t)n_total * 512))) return rc;
    if ((rc = e->h_qinit.reserve((size_t)ns * 512))) return rc;
    memcpy(e->h_qinit.p, e->qsets.data(), (size_t)ns * 512);              // every image starts from its own tables
  }
  if ((rc = e->d_out.reserve(e->out_cap_per_image * n_total))) return rc;
  if ((rc = e->d_qt.reserve(sizeof(QuantTables) * ns))) return rc;
  if ((rc = e->d_tc.reserve(sizeof(TrellisConsts) * ns))) return rc;
  if ((rc = e->h_qt.reserve(sizeof(QuantTables) * ns))) return rc;
  if ((rc = e->h_tc.reserve(sizeof(TrellisConsts) * ns))) return rc;
  if ((rc = e->h_fixed.reserve(tabset))) return rc;

  // the constants of every distinct table set (a parameter block that differs from p in quant_tbl only)
  for (int si = 0; si < ns; si++) {
    static thread_local b200jpeg_params ps;
    ps = *p; memcpy(ps.quant_tbl, &e->qsets[(size_t)si * 256], 512);
    make_quant_consts(&ps, e->h_qt.as<QuantTables>() + si);
    make_trellis_consts(&ps, e->h_tc.as<TrellisConsts>() + si);
    if (pl.trellis) for (int t = 0; t < 4; t++) {
      if (!ps.quant_tbl_present[t]) continue;
      unsigned dmin = ~0u; for (int k = 0; k < 64; k++) dmin = std::min(dmin, 8u * ps.quant_tbl[t][k]);
      if ((((1ull << (18 + e->h_tc.as<TrellisConsts>()[si].qL[t])) + dmin - 1) / dmin) >= (1ull << 32)) {
        if (e->img_set.empty()) set_error("trellis quantization: quantization table %d mixes values too far apart for the device divider", t);
        else {
          int img = 0; while (e->img_set[img] != si) img++;
          set_error("trellis quantization: image %d: quantization table %d mixes values too far apart for the device divider", img, t);
        }
        return B200JPEG_ERR_UNSUPPORTED;
      }
    }
  }
  if (!e->img_set.empty()) {
    if ((rc = e->d_qset.reserve((size_t)n_total * sizeof(int)))) return rc;
    if ((rc = e->h_qset.reserve((size_t)n_total * sizeof(int)))) return rc;
    memcpy(e->h_qset.p, e->img_set.data(), (size_t)n_total * sizeof(int));
    CU(cudaMemcpyAsync(e->d_qset.p, e->h_qset.p, (size_t)n_total * sizeof(int), cudaMemcpyHostToDevice, s));
  }
  {
    DevHuff *f = e->h_fixed.as<DevHuff>();
    for (int t = 0; t < 4; t++) {
      if (make_fixed_table(p->dc_huff_tbl[t], true, &f[t]) || make_fixed_table(p->ac_huff_tbl[t], false, &f[4 + t])) { set_error("Bogus Huffman table definition"); return B200JPEG_ERR_PARAM; }
    }
  }
  CU(cudaMemcpyAsync(e->d_qt.p, e->h_qt.p, sizeof(QuantTables) * ns, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_tc.p, e->h_tc.p, sizeof(TrellisConsts) * ns, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_tabs_fixed.p, e->h_fixed.p, tabset, cudaMemcpyHostToDevice, s));
  return B200JPEG_OK;
}

// The lossless pipeline for one chunk: per scan, differences + category counts -> optimal DC tables (one set per scan,
// finish_pass_gather, jclhuff.c:531-556) -> bits per MCU -> layout -> packing -> byte stuffing.
static int run_lossless(b200jpeg_encoder *e, const ChunkIO &io, Timer &tm)
{
  Plan &pl = e->plan; const b200jpeg_params *p = &e->params; const int n = io.n; cudaStream_t s = e->sc[io.slot];
  Arena &A = e->ar[io.slot];
  const Geom &g = A.g;
  tm.s = s;
  const int nscans = (int)pl.scans.size();
  const size_t hist_bytes = (size_t)n * HIST_SLOTS * HIST_BINS * 4;
  const size_t tabset = sizeof(DevHuff) * HIST_SLOTS, tstride = tabset * nscans;
  const size_t mark_words = (e->bitbuf_words_per_image * 4 / 8 + 64) / 4;
  for (size_t j = 0; j < pl.order.size(); j++) {
    const int si = pl.order[j];
    const ScanDesc &sd = pl.scans[si];
    DevHuff *tset = io.tabs_scan + (size_t)si * HIST_SLOTS;
    tm.mark("lossless_diff");
    CU(cudaMemsetAsync(A.d_hist.p, 0, hist_bytes, s));
    launch_lossless_diff(g, sd, p->data_precision, io.src, A.d_diff.as<uint16_t>(), A.d_hist.as<uint32_t>(), n, s);
    tm.mark("scan_tables");
    SlotMasks masks; memset(&masks, 0, sizeof masks); masks.period = 1;
    for (int i = 0; i < sd.ncomps; i++) masks.m[0] |= 1u << g.c[sd.ci[i]].dc_tbl;
    launch_gen_tables(A.d_hist.as<uint32_t>(), tset, tstride, masks, n, s);
    tm.mark("block_bits");
    launch_lossless_bits(g, sd, A.d_diff.as<uint16_t>(), tset, tstride, A.d_blk_bits.as<uint32_t>(), A.d_tile_bits.as<uint32_t>(), io.status, n, s);
    tm.mark("scan_layout");
    launch_scan_layout(sd, A.d_blk_bits.as<uint32_t>(), A.d_tile_bits.as<uint32_t>(), A.d_tile_base.as<unsigned long long>(),
                       A.d_seg_corr.as<uint32_t>(), pl.max_scan_blocks, A.d_total_bits.as<unsigned long long>(),
                       (size_t)e->bitbuf_words_per_image * 32, io.status, n, s);
    tm.mark("encode");
    launch_zero_stream(A.d_bitbuf.as<uint32_t>(), e->bitbuf_words_per_image, A.d_total_bits.as<unsigned long long>(), n, s);
    if (sd.ri) CU(cudaMemsetAsync(A.d_mark.p, 0, mark_words * 4 * n, s));
    launch_lossless_encode(g, sd, A.d_diff.as<uint16_t>(), tset, tstride, A.d_blk_bits.as<uint32_t>(), A.d_tile_base.as<unsigned long long>(),
                           A.d_seg_corr.as<uint32_t>(), pl.max_scan_blocks, A.d_bitbuf.as<uint32_t>(), e->bitbuf_words_per_image,
                           A.d_mark.as<uint32_t>(), mark_words, io.status, n, s);
    tm.mark("stuff");
    CU(cudaMemsetAsync(A.d_stuff_lb.p, 0, stuff_lookback_bytes(e->bitbuf_words_per_image, n), s));
    launch_stuff(A.d_bitbuf.as<uint32_t>(), e->bitbuf_words_per_image, A.d_total_bits.as<unsigned long long>(), A.d_stuff_lb.p,
                 io.out, e->out_cap_per_image, e->out_cap_per_image, io.out_pos + j * n, io.out_pos + (j + 1) * n,
                 io.scan_size + (size_t)si * n, io.status, sd.ri ? A.d_mark.as<uint32_t>() : nullptr, mark_words, n, s);
  }
  tm.mark("end");
  CU(cudaGetLastError());
  e->last_chunk_i0 = io.i0; e->last_chunk_n = io.n; e->last_chunk_slot = io.slot;
  return B200JPEG_OK;
}

// The device pipeline for one chunk (pixels already in HBM): the pass plan of
// jcmaster.c with every pass one launch over all images of the chunk.
static int run_pipeline(b200jpeg_encoder *e, const ChunkIO &io, Timer &tm)
{
  if (e->plan.lossless) return run_lossless(e, io, tm);
  Plan &pl = e->plan; const b200jpeg_params *p = &e->params; const int n = io.n; cudaStream_t s = e->sc[io.slot];
  Arena &A = e->ar[io.slot];
  Geom &g = A.g;
  tm.s = s;
  const int nscans = (int)pl.scans.size();
  const size_t hist_bytes = (size_t)n * HIST_SLOTS * HIST_BINS * 4;
  const size_t tabset = sizeof(DevHuff) * HIST_SLOTS;
  const uint8_t *src_dev = io.src;
  for (int ci = 0; ci < 4; ci++) g.plane[ci] = io.plane[ci];
  g.qset = io.qset;
  uint32_t *status = io.status;

  const bool symrec = use_symrec(pl, p);
  const bool symstats = symrec && pl.optimize && nscans == 1;
  // ---- pass 0 data path: colour/downsample/FDCT/quantize (compress_first_pass) ----
  RecLayout rl; memset(&rl, 0, sizeof rl);
  for (int ci = 0; ci < g.nc; ci++) { rl.comp_off[ci] = rl.per_image; rl.per_image += (long long)g.c[ci].wib * g.c[ci].hib; }
  rl.sym_hi = (long long)n * rl.per_image * (SYMREC_BYTES / 2);      // second plane of the symbol records (SYMREC_SPLIT)
  tm.mark("forward");
  // the fast quantizer / DC-trellis forms serve a launch only if every table set allows them for the launch's components
  int qfast = 1;
  for (int si = 0; si < e->nsets; si++)
    for (int ci = 0; ci < g.nc; ci++) qfast &= e->h_qt.as<QuantTables>()[si].fast[g.c[ci].qt];
  auto dc_fast_of = [&](const Geom &gr) {
    int f = 1;
    for (int si = 0; si < e->nsets; si++)
      for (int ci = 0; ci < gr.nc; ci++) f &= e->h_tc.as<TrellisConsts>()[si].dc_fast[gr.c[ci].qt];
    return f;
  };
  Geom gf = g;
  // the default sequential trellis behind the tiled forward kernel: that kernel counts the trellis-phase AC statistics
  // and leaves the plain DC values in dcq, so the plain-quantized planes are neither written nor read (the debug taps
  // of B200JPEG_KEEP_PLAIN read them, and keep the separate statistics pass)
  bool fwd_stats = false;
  if (g.raw_in == 2) {
    launch_import_coefs(g, e->xform, n, s);
  } else {
  if (pl.smooth && !g.raw_in) {
    // input smoothing: conversion + context-mode downsampling as a pre-pass; the forward kernel then reads planes
    tm.mark("smooth_planes");
    const size_t sb = g.max_coef_bits == 14 ? 2 : 1;
    PlanesOut po; memset(&po, 0, sizeof po); size_t off = 0;
    for (int ci = 0; ci < g.nc; ci++) {
      po.pitch[ci] = (size_t)g.c[ci].wib * 8 * sb; po.stride[ci] = (po.pitch[ci] * g.c[ci].hib * 8 + 255) & ~(size_t)255;
      po.p[ci] = A.d_planes.as<uint8_t>() + off; off += po.stride[ci] * n;
      gf.plane[ci] = po.p[ci]; gf.plane_pitch[ci] = po.pitch[ci]; gf.plane_stride[ci] = po.stride[ci];
    }
    launch_prep_planes(g, src_dev, pl.smooth, po, n, s);
    gf.raw_in = 1;
    tm.mark("forward");
  }
  fwd_stats = symrec && !e->keep_plain && forward_tiled(gf, p->dct_method);
  FwdStats fs = {nullptr, nullptr, nullptr};
  if (fwd_stats) {
    CU(cudaMemsetAsync(A.d_hist.p, 0, hist_bytes * g.nc, s));
    fs = {A.d_hist.as<uint32_t>(), A.d_dcq.as<int16_t>(), status};
  }
  launch_forward(gf, src_dev, e->d_qt.as<QuantTables>(), qfast, p->dct_method, pl.dering, pl.trellis ? A.d_rec.as<DcRec>() : nullptr, rl, e->keep_plain ? 1 : 0, fs, n, s);
  }
  // dummy blocks: on the fwd_stats path nothing reads them from the planes (the scans take a dummy block as an EOB with
  // the DC of dense_dc)
  if (!fwd_stats) {
    tm.mark("dummy");
    launch_dummy(g, n, s);
  }

  // ---- trellis phase (jcmaster.c pass list, SURVEY 3.1).  The three
  //      per-component chains (statistics on the plain-quantized coefficients
  //      -> optimal tables -> quantize_trellis) are independent, so each step
  //      is ONE launch over all components of all images. ----
  if (pl.trellis) {
    if (e->keep_plain) for (int ci = 0; ci < g.nc; ci++) CU(cudaMemcpyAsync(A.d_plain[ci].p, A.d_coef[ci].p, pl.coef_bytes[ci] * n, cudaMemcpyDeviceToDevice, s));
    DevHuff *tset = A.d_tabs_trellis.as<DevHuff>();                                       // [img*nc + ci][8]
    // use_scans_in_trellis (jcmaster.c:451-467): two statistics -> tables -> quantize_trellis rounds per component, on
    // the zigzag bands 1..trellis_freq_split and the rest; otherwise one round on 1..63
    const int nband = p->use_scans_in_trellis ? 2 : 1;
    // trellis_num_loops > 1 repeats the rounds (jcmaster.c:453-465); later rounds start from the requantized
    // coefficients, which the band kernel honours (it reads the values a block has on entry), so it serves those too;
    // trellis_eob_opt and trellis_q_opt also run on it (it reports the per-block costs the EOB-run pass needs and takes
    // per-image tables)
    const bool qopt = p->trellis_q_opt != 0, eobopt = p->trellis_eob_opt != 0;
    const bool generic_rounds = nband == 2 || p->trellis_num_loops > 1 || qopt || eobopt;
    // symbol records for the sequential scans that follow; with optimal tables for ONE scan over all components, the
    // back-track also counts that scan's AC symbols (the histograms are free again once the trellis tables are built)
    SymOut so; so.sym = symrec ? A.d_sym.as<uint8_t>() : nullptr; so.dcq = symrec ? A.d_dcq.as<int16_t>() : nullptr;
    so.hist = symstats ? A.d_hist.as<uint32_t>() : nullptr;
    so.keep_coef = e->keep_plain ? 1 : 0;                       // B200JPEG_KEEP_PLAIN=1: the debug taps read the final planes
    so.dcq_ac = (p->trellis_quant_dc || fwd_stats) ? 0 : 1;    // (the forward kernel wrote the plain DC values)
    uint16_t *qimg = qopt ? A.d_qimg.as<uint16_t>() : nullptr;
    if (qopt) {
      // every image starts from its own table set (natural order, like JQUANT_TBL.quantval)
      for (int i = 0; i < n; i++) {
        const int si = e->img_set.empty() ? 0 : e->img_set[io.i0 + i];
        CU(cudaMemcpyAsync(qimg + (size_t)i * 256, e->h_qinit.as<uint16_t>() + (size_t)si * 256, 512, cudaMemcpyHostToDevice, s));
      }
    }
    // one statistics -> tables -> quantize_trellis round over the components of gr (all of them, or one)
    auto round = [&](const Geom &gr, const RecLayout &rlr, int bSs, int bSe) -> int {
    if (!pl.progressive) {
      if (fwd_stats) {                                        // one round, its AC counts are in already
        tm.mark("trellis_dc_stats");
        launch_gather_comp_dc(gr, pl.rs, so.dcq, rlr, A.d_hist.as<uint32_t>(), status, n, s);
      } else {
        tm.mark("trellis_stats");
        CU(cudaMemsetAsync(A.d_hist.p, 0, hist_bytes * gr.nc, s));
        launch_gather_comp(gr, pl.rs, A.d_hist.as<uint32_t>(), status, n, s);
      }
      tm.mark("trellis_tables");
      SlotMasks masks; memset(&masks, 0, sizeof masks); masks.period = gr.nc;
      for (int ci = 0; ci < gr.nc; ci++) masks.m[ci] = (1u << gr.c[ci].dc_tbl) | (1u << (4 + gr.c[ci].ac_tbl));
      launch_gen_tables(A.d_hist.as<uint32_t>(), tset, tabset, masks, n * gr.nc, s);
    } else {
      // jcphuff statistics with Ss=1..63 (or the band), Al=0 (jcmaster.c:462-466), every AC symbol
      // pre-counted once (jcphuff.c:257-264); the DC table stays the supplied one.
      for (int ci = 0; ci < gr.nc; ci++) {
        ScanDesc ts; memset(&ts, 0, sizeof ts);
        ts.ncomps = 1; ts.ci[0] = ci; ts.Ss = bSs; ts.Se = bSe; ts.bim = 1; ts.k_count[0] = 1;
        ts.per_row = gr.c[ci].wib; ts.rows = gr.c[ci].hib; ts.nblocks = (long long)ts.per_row * ts.rows;
        ts.ri = p->restart_in_rows > 0 ? (int)std::min((long long)p->restart_in_rows * ts.per_row, 65535LL) : p->restart_interval;
        tm.mark("trellis_stats");
        CU(cudaMemsetAsync(A.d_hist.p, 0, hist_bytes, s));
        launch_seed_hist(A.d_hist.as<uint32_t>(), 4 + gr.c[ci].ac_tbl, n, s);
        launch_prog_prepare(gr, ts, A.d_blk_aux.as<uint32_t>(), A.d_blk_run.as<uint32_t>(), A.d_blk_mask.as<unsigned long long>(), A.d_tile_bits.as<int>(), A.d_tile_base.as<int>(), n, s);
        launch_gather_prog(gr, ts, A.d_blk_aux.as<uint32_t>(), A.d_blk_run.as<uint32_t>(), A.d_blk_mask.as<unsigned long long>(), A.d_hist.as<uint32_t>(), status, n, s);
        tm.mark("trellis_tables");
        SlotMasks masks; memset(&masks, 0, sizeof masks); masks.period = 1; masks.m[0] = 1u << (4 + gr.c[ci].ac_tbl);
        launch_gen_tables(A.d_hist.as<uint32_t>(), tset + (size_t)ci * HIST_SLOTS, tabset * gr.nc, masks, n, s);
      }
    }
    if (!generic_rounds) {
      tm.mark("trellis_sort");
      launch_trellis_sort(gr, A.d_rec.as<DcRec>(), rlr, A.d_srec.p, A.d_splits.as<uint32_t>(), n, s);
      tm.mark("trellis_ac");
      if (so.hist) CU(cudaMemsetAsync(A.d_hist.p, 0, hist_bytes, s));
      launch_trellis_ac3(gr, e->d_tc.as<TrellisConsts>(), tset, tabset, A.d_rec.as<DcRec>(), rlr, A.d_srec.p, A.d_splits.as<uint32_t>(), so, n, e->sms, s);
    } else {
      tm.mark("trellis_ac");
      float4 *eo = eobopt ? A.d_eo.as<float4>() : nullptr;
      launch_trellis_ac_band(gr, e->d_tc.as<TrellisConsts>(), tset, tabset, A.d_rec.as<DcRec>(), rlr, bSs, bSe, qimg, eo, n, s);
      if (eobopt) launch_trellis_eob_rows(gr, tset, tabset, A.d_rec.as<DcRec>(), rlr, bSs, bSe, eo, A.d_es.p, n, s);
      if (qopt) launch_qopt_sums(gr, A.d_qsum.as<long long>(), n, s);
    }
    if (p->trellis_quant_dc) {
      tm.mark("trellis_dc");
      // behind k_trellis_ac3 the records still hold the norm; the band kernel stores lambda_dc (from re-fitted tables
      // with trellis_q_opt)
      const int lambda_from_norm = generic_rounds ? 0 : 1;
      if (pl.progressive) launch_trellis_dc(gr, e->d_tc.as<TrellisConsts>(), e->d_tabs_fixed.as<DevHuff>(), 0, A.d_rec.as<DcRec>(), rlr, p->trellis_delta_dc_weight > 0.0f, dc_fast_of(gr), nullptr, 1, lambda_from_norm, n, s);
      else launch_trellis_dc(gr, e->d_tc.as<TrellisConsts>(), tset, tabset, A.d_rec.as<DcRec>(), rlr, p->trellis_delta_dc_weight > 0.0f, dc_fast_of(gr), so.dcq, so.keep_coef, lambda_from_norm, n, s);
    }
    return B200JPEG_OK;
    };
    auto band_Ss = [&](int band) { return (nband == 2 && band == 1) ? p->trellis_freq_split + 1 : 1; };
    auto band_Se = [&](int band) { return (nband == 2 && band == 0) ? p->trellis_freq_split : 63; };
    if (!qopt) {
      // the components' chains are independent: every round is one launch set over all of them
      for (int loop = 0; loop < p->trellis_num_loops; loop++)
        for (int band = 0; band < nband; band++) { int rc = round(g, rl, band_Ss(band), band_Se(band)); if (rc) return rc; }
    } else {
      // trellis_q_opt re-fits the tables every `group` passes of the reference's pass list (jcmaster.c:1014-1030), which
      // walks the components one after the other (pass -> component, :453-465): a table one component updates is the
      // table the next component's rounds use, so the rounds run in that order, one component at a time
      const int group = g.nc * (nband == 2 ? 4 : 2);
      int pass_number = 0;
      CU(cudaMemsetAsync(A.d_qsum.p, 0, (size_t)n * 4 * 2 * 64 * 8, s));
      for (int ci = 0; ci < g.nc; ci++) {
        Geom gs = g; gs.nc = 1; gs.c[0] = g.c[ci];
        RecLayout rls = rl; rls.comp_off[0] = rl.comp_off[ci];
        for (int loop = 0; loop < p->trellis_num_loops; loop++)
          for (int band = 0; band < nband; band++) {
            pass_number++;                                          // the statistics pass
            if (pass_number % group == 1) CU(cudaMemsetAsync(A.d_qsum.p, 0, (size_t)n * 4 * 2 * 64 * 8, s));   // prepare_for_pass, jcmaster.c:687-698
            int rc = round(gs, rls, band_Ss(band), band_Se(band)); if (rc) return rc;
            if ((pass_number + 1) % group == 0) launch_qopt_update(A.d_qsum.as<long long>(), qimg, n, s);
            pass_number++;                                          // the trellis pass
          }
      }
      CU(cudaMemcpyAsync(io.qimg, qimg, (size_t)n * 512, cudaMemcpyDeviceToDevice, s));      // kept per chunk for the DQT markers
    }
    if (!fwd_stats) {
      tm.mark("dummy");
      launch_dummy(g, n, s);
    }
  }

  // ---- scans: huff_opt_pass (statistics -> tables) + output_pass.  With the scan search on, all 64 (23) candidate
  //      scans are coded (the reference codes them one by one into memory buffers, jcmaster.c:668-674); the two
  //      frequency-split groups are coded at each image's best Al, chosen on the device in between. ----
  int *best_al = A.d_best_al.as<int>();                       // [2][n]: luma, chroma
  // sequential scans after the trellis: the side records hold every block's final non-zero positions
  const DcRec *nz_rec = (pl.trellis && !pl.progressive && !symrec) ? A.d_rec.as<DcRec>() : nullptr;
  const uint8_t *sym = symrec ? A.d_sym.as<uint8_t>() : nullptr;
  const int16_t *dcq = symrec ? A.d_dcq.as<int16_t>() : nullptr;
  for (size_t j = 0; j < pl.order.size(); j++) {
    const int si = pl.order[j];
    ScanDesc sd = pl.scans[si];
    if (pl.search) {
      const bool colour = nscans > pl.n_luma;
      if (si == pl.luma_split0) {                               // all luma Al-search scans are done: pick the best Al per image
        AlSearch as; memset(&as, 0, sizeof as);
        as.first = 1; as.per_al = 3; as.nband = 2; as.al_max = 3; as.nscans_total = nscans;
        for (int k = 0; k < pl.luma_split0 - 1; k++) as.sd[k] = pl.scans[1 + k];
        tm.mark("select_al");
        launch_select_al(g, as, io.tabs_scan, io.scan_size, n, best_al, s);
        if (colour) {
          AlSearch ac; memset(&ac, 0, sizeof ac);
          ac.first = pl.chroma_al0; ac.per_al = 6; ac.nband = 4; ac.al_max = 2; ac.nscans_total = nscans;
          for (int k = 0; k < pl.chroma_split0 - pl.chroma_al0; k++) ac.sd[k] = pl.scans[pl.chroma_al0 + k];
          launch_select_al(g, ac, io.tabs_scan, io.scan_size, n, best_al + n, s);
        }
      }
      if (si >= pl.luma_split0 && si < pl.n_luma) sd.al_img = best_al;            // jcmaster.c:477-482
      if (si >= pl.chroma_split0) sd.al_img = best_al + n;                         // jcmaster.c:483-488
    }
    const DevHuff *tabs; size_t tstride;
    const bool dc_refine = pl.progressive && sd.Ss == 0 && sd.Ah != 0;
    uint32_t *aux = A.d_blk_aux.as<uint32_t>(), *run_e = A.d_blk_run.as<uint32_t>();
    unsigned long long *pm = A.d_blk_mask.as<unsigned long long>();
    if (pl.progressive && sd.Ss != 0) { tm.mark("eobrun_runs"); launch_prog_prepare(g, sd, aux, run_e, pm, A.d_tile_bits.as<int>(), A.d_tile_base.as<int>(), n, s); }
    if (pl.optimize) {
      DevHuff *tset = io.tabs_scan + (size_t)si * HIST_SLOTS;                              // [img][scan][8]
      tstride = tabset * nscans;
      if (!dc_refine) {                                                                    // jcmaster.c:650-662
        tm.mark("scan_stats");
        if (!symstats) CU(cudaMemsetAsync(A.d_hist.p, 0, hist_bytes, s));
        if (pl.progressive) launch_gather_prog(g, sd, aux, run_e, pm, A.d_hist.as<uint32_t>(), status, n, s);
        else if (symstats) launch_gather_seq_dc(g, sd, dcq, rl, A.d_hist.as<uint32_t>(), status, n, s);      // the AC counts are there already
        else launch_gather_seq(g, sd, nz_rec, sym, dcq, rl, A.d_hist.as<uint32_t>(), status, n, s);
        tm.mark("scan_tables");
        SlotMasks masks; memset(&masks, 0, sizeof masks); masks.period = 1; masks.m[0] = scan_slot_mask(pl, sd);
        launch_gen_tables(A.d_hist.as<uint32_t>(), tset, tstride, masks, n, s);
      }
      tabs = tset;
    } else { tabs = e->d_tabs_fixed.as<DevHuff>(); tstride = 0; }
    const size_t mark_words = (e->bitbuf_words_per_image * 4 / 8 + 64) / 4;
    tm.mark("block_bits");
    launch_block_bits(g, sd, nz_rec, sym, dcq, rl, tabs, tstride, pl.progressive, A.d_blk_bits.as<uint32_t>(), A.d_tile_bits.as<uint32_t>(), aux, run_e, pm, status, n, s);
    tm.mark("scan_layout");
    launch_scan_layout(sd, A.d_blk_bits.as<uint32_t>(), A.d_tile_bits.as<uint32_t>(), A.d_tile_base.as<unsigned long long>(),
                       A.d_seg_corr.as<uint32_t>(), pl.max_scan_blocks, A.d_total_bits.as<unsigned long long>(),
                       (size_t)e->bitbuf_words_per_image * 32, status, n, s);
    tm.mark("encode");
    launch_zero_stream(A.d_bitbuf.as<uint32_t>(), e->bitbuf_words_per_image, A.d_total_bits.as<unsigned long long>(), n, s);
    if (sd.ri) CU(cudaMemsetAsync(A.d_mark.p, 0, mark_words * 4 * n, s));
    launch_encode(g, sd, nz_rec, sym, dcq, rl, tabs, tstride, pl.progressive, A.d_blk_bits.as<uint32_t>(), A.d_tile_bits.as<uint32_t>(), A.d_tile_base.as<unsigned long long>(),
                  A.d_seg_corr.as<uint32_t>(), pl.max_scan_blocks, aux, run_e, pm,
                  A.d_bitbuf.as<uint32_t>(), e->bitbuf_words_per_image, A.d_mark.as<uint32_t>(), mark_words, status, n, s);
    tm.mark("stuff");
    CU(cudaMemsetAsync(A.d_stuff_lb.p, 0, stuff_lookback_bytes(e->bitbuf_words_per_image, n), s));
    launch_stuff(A.d_bitbuf.as<uint32_t>(), e->bitbuf_words_per_image, A.d_total_bits.as<unsigned long long>(), A.d_stuff_lb.p,
                 io.out, e->out_cap_per_image, e->out_cap_per_image, io.out_pos + j * n, io.out_pos + (j + 1) * n,
                 io.scan_size + (size_t)si * n, status, sd.ri ? A.d_mark.as<uint32_t>() : nullptr, mark_words, n, s);
  }
  if (pl.search) CU(cudaMemcpyAsync(io.best_al, best_al, (size_t)n * 2 * sizeof(int), cudaMemcpyDeviceToDevice, s));   // kept per chunk for the host
  tm.mark("end");
  CU(cudaGetLastError());
  e->last_chunk_i0 = io.i0; e->last_chunk_n = io.n; e->last_chunk_slot = io.slot;
  return B200JPEG_OK;
}

// ------------------------------------------------------------------ host-side file assembly (jcmarker.c)
struct Bytes {
  std::vector<uint8_t> &v;
  void b(int x) { v.push_back((uint8_t)x); }
  void w(int x) { v.push_back((uint8_t)(x >> 8)); v.push_back((uint8_t)x); }
};

static void write_file_header(const b200jpeg_params *p, Bytes o)                     // jcmarker.c:649-663
{
  o.w(0xFFD8);
  if (p->write_JFIF_header) {                                                         // :529-561
    o.w(0xFFE0); o.w(16); o.b('J'); o.b('F'); o.b('I'); o.b('F'); o.b(0);
    o.b(p->JFIF_major_version); o.b(p->JFIF_minor_version); o.b(p->density_unit);
    o.w(p->X_density); o.w(p->Y_density); o.b(0); o.b(0);
  }
  if (p->write_Adobe_marker) {                                                        // :564-620
    o.w(0xFFEE); o.w(14); o.b('A'); o.b('d'); o.b('o'); o.b('b'); o.b('e'); o.w(100); o.w(0); o.w(0);
    o.b(p->jpeg_color_space == B200JPEG_CS_YCbCr ? 1 : p->jpeg_color_space == B200JPEG_CS_YCCK ? 2 : 0);   // colour transform
  }
}
static void write_frame_header(const b200jpeg_params *p, bool progressive, Bytes o)   // jcmarker.c:674-735
{
  int nc = p->num_components, prec = 0;
  const bool lossless = is_lossless(p);
  bool multi = p->compress_profile != B200JPEG_PROFILE_FASTEST;                       // emit_multi_dqt :189-254
  // emit_multi_dqt runs before the lossless test (:684-697) and gives up when a component's table is missing (:207-208)
  for (int ci = 0; ci < nc; ci++) if (!p->quant_tbl_present[p->comp_info[ci].quant_tbl_no & 3]) multi = false;
  bool sent[4] = {false, false, false, false};
  if (multi) {
    int precs[4] = {0, 0, 0, 0}, size = 0; bool seen[4] = {false, false, false, false};
    for (int ci = 0; ci < nc; ci++) { int t = p->comp_info[ci].quant_tbl_no; for (int i = 0; i < 64; i++) if (p->quant_tbl[t][i] > 255) precs[ci] = 1; prec += precs[ci]; }
    o.w(0xFFDB);
    for (int ci = 0; ci < nc; ci++) { int t = p->comp_info[ci].quant_tbl_no; if (!seen[t]) { size += 64 * (precs[ci] + 1) + 1; seen[t] = true; } }
    o.w(size + 2);
    for (int ci = 0; ci < nc; ci++) {
      int t = p->comp_info[ci].quant_tbl_no;
      if (sent[t]) continue;
      o.b(t + (precs[ci] << 4));
      for (int i = 0; i < 64; i++) { unsigned q = p->quant_tbl[t][kZigzag[i]]; if (precs[ci]) o.b(q >> 8); o.b(q & 0xFF); }
      sent[t] = true;
    }
  } else if (!lossless) {
    for (int ci = 0; ci < nc; ci++) {                                                  // emit_dqt :140-187
      int t = p->comp_info[ci].quant_tbl_no, pr = 0;
      for (int i = 0; i < 64; i++) if (p->quant_tbl[t][i] > 255) pr = 1;
      if (!sent[t]) {
        o.w(0xFFDB); o.w(pr ? 64 * 2 + 1 + 2 : 64 + 1 + 2); o.b(t + (pr << 4));
        for (int i = 0; i < 64; i++) { unsigned q = p->quant_tbl[t][kZigzag[i]]; if (pr) o.b(q >> 8); o.b(q & 0xFF); }
        sent[t] = true;
      }
      prec += pr;
    }
  }
  bool is_baseline;
  if (progressive || lossless || p->data_precision != 8) is_baseline = false;
  else {
    is_baseline = true;
    for (int ci = 0; ci < nc; ci++) if (p->comp_info[ci].dc_tbl_no > 1 || p->comp_info[ci].ac_tbl_no > 1) is_baseline = false;
    if (prec && is_baseline) is_baseline = false;
  }
  o.w(progressive ? 0xFFC2 : lossless ? 0xFFC3 : (is_baseline ? 0xFFC0 : 0xFFC1));     // emit_sof :464-491, :720-733
  o.w(3 * nc + 2 + 5 + 1); o.b(p->data_precision); o.w(p->image_height); o.w(p->image_width); o.b(nc);
  for (int ci = 0; ci < nc; ci++) { o.b(p->comp_info[ci].component_id); o.b((p->comp_info[ci].h_samp_factor << 4) + p->comp_info[ci].v_samp_factor); o.b(p->comp_info[ci].quant_tbl_no); }
}
// table state across scans (JHUFF_TBL.sent_table)
struct TblState { const HostHuff *dc[4]; const HostHuff *ac[4]; bool dc_sent[4]; bool ac_sent[4]; };

static int huff_len(const HostHuff *h) { int n = 0; for (int l = 1; l <= 16; l++) n += h->bits[l]; return n; }
static void write_scan_header(const b200jpeg_params *p, const ScanDesc &sd, TblState &ts, int &last_ri, unsigned ri, Bytes o)   // jcmarker.c:744-784
{
  bool multi = p->compress_profile != B200JPEG_PROFILE_FASTEST;
  bool done_multi = false;
  if (multi) {                                                                           // emit_multi_dht :293-401
    int length = 2, dclens[4] = {0, 0, 0, 0}, aclens[4] = {0, 0, 0, 0}; int dcseen[4] = {-1, -1, -1, -1}, acseen[4] = {-1, -1, -1, -1};
    for (int i = 0; i < sd.ncomps; i++) {
      const b200jpeg_component_info &c = p->comp_info[sd.ci[i]];
      int dcidx = c.dc_tbl_no, acidx = c.ac_tbl_no, seen = 0;
      if (sd.Ss == 0 && sd.Ah == 0) {
        if (ts.dc_sent[dcidx]) continue;
        for (int j = 0; j < 4; j++) seen += (dcseen[j] == dcidx);
        if (seen) continue;
        dcseen[i] = dcidx; dclens[i] = huff_len(ts.dc[dcidx]); length += dclens[i] + 16 + 1;
      }
      if (sd.Se) {
        if (ts.ac_sent[acidx]) continue;
        seen = 0; for (int j = 0; j < 4; j++) seen += (acseen[j] == acidx);
        if (seen) continue;
        acseen[i] = acidx; aclens[i] = huff_len(ts.ac[acidx]); length += aclens[i] + 16 + 1;
      }
    }
    if (length <= 65535) {
      o.w(0xFFC4); o.w(length);
      for (int i = 0; i < sd.ncomps; i++) {
        const b200jpeg_component_info &c = p->comp_info[sd.ci[i]];
        int dcidx = c.dc_tbl_no, acidx = c.ac_tbl_no;
        if (sd.Ss == 0 && sd.Ah == 0 && !ts.dc_sent[dcidx]) {
          o.b(dcidx); for (int j = 1; j <= 16; j++) o.b(ts.dc[dcidx]->bits[j]); for (int j = 0; j < dclens[i]; j++) o.b(ts.dc[dcidx]->huffval[j]);
          ts.dc_sent[dcidx] = true;
        }
        if (sd.Se && !ts.ac_sent[acidx]) {
          o.b(acidx + 0x10); for (int j = 1; j <= 16; j++) o.b(ts.ac[acidx]->bits[j]); for (int j = 0; j < aclens[i]; j++) o.b(ts.ac[acidx]->huffval[j]);
          ts.ac_sent[acidx] = true;
        }
      }
      done_multi = true;
    }
  }
  if (!done_multi) {
    for (int i = 0; i < sd.ncomps; i++) {                                                // emit_dht :256-291
      const b200jpeg_component_info &c = p->comp_info[sd.ci[i]];
      for (int z = 0; z < 2; z++) {
        bool is_ac = z == 1;
        if (!is_ac && !((sd.Ss == 0 && sd.Ah == 0) || is_lossless(p))) continue;        // lossless: DC tables only (:765-770)
        if (is_ac && (!sd.Se || is_lossless(p))) continue;
        int idx = is_ac ? c.ac_tbl_no : c.dc_tbl_no;
        bool &sent = is_ac ? ts.ac_sent[idx] : ts.dc_sent[idx];
        const HostHuff *h = is_ac ? ts.ac[idx] : ts.dc[idx];
        if (sent) continue;
        int len = huff_len(h);
        o.w(0xFFC4); o.w(len + 2 + 1 + 16); o.b(idx + (is_ac ? 0x10 : 0));
        for (int j = 1; j <= 16; j++) o.b(h->bits[j]);
        for (int j = 0; j < len; j++) o.b(h->huffval[j]);
        sent = true;
      }
    }
  }
  if ((int)ri != last_ri) { o.w(0xFFDD); o.w(4); o.w((int)ri); last_ri = (int)ri; }       // emit_dri
  o.w(0xFFDA); o.w(2 * sd.ncomps + 2 + 1 + 3); o.b(sd.ncomps);                          // emit_sos :494-526
  for (int i = 0; i < sd.ncomps; i++) {
    const b200jpeg_component_info &c = p->comp_info[sd.ci[i]];
    int td = (sd.Ss == 0 && sd.Ah == 0) ? c.dc_tbl_no : 0, ta = sd.Se ? c.ac_tbl_no : 0;
    o.b(c.component_id); o.b((td << 4) + ta);
  }
  o.b(sd.Ss); o.b(sd.Se); o.b((sd.Ah << 4) + sd.Al);
}

// ---- finished files live in pinned arenas (bump allocation; steady state = one arena, no allocation) ----
static void arena_reset(b200jpeg_encoder *e, size_t expect)
{
  size_t have = 0; for (PinBuf &b : e->file_arenas) have += b.cap;
  if (e->file_arenas.size() != 1 || have < expect) {
    size_t want = std::max(have, expect);
    for (PinBuf &b : e->file_arenas) b.release();
    e->file_arenas.clear();
    e->file_arenas.emplace_back();
    if (e->file_arenas[0].reserve(want)) e->file_arenas.clear();
  }
  e->arena_idx = 0; e->arena_off = 0;
}
static uint8_t *arena_alloc(b200jpeg_encoder *e, size_t size)
{
  size = (size + 63) & ~(size_t)63;
  while (e->arena_idx < e->file_arenas.size()) {
    PinBuf &b = e->file_arenas[e->arena_idx];
    if (e->arena_off + size <= b.cap) { uint8_t *r = b.as<uint8_t>() + e->arena_off; e->arena_off += size; return r; }
    e->arena_idx++; e->arena_off = 0;
  }
  e->file_arenas.emplace_back();
  if (e->file_arenas.back().reserve(std::max(size, (size_t)64 << 20))) { e->file_arenas.pop_back(); return nullptr; }
  e->arena_idx = e->file_arenas.size() - 1; e->arena_off = size;
  return e->file_arenas.back().as<uint8_t>();
}

// Queue the read-back of chunk k's metadata (status, sizes, DHT payloads) behind its pipeline.
static int queue_meta(b200jpeg_encoder *e, const ChunkIO &io, int k)
{
  Plan &pl = e->plan; cudaStream_t s = e->sc[io.slot];
  const int nscans = (int)pl.scans.size();
  CU(cudaMemcpyAsync(e->h_status.as<uint32_t>() + io.i0, io.status, (size_t)io.n * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(e->h_out_pos.as<unsigned long long>() + (size_t)io.i0 * (nscans + 1), io.out_pos, (size_t)io.n * (nscans + 1) * 8, cudaMemcpyDeviceToHost, s));
  if (pl.search) CU(cudaMemcpyAsync(e->h_best_al.as<int>() + (size_t)io.i0 * 2, io.best_al, (size_t)io.n * 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (pl.trellis && e->params.trellis_q_opt) CU(cudaMemcpyAsync(e->h_qimg.as<uint16_t>() + (size_t)io.i0 * 256, io.qimg, (size_t)io.n * 512, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(e->h_scan_size.as<uint32_t>() + (size_t)io.i0 * nscans, io.scan_size, (size_t)io.n * nscans * 4, cudaMemcpyDeviceToHost, s));
  if (pl.optimize) {
    size_t ntab = (size_t)io.n * nscans * HIST_SLOTS;
    CU(cudaMemcpy2DAsync(e->h_tabs.as<HostHuff>() + (size_t)io.i0 * nscans * HIST_SLOTS, sizeof(HostHuff), io.tabs_scan, sizeof(DevHuff), sizeof(HostHuff), ntab, cudaMemcpyDeviceToHost, s));
  } else if (k == 0) {
    CU(cudaMemcpy2DAsync(e->h_tabs.p, sizeof(HostHuff), e->d_tabs_fixed.p, sizeof(DevHuff), sizeof(HostHuff), HIST_SLOTS, cudaMemcpyDeviceToHost, s));
  }
  CU(cudaEventRecord(e->ev_done[k], s));
  return B200JPEG_OK;
}

// ---- scan search on the host: the decisions of select_scans (jcmaster.c:773-962) replayed on the sizes of the
// candidate scans.  total[si] = DHT + SOS + entropy-coded bytes of scan si, i.e. what the reference has in
// master->scan_size[si] (its memory destination receives write_scan_header too, jcmaster.c:668-681; scan 0 also holds
// the frame header, but scan 0 never enters a comparison). ----
static unsigned long scan_header_bytes(const Plan &pl, const ScanDesc &sd, const HostHuff *set)
{
  unsigned long dht = 0; unsigned seen = 0;
  for (int i = 0; i < sd.ncomps; i++) {
    const CompGeom &c = pl.g.c[sd.ci[i]];
    if (sd.Ss == 0 && sd.Ah == 0 && !((seen >> c.dc_tbl) & 1u)) { seen |= 1u << c.dc_tbl; dht += 17 + huff_len(&set[c.dc_tbl]); }
    if (sd.Se != 0 && !((seen >> (4 + c.ac_tbl)) & 1u)) { seen |= 1u << (4 + c.ac_tbl); dht += 17 + huff_len(&set[4 + c.ac_tbl]); }
  }
  if (dht) dht += 4;
  return dht + (sd.dri ? 6 : 0) + (2 + 2 + 1 + 2 * sd.ncomps + 3);       // emit_dri: FFDD 0004 xxxx (jcmarker.c)
}
// The layout of jpeg_search_progression's script (jcparam.c:733-852) as three kinds of groups per component set:
//   * an Al ladder: `nband` band scans coded at Al = 0, then per step a: `nrefine` refinement scans (Ah = a, Al = a-1)
//     followed by the `nband` band scans at Al = a;
//   * a split menu: the unsplit candidate (`width` scans) followed by 5 two-band candidates (2*width scans each, at
//     the split points 2, 8, 5, 12, 18 in that order).
// select_scans (jcmaster.c:773-962) walks them with the early exits below; every candidate is coded here, so only
// its DECISIONS are replayed, on the candidates' sizes.
struct AlLadder { int base, nband, nrefine, al_max;
  int refine(int a, int r) const { return base + nband + (nband + nrefine) * a + r; }            // refinement r of step a+1
  int band(int a, int b) const { return a == 0 ? base + b : refine(a - 1, nrefine) + b; } };
struct SplitMenu { int first, width;
  int scan(int idx, int w) const { return idx == 0 ? first + w : first + width + 2 * width * (idx - 1) + w; }
  int count(int idx) const { return idx == 0 ? width : 2 * width; } };

// cheapest point transform: total bytes of the bands at Al = a plus the refinement scans that restore the dropped bits;
// the search stops at the first step that does not improve (jcmaster.c:792-812, :879-903)
static int pick_al(const unsigned long *size, const AlLadder &L)
{
  unsigned long best = 0; int best_a = 0;
  for (int a = 0; a <= L.al_max; a++) {
    unsigned long cost = 0;
    for (int b = 0; b < L.nband; b++) cost += size[L.band(a, b)];
    for (int i = 0; i < a; i++) for (int r = 0; r < L.nrefine; r++) cost += size[L.refine(i, r)];
    if (a > 0 && cost >= best) break;
    best = cost; best_a = a;
  }
  return best_a;
}
// cheapest frequency split; candidates are visited in script order and the walk ends once the trend is settled:
// after the second split point if nothing beat "unsplit", after the third unless the second won, after the fourth
// unless it won itself (jcmaster.c:814-858, :905-941)
static int pick_split(const unsigned long *size, const SplitMenu &M)
{
  unsigned long best = 0; int best_idx = 0;
  for (int idx = 0; idx <= 5; idx++) {
    unsigned long cost = 0;
    for (int w = 0; w < M.count(idx); w++) cost += size[M.scan(idx, w)];
    if (idx == 0 || cost < best) { best = cost; best_idx = idx; }
    if ((idx == 2 && best_idx == 0) || (idx == 3 && best_idx != 2) || (idx == 4 && best_idx != 4)) break;
  }
  return best_idx;
}
static void select_scans_host(const Plan &pl, const b200jpeg_params *p, int num_scans, const unsigned long *scan_size,
                              std::vector<int> &copy, int &best_Al_luma_out, int &best_Al_chroma_out)
{
  const bool colour = num_scans > pl.n_luma;
  const AlLadder luma_al{1, 2, 1, 3}, chroma_al{pl.n_luma + 3, 4, 2, 2};
  const SplitMenu luma_split{pl.luma_split0, 1}, chroma_split{pl.chroma_split0, 2};
  const int al_y = pick_al(scan_size, luma_al), split_y = pick_split(scan_size, luma_split);
  const int al_c = colour ? pick_al(scan_size, chroma_al) : 0, split_c = colour ? pick_split(scan_size, chroma_split) : 0;
  // one interleaved chroma DC scan unless the two separate ones are smaller (jcmaster.c:871-877)
  const bool joint_dc = colour && scan_size[pl.n_luma] <= scan_size[pl.n_luma + 1] + scan_size[pl.n_luma + 2];
  // output order (jcmaster.c:943-1007... copy_buffer calls): DC, chroma DC, luma bands, the refinements only luma needs,
  // chroma bands, the refinements only chroma needs, then the shared refinement steps from coarse to fine
  copy.clear();
  copy.push_back(0);
  if (colour && p->dc_scan_opt_mode != 0) {
    if (joint_dc && p->dc_scan_opt_mode != 1) copy.push_back(pl.n_luma);
    else { copy.push_back(pl.n_luma + 1); copy.push_back(pl.n_luma + 2); }
  }
  const int al_shared = std::min(al_y, al_c);
  for (int w = 0; w < luma_split.count(split_y); w++) copy.push_back(luma_split.scan(split_y, w));
  for (int a = al_y - 1; a >= al_shared; a--) copy.push_back(luma_al.refine(a, 0));
  if (colour) {
    for (int w = 0; w < chroma_split.count(split_c); w++) copy.push_back(chroma_split.scan(split_c, w));
    for (int a = al_c - 1; a >= al_shared; a--) for (int r = 0; r < 2; r++) copy.push_back(chroma_al.refine(a, r));
  }
  for (int a = al_shared - 1; a >= 0; a--) {
    copy.push_back(luma_al.refine(a, 0));
    if (colour) for (int r = 0; r < 2; r++) copy.push_back(chroma_al.refine(a, r));
  }
  best_Al_luma_out = al_y; best_Al_chroma_out = al_c;
}

// Chunk k's pipeline has finished: lay out its files in pinned memory, write the
// markers (jcmarker.c) on the host and queue the copies of the entropy-coded
// bytes straight into place.  Returns 1 if an image overflowed its output buffer.
static int finish_chunk(b200jpeg_encoder *e, const ChunkIO &io, int k)
{
  Plan &pl = e->plan; const b200jpeg_params *p = &e->params;
  const int nscans = (int)pl.scans.size();
  CU(cudaEventSynchronize(e->ev_done[k]));
  const uint32_t *st = e->h_status.as<uint32_t>() + io.i0;
  bool overflow = false;
  for (int i = 0; i < io.n; i++) {
    if (st[i] & 2u) { set_error("DCT coefficient out of range (image %d)", io.i0 + i); return B200JPEG_ERR_BAD_DCT_COEF; }
    if (st[i] & 4u) overflow = true;
  }
  if (overflow) return 1;
  const HostHuff *ht = e->h_tabs.as<HostHuff>();
  const uint32_t *ss = e->h_scan_size.as<uint32_t>() + (size_t)io.i0 * nscans;
  const unsigned long long *pos = e->h_out_pos.as<unsigned long long>() + (size_t)io.i0 * (nscans + 1);    // [slot][n]
  std::vector<int> slot_of(nscans);
  for (size_t j = 0; j < pl.order.size(); j++) slot_of[pl.order[j]] = (int)j;
  std::vector<uint8_t> hdr; std::vector<size_t> hdr_end;
  std::vector<int> emit; std::vector<int> actual_al(nscans);
  std::vector<unsigned long> total(nscans);
  for (int i = 0; i < io.n; i++) {
    const int gi = io.i0 + i;
    const HostHuff *img_tabs = pl.optimize ? ht + (size_t)gi * nscans * HIST_SLOTS : nullptr;
    // which scans go into the file, in which order, with which Al
    emit.clear();
    for (int si = 0; si < nscans; si++) actual_al[si] = pl.scans[si].Al;
    if (pl.search) {
      const int *dev_al = e->h_best_al.as<int>() + (size_t)io.i0 * 2;
      int al_l = dev_al[i], al_c = nscans > pl.n_luma ? dev_al[io.n + i] : 0;
      for (int si = pl.luma_split0; si < pl.n_luma; si++) actual_al[si] = al_l;
      for (int si = pl.chroma_split0; si < nscans; si++) actual_al[si] = al_c;
      for (int si = 0; si < nscans; si++) total[si] = scan_header_bytes(pl, pl.scans[si], img_tabs + (size_t)si * HIST_SLOTS) + ss[(size_t)si * io.n + i];
      int hl = -1, hc = -1;
      select_scans_host(pl, p, nscans, total.data(), emit, hl, hc);
      if (hl != al_l || (nscans > pl.n_luma && hc != al_c)) { set_error("scan search: device and host disagree on the best Al (image %d: %d/%d vs %d/%d)", gi, al_l, al_c, hl, hc); return B200JPEG_ERR_CUDA; }
    } else for (int si = 0; si < nscans; si++) emit.push_back(si);
    hdr.clear(); hdr_end.assign(emit.size(), 0);
    Bytes o{hdr};
    write_file_header(p, o);
    if (e->copy_markers) {
      // cjpeg's copy of the source's saved markers right behind jpeg_start_compress (cjpeg.c:960-990): all but a JFIF
      // APP0 / Adobe APP14 where the file header above already holds the compressor's own
      const std::vector<uint8_t> &mk = (*e->copy_markers)[gi];
      for (size_t q = 0; q + 4 <= mk.size();) {
        const size_t len = 2 + ((size_t)mk[q + 2] << 8 | mk[q + 3]);
        const uint8_t *dat = mk.data() + q + 4; const size_t dl = len - 4;
        const bool dup = (p->write_JFIF_header && mk[q + 1] == 0xE0 && dl >= 5 && !memcmp(dat, "JFIF\0", 5)) ||
                         (p->write_Adobe_marker && mk[q + 1] == 0xEE && dl >= 5 && !memcmp(dat, "Adobe", 5));
        if (!dup) hdr.insert(hdr.end(), mk.begin() + q, mk.begin() + q + len);
        q += len;
      }
    }
    TblState ts;
    const HostHuff *fixed = pl.optimize ? nullptr : ht;
    for (int t = 0; t < 4; t++) { ts.dc[t] = fixed ? &fixed[t] : nullptr; ts.ac[t] = fixed ? &fixed[4 + t] : nullptr; ts.dc_sent[t] = ts.ac_sent[t] = false; }
    int last_ri = 0;
    size_t scan_bytes = 0;
    for (size_t k2 = 0; k2 < emit.size(); k2++) {
      const int si = emit[k2];
      ScanDesc sd = pl.scans[si];
      sd.Al = actual_al[si];
      if (pl.optimize) {
        uint32_t m = scan_slot_mask(pl, sd);
        const HostHuff *set = img_tabs + (size_t)si * HIST_SLOTS;
        for (int t = 0; t < 4; t++) {
          if (m & (1u << t)) { ts.dc[t] = &set[t]; ts.dc_sent[t] = false; }               // jpeg_gen_optimal_table clears sent_table (jchuff.c:1105)
          if (m & (1u << (4 + t))) { ts.ac[t] = &set[4 + t]; ts.ac_sent[t] = false; }
        }
      }
      if (k2 == 0) {
        // the image's own tables go into its DQT and decide its SOF0 / SOF1: the re-fitted ones under trellis_q_opt
        // (jcmaster.c:1014-1030), else those of its table set
        const uint16_t *qimg = pl.trellis && p->trellis_q_opt ? e->h_qimg.as<uint16_t>() + (size_t)gi * 256
                             : !e->img_set.empty() ? &e->qsets[(size_t)e->img_set[gi] * 256] : nullptr;
        if (qimg) {
          static thread_local b200jpeg_params pq;
          pq = *p; memcpy(pq.quant_tbl, qimg, 512);
          write_frame_header(&pq, pl.progressive, o);
        } else write_frame_header(p, pl.progressive, o);
      }
      if (pl.search) last_ri = sd.dri ? -1 : sd.ri;               // the candidate's header as it was buffered when it was coded
      write_scan_header(p, sd, ts, last_ri, (unsigned)sd.ri, o);
      hdr_end[k2] = hdr.size();
      scan_bytes += ss[(size_t)si * io.n + i];
    }
    const size_t total_file = hdr.size() + scan_bytes + 2;
    uint8_t *f = arena_alloc(e, total_file);
    if (!f) return B200JPEG_ERR_CUDA;
    const uint8_t *dimg = io.out + (size_t)i * e->out_cap_per_image;
    size_t w = 0, hprev = 0;
    for (size_t k2 = 0; k2 < emit.size(); k2++) {
      const int si = emit[k2];
      memcpy(f + w, hdr.data() + hprev, hdr_end[k2] - hprev); w += hdr_end[k2] - hprev; hprev = hdr_end[k2];
      size_t sz = ss[(size_t)si * io.n + i];
      if (sz) CU(cudaMemcpyAsync(f + w, dimg + pos[(size_t)slot_of[si] * io.n + i], sz, cudaMemcpyDeviceToHost, e->s_out));
      w += sz;
    }
    f[w++] = 0xFF; f[w++] = 0xD9;
    e->files[gi] = std::make_pair(f, w);
    e->last_scan_bytes += scan_bytes;
    e->max_image_scan_bytes = std::max(e->max_image_scan_bytes, scan_bytes);
    e->last_file_bytes += w;
  }
  return B200JPEG_OK;
}

static int choose_chunk(const b200jpeg_encoder *e, const Plan &pl, int n_images, bool host_pixels)
{
  // several kernels put (image, component) or the image index into gridDim.y / gridDim.z (limit 65535)
  const int grid_cap = 65535 / std::max(1, pl.g.nc);
  if (e->chunk_images_override > 0) return std::min(std::min(n_images, e->chunk_images_override), grid_cap);
  long long per = 0; for (int ci = 0; ci < pl.g.nc; ci++) per += pl.g.c[ci].blocks_per_image;
  // pixels already in HBM: no staging to overlap, so chunks only bound the arenas and give the two compute streams one
  // large chunk each to run against each other (131 images of 4K 4:2:0: two such arenas fit an 80 GB H100 beside a
  // resident batch of 256)
  static const long long resident_target = getenv("B200JPEG_RESIDENT_CHUNK_BLOCKS") ? atoll(getenv("B200JPEG_RESIDENT_CHUNK_BLOCKS")) : 25600000LL;
  if (!host_pixels) {
    long long c = std::min<long long>(std::min(n_images, grid_cap), std::max(1LL, resident_target / std::max(1LL, per)));
    // a batch that fits one chunk goes out as two, one per compute stream, when the halves stay large (6.4 M blocks, 33
    // images of 4K 4:2:0); smaller halves are not split: the 64 candidate scans' kernels of the library default profile
    // lose more by shrinking than the latency-bound table / layout launches gain by overlapping
    if (c >= n_images && e->n_streams > 1 && (long long)n_images * per >= 2 * 6400000LL) c = (n_images + 1) / 2;
    return (int)c;
  }
  // about 1.6 M blocks (8 images of 3840x2160 4:2:0) per chunk: large enough to fill
  // the 132 SMs several waves deep, small enough that staging the next chunk's
  // pixels overlaps this chunk's kernels.
  static const long long target = getenv("B200JPEG_CHUNK_BLOCKS") ? atoll(getenv("B200JPEG_CHUNK_BLOCKS")) : 1600000LL;
  long long c = std::max(1LL, target / std::max(1LL, per));
  // scan search: the 64 candidate scans make the device the slower side (1 ms per 4K image against 0.45 ms of staging) and
  // launch ~700 kernels per chunk, so chunks are four times larger, but a batch still goes out in at least two so that the
  // second half's staging hides behind the first half's kernels
  if (pl.search) c = std::max(1LL, std::min(4 * c, ((long long)n_images + 1) / 2));
  return (int)std::min<long long>(std::min(n_images, grid_cap), c);
}

// raw-data input (jpeg_write_raw_data): one plane per component instead of interleaved pixels
// pitch, stride in bytes; coefs: planes hold JBLOCK rows; xf (coefficients only, or nullptr): a lossless transform's
// mapping, the planes are then in the source's geometry
struct RawDesc { const uint8_t *plane[4]; size_t pitch[4], stride[4]; bool coefs; const b200jpeg_transform_info *xf; };

// The batch's quantization table sets: without per-image tables one set, the parameter block's; with them
// (qtables: [n_images][4][64], natural order, the slots quant_tbl_present names) the distinct ones, in order of first
// use, and every image's set.
static int collect_qsets(b200jpeg_encoder *e, const b200jpeg_params *p, const uint16_t *qtables, int n_images)
{
  e->qsets.assign(&p->quant_tbl[0][0], &p->quant_tbl[0][0] + 256);
  e->img_set.clear(); e->nsets = 1;
  if (!qtables) return B200JPEG_OK;
  for (int i = 0; i < n_images; i++)
    for (int t = 0; t < 4; t++) {
      if (!p->quant_tbl_present[t]) continue;
      for (int k = 0; k < 64; k++) {
        const unsigned v = qtables[((size_t)i * 4 + t) * 64 + k];
        if (v < 1 || v > 32767) { set_error("image %d: quantization table %d: entry %d is %u, outside 1..32767", i, t, k, v); return B200JPEG_ERR_PARAM; }
      }
    }
  e->qsets.clear(); e->img_set.resize(n_images);
  std::map<std::string, int> seen;
  std::vector<uint16_t> set(256);
  for (int i = 0; i < n_images; i++) {
    for (int t = 0; t < 4; t++)
      memcpy(&set[(size_t)t * 64], p->quant_tbl_present[t] ? qtables + ((size_t)i * 4 + t) * 64 : p->quant_tbl[t], 128);
    auto ins = seen.emplace(std::string(reinterpret_cast<const char *>(set.data()), 512), (int)seen.size());
    if (ins.second) e->qsets.insert(e->qsets.end(), set.begin(), set.end());
    e->img_set[i] = ins.first->second;
  }
  e->nsets = (int)seen.size();
  return B200JPEG_OK;
}

static int encode_common(b200jpeg_encoder *e, const b200jpeg_params *p, const void *pixels, int on_device,
                         size_t row_pitch, size_t image_stride, int n_images, bool device_only, const RawDesc *raw = nullptr,
                         const uint16_t *qtables = nullptr, const std::vector<std::vector<uint8_t>> *markers = nullptr)
{
  if (!e || !p || (!pixels && !raw) || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  e->copy_markers = markers;
  int rc = b200jpeg_validate(p);
  if (rc) return rc;
  // lossless mode: the block jpeg_start_compress works with (jcmaster.c:1072-1094); the plan and the markers follow it
  b200jpeg_params eff;
  if (is_lossless(p)) {
    if (raw) { set_error("%s input cannot be coded lossless (jcmaster.c:1076 clears raw_data_in)", raw->coefs ? "coefficient" : "raw-data"); return B200JPEG_ERR_PARAM; }
    if (qtables) { set_error("per-image quantization tables have no meaning in lossless mode"); return B200JPEG_ERR_PARAM; }
    lossless_start(p, &eff);
    p = &eff;
  }
  const size_t sample_bytes = p->data_precision > 8 ? 2 : 1;                       // 12- and 16-bit samples are uint16 (J12SAMPLE / J16SAMPLE)
  const size_t row_bytes = (size_t)p->image_width * p->input_components * sample_bytes;
  // per-image tables allow a zero image stride: every image reads the same input (a quality ladder)
  const bool shared_ok = qtables != nullptr;
  if (!raw) {
    if (row_pitch < row_bytes) { set_error("row_pitch smaller than a row"); return B200JPEG_ERR_PARAM; }
    if (n_images > 1 && !(shared_ok && image_stride == 0) && image_stride < row_pitch * (size_t)(p->image_height - 1) + row_bytes) { set_error("image_stride smaller than an image"); return B200JPEG_ERR_PARAM; }
  }
  if ((rc = collect_qsets(e, p, qtables, n_images))) return rc;
  CU(cudaSetDevice(e->device));
  e->params = *p; e->n = n_images;
  if ((rc = build_plan(p, row_pitch, image_stride, e->plan))) return rc;
  Plan &pl = e->plan;
  size_t raw_plane_bytes[4] = {0, 0, 0, 0}, raw_total[4] = {0, 0, 0, 0}, raw_off[4] = {0, 0, 0, 0}, raw_sum = 0;
  if (raw && raw->coefs) {
    // jpeg_write_coefficients: no forward stage, no trellis (jpeg_copy_critical_parameters turns it off, jctrans.c:103)
    Geom &g = pl.g;
    if (p->trellis_quant) { set_error("coefficient input: trellis quantization needs the unquantized coefficients (trellis_quant must be 0, as jpeg_copy_critical_parameters sets it)"); return B200JPEG_ERR_PARAM; }
    g.raw_in = 2;
    e->xform = CoefXform{};
    if (const b200jpeg_transform_info *t = raw->xf) {
      e->xform.transposed = t->transposed;
      for (int ci = 0; ci < g.nc; ci++) {
        e->xform.x_crop[ci] = t->x_crop_blocks[ci]; e->xform.y_crop[ci] = t->y_crop_blocks[ci];
        e->xform.x_mirror[ci] = t->x_mirror[ci]; e->xform.y_mirror[ci] = t->y_mirror[ci];
      }
    }
    for (int ci = 0; ci < g.nc; ci++) {
      const size_t rows = (size_t)(raw->xf ? raw->xf->src_hib[ci] : g.c[ci].hib), cols = (size_t)(raw->xf ? raw->xf->src_wib[ci] : g.c[ci].wib) * 128;
      if (!raw->plane[ci] || raw->pitch[ci] < cols || (n_images > 1 && !(shared_ok && raw->stride[ci] == 0) && raw->stride[ci] < raw->pitch[ci] * (rows - 1) + cols)) { set_error("coefficient plane %d: bad pointer, pitch or stride (needs %zu rows of %zu blocks)", ci, rows, cols / 128); return B200JPEG_ERR_PARAM; }
      raw_plane_bytes[ci] = raw->pitch[ci] * (rows - 1) + cols;
      raw_total[ci] = raw->stride[ci] * (size_t)(n_images - 1) + raw_plane_bytes[ci];
      raw_off[ci] = raw_sum; raw_sum += (raw_total[ci] + 255) & ~(size_t)255;
      g.plane_pitch[ci] = raw->pitch[ci]; g.plane_stride[ci] = raw->stride[ci];
    }
  } else if (raw) {
    Geom &g = pl.g;
    if (p->data_precision != 8) { set_error("raw-data input is 8-bit only on the device path"); return B200JPEG_ERR_UNSUPPORTED; }
    g.raw_in = 1;
    for (int ci = 0; ci < g.nc; ci++) {
      const size_t rows = (size_t)g.c[ci].hib * 8, cols = (size_t)g.c[ci].wib * 8;      // what compress_first_pass reads (jccoefct.c:262-353)
      if (!raw->plane[ci] || raw->pitch[ci] < cols || (n_images > 1 && !(shared_ok && raw->stride[ci] == 0) && raw->stride[ci] < raw->pitch[ci] * (rows - 1) + cols)) { set_error("raw-data plane %d: bad pointer, pitch or stride (needs %zu rows of %zu samples)", ci, rows, cols); return B200JPEG_ERR_PARAM; }
      raw_plane_bytes[ci] = raw->pitch[ci] * (rows - 1) + cols;
      raw_total[ci] = raw->stride[ci] * (size_t)(n_images - 1) + raw_plane_bytes[ci];
      raw_off[ci] = raw_sum; raw_sum += (raw_total[ci] + 255) & ~(size_t)255;
      g.plane_pitch[ci] = raw->pitch[ci]; g.plane_stride[ci] = raw->stride[ci];
    }
  }
  const int nscans = (int)pl.scans.size();
  const int C = choose_chunk(e, pl, n_images, !on_device);
  const int nchunks = (n_images + C - 1) / C;
  e->chunk = C;
  const size_t image_bytes = row_pitch * (size_t)(p->image_height - 1) + row_bytes;
  const size_t src_bytes = raw ? raw_sum : image_stride * (size_t)(n_images - 1) + image_bytes;
  while ((int)e->ev_in.size() < nchunks) { cudaEvent_t ev; CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); e->ev_in.push_back(ev); }
  while ((int)e->ev_done.size() < nchunks) { cudaEvent_t ev; CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); e->ev_done.push_back(ev); }
  if (!device_only) {
    if ((rc = e->h_status.reserve((size_t)n_images * 4))) return rc;
    if ((rc = e->h_out_pos.reserve((size_t)n_images * (nscans + 1) * 8))) return rc;
    if ((rc = e->h_best_al.reserve((size_t)n_images * 2 * 4))) return rc;
    if (p->trellis_quant && p->trellis_q_opt && (rc = e->h_qimg.reserve((size_t)n_images * 512))) return rc;
    if ((rc = e->h_scan_size.reserve((size_t)n_images * nscans * 4))) return rc;
    if ((rc = e->h_tabs.reserve((pl.optimize ? (size_t)n_images * nscans : 1) * HIST_SLOTS * sizeof(HostHuff)))) return rc;
  }
  Timer tm{e};
  const int nstreams = std::max(1, std::min(std::min(e->n_streams, MAX_ARENAS), nchunks));
  e->sc[0] = e->stream;
  // one incompressible batch does not enlarge the buffers for good: after two batches without growth whose largest
  // image would have fitted the initial size eight times over, fall back to it (batches that keep needing the room,
  // e.g. 12-bit noise at 15 MB per image, keep it; device-only runs never shrink: their sizes are not read back)
  {
    long long tb = 0; for (int ci = 0; ci < pl.g.nc; ci++) tb += pl.g.c[ci].blocks_per_image;
    if (pl.lossless) tb = (tb + 7) / 8;                      // the per-sample scale prepare_batch sizes the buffers with
    if (e->calm_batches >= 2 && !device_only && e->cap_factor > 0.25 && e->max_image_scan_bytes * 8 < (size_t)((double)tb * 64 * 0.25)) e->cap_factor = 0.25;
    if (!device_only) e->max_image_scan_bytes = 0;
  }
  bool grew = false;
  for (int attempt = 0; attempt < 6; attempt++) {
    tm.idx = 0;
    if ((rc = prepare_batch(e, n_images, C, !on_device, src_bytes, nstreams))) return rc;
    CU(cudaMemsetAsync(e->d_status.p, 0, (size_t)n_images * 4, e->stream));
    CU(cudaMemsetAsync(e->d_out_pos.p, 0, (size_t)n_images * (nscans + 1) * 8, e->stream));
    if (nstreams > 1) { CU(cudaEventRecord(e->ev_fork, e->stream)); for (int i = 1; i < nstreams; i++) CU(cudaStreamWaitEvent(e->sc[i], e->ev_fork, 0)); }
    // stage every chunk's pixels up front on the copy stream; chunk k's kernels wait only for chunk k
    const uint8_t *src_base = static_cast<const uint8_t *>(pixels);
    const uint8_t *plane_base[4] = {nullptr, nullptr, nullptr, nullptr};
    if (raw) for (int ci = 0; ci < pl.g.nc; ci++) plane_base[ci] = on_device ? raw->plane[ci] : e->d_src.as<uint8_t>() + raw_off[ci];
    if (!on_device) {
      for (int k = 0; k < nchunks; k++) {
        const int i0 = k * C, nk = std::min(C, n_images - i0);
        // input shared by every image (zero stride) is staged once, with the first chunk
        if (raw) {
          for (int ci = 0; ci < pl.g.nc; ci++) {
            if (k > 0 && raw->stride[ci] == 0) continue;
            const size_t off = (size_t)i0 * raw->stride[ci], bytes = raw->stride[ci] * (size_t)(nk - 1) + raw_plane_bytes[ci];
            CU(cudaMemcpyAsync(e->d_src.as<uint8_t>() + raw_off[ci] + off, raw->plane[ci] + off, bytes, cudaMemcpyHostToDevice, e->s_in));
          }
        } else if (k == 0 || image_stride != 0) {
          const size_t off = (size_t)i0 * image_stride, bytes = image_stride * (size_t)(nk - 1) + image_bytes;
          CU(cudaMemcpyAsync(e->d_src.as<uint8_t>() + off, static_cast<const uint8_t *>(pixels) + off, bytes, cudaMemcpyHostToDevice, e->s_in));
        }
        CU(cudaEventRecord(e->ev_in[k], e->s_in));
      }
      src_base = e->d_src.as<uint8_t>();
    }
    if (!device_only) {
      e->files.assign(n_images, std::make_pair((uint8_t *)nullptr, (size_t)0));
      size_t expect = e->last_file_bytes ? (size_t)((double)e->last_file_bytes / std::max(1, (int)e->files.size()) * 1.3 * n_images)
                                         : (size_t)n_images * ((size_t)p->image_width * p->image_height * p->num_components / 6 + 65536);
      e->last_scan_bytes = 0; e->last_file_bytes = 0;
      arena_reset(e, expect + (size_t)n_images * 4096);
    }
    rc = B200JPEG_OK;
    ChunkIO prev{}; bool have_prev = false;
    for (int k = 0; k < nchunks && rc == B200JPEG_OK; k++) {
      ChunkIO io;
      io.i0 = k * C; io.n = std::min(C, n_images - io.i0);
      io.slot = k % nstreams;
      io.src = raw ? nullptr : src_base + (size_t)io.i0 * image_stride;
      for (int ci = 0; ci < 4; ci++) io.plane[ci] = raw && plane_base[ci] ? plane_base[ci] + (size_t)io.i0 * raw->stride[ci] : nullptr;
      io.out = e->d_out.as<uint8_t>() + (size_t)io.i0 * e->out_cap_per_image;
      io.out_pos = e->d_out_pos.as<unsigned long long>() + (size_t)io.i0 * (nscans + 1);
      io.status = e->d_status.as<uint32_t>() + io.i0;
      io.scan_size = e->d_scan_size.as<uint32_t>() + (size_t)io.i0 * nscans;
      io.tabs_scan = e->d_tabs_scan.as<DevHuff>() + (size_t)io.i0 * nscans * HIST_SLOTS;
      io.best_al = e->d_best_al_all.as<int>() + (size_t)io.i0 * 2;
      io.qimg = e->d_qimg_all.as<uint16_t>() + (size_t)io.i0 * 256;
      io.qset = e->img_set.empty() ? nullptr : e->d_qset.as<int>() + io.i0;
      if (!on_device) { tm.s = e->sc[io.slot]; tm.mark("h2d_wait"); CU(cudaStreamWaitEvent(e->sc[io.slot], e->ev_in[k], 0)); }
      if ((rc = run_pipeline(e, io, tm))) break;
      if (!device_only) {
        if ((rc = queue_meta(e, io, k))) break;
        if (have_prev) rc = finish_chunk(e, prev, k - 1);
        prev = io; have_prev = true;
      }
    }
    if (rc == B200JPEG_OK && !device_only && have_prev) rc = finish_chunk(e, prev, nchunks - 1);
    // the second stream joins the caller-visible one
    for (int i = 1; i < nstreams; i++) { cudaEventRecord(e->ev_join, e->sc[i]); cudaStreamWaitEvent(e->stream, e->ev_join, 0); }   // (a wait takes the record in front of it)
    if (rc < 0) { cudaStreamSynchronize(e->stream); cudaStreamSynchronize(e->s_in); cudaStreamSynchronize(e->s_out); return rc; }
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->s_in));
    CU(cudaStreamSynchronize(e->s_out));
    if (device_only) {
      // the overflow flag still matters for a meaningful timing run
      if ((rc = e->h_status.reserve((size_t)n_images * 4))) return rc;
      CU(cudaMemcpy(e->h_status.p, e->d_status.p, (size_t)n_images * 4, cudaMemcpyDeviceToHost));
      bool ovf = false; for (int i = 0; i < n_images; i++) if (e->h_status.as<uint32_t>()[i] & 4u) ovf = true;
      rc = ovf ? 1 : B200JPEG_OK;
    }
    if (rc != 1) break;
    e->cap_factor *= 4.0;          // entropy-coded data did not fit: grow and rerun
    grew = true;
  }
  e->calm_batches = grew ? 0 : e->calm_batches + 1;
  if (rc == 1) { set_error("output does not fit even after growing buffers"); return B200JPEG_ERR_BUFFER; }
  if (rc) return rc;
  collect_stage_times(e, tm.idx);
  return B200JPEG_OK;
}

// tj3EncodeYUVPlanes8 on the device (b200jpeg_encode_yuv_batch)
static int encode_yuv(b200jpeg_encoder *e, const b200jpeg_params *p, const void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride,
                      uint8_t *const *planes, int planes_on_device, const size_t *plane_pitch, const size_t *plane_stride, int n_images)
{
  if (!e || !p || !pixels || !planes || !plane_pitch || !plane_stride || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  int rc = b200jpeg_validate(p);
  if (rc) return rc;
  if (is_lossless(p)) { set_error("YUV encoding has no lossless mode"); return B200JPEG_ERR_PARAM; }
  if (p->data_precision != 8) { set_error("YUV encoding takes 8-bit samples only (data precision %d)", p->data_precision); return B200JPEG_ERR_PARAM; }
  if (p->smoothing_factor) { set_error("YUV encoding with input smoothing is not on the device path"); return B200JPEG_ERR_UNSUPPORTED; }
  if ((rc = build_plan(p, row_pitch, image_stride, e->plan))) return rc;
  const Geom &g = e->plan.g;
  const bool pow2 = (g.hmax == 1 || g.hmax == 2 || g.hmax == 4) && (g.vmax == 1 || g.vmax == 2 || g.vmax == 4);
  const bool layout = (g.nc == 1 || g.nc == 3) && g.c[0].h == g.hmax && g.c[0].v == g.vmax &&
                      (g.nc == 1 || (g.c[1].h == 1 && g.c[1].v == 1 && g.c[2].h == 1 && g.c[2].v == 1));
  if (!pow2 || !layout) { set_error("YUV encoding: the device path takes component 0 at sampling factors of 1, 2 or 4 and 1x1 components 1 and 2 (the TJSAMP_* layouts)"); return B200JPEG_ERR_UNSUPPORTED; }
  const size_t row_bytes = (size_t)g.W * g.in_comps, image_bytes = row_pitch * (size_t)(g.H - 1) + row_bytes;
  if (row_pitch < row_bytes) { set_error("row_pitch smaller than a row"); return B200JPEG_ERR_PARAM; }
  if (n_images > 1 && image_stride < image_bytes) { set_error("image_stride smaller than an image"); return B200JPEG_ERR_PARAM; }
  YuvOut out; memset(&out, 0, sizeof out);
  size_t plane_bytes[3] = {0, 0, 0};
  for (int ci = 0; ci < g.nc; ci++) {
    b200jpeg_yuv_plane_dims(p, ci, &out.pw[ci], &out.ph[ci]);
    plane_bytes[ci] = plane_pitch[ci] * (size_t)(out.ph[ci] - 1) + out.pw[ci];
    if (!planes[ci] || plane_pitch[ci] < (size_t)out.pw[ci] || (n_images > 1 && plane_stride[ci] < plane_bytes[ci])) {
      set_error("YUV plane %d: bad pointer, pitch or stride (needs %d rows of %d samples)", ci, out.ph[ci], out.pw[ci]); return B200JPEG_ERR_PARAM;
    }
  }
  CU(cudaSetDevice(e->device));
  e->n = 0; e->files.clear();                    // no JPEG files from this call
  Timer tm{e};
  if (pixels_on_device && planes_on_device) {
    // launches only, on the encoder's (or the caller's) stream: stage times are read when asked for
    for (int ci = 0; ci < g.nc; ci++) { out.p[ci] = planes[ci]; out.pitch[ci] = plane_pitch[ci]; out.stride[ci] = plane_stride[ci]; }
    for (int i0 = 0; i0 < n_images; i0 += 65535) {
      const int nk = std::min(65535, n_images - i0);
      YuvOut o = out;
      for (int ci = 0; ci < g.nc; ci++) o.p[ci] += (size_t)i0 * plane_stride[ci];
      tm.mark("encode_yuv");
      launch_encode_yuv(g, static_cast<const uint8_t *>(pixels) + (size_t)i0 * image_stride, o, nk, e->stream);
      tm.mark("end");
    }
    CU(cudaGetLastError());
    e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
    e->pending_marks = tm.idx;
    return B200JPEG_OK;
  }
  // host input and / or output: chunks of about 128 MB of pixels rotating over three staging slots, so that chunk k+1's
  // host->device copy (s_in) and chunk k-1's device->host copy (s_out) overlap chunk k's kernel (e->stream)
  int C = e->chunk_images_override > 0 ? e->chunk_images_override : (int)std::max<size_t>(1, ((size_t)128 << 20) / std::max(image_bytes, image_stride));
  C = std::min(std::min(C, n_images), 65535);
  const int nchunks = (n_images + C - 1) / C, NSLOT = 3;
  e->chunk = C;
  const size_t in_slot = pixels_on_device ? 0 : ((image_stride * (size_t)(C - 1) + image_bytes + 255) & ~(size_t)255);
  size_t out_off[3] = {0, 0, 0}, out_slot = 0;
  if (!planes_on_device)
    for (int ci = 0; ci < g.nc; ci++) { out_off[ci] = out_slot; out_slot += ((size_t)out.pw[ci] * out.ph[ci] * C + 255) & ~(size_t)255; }
  if (in_slot && (rc = e->d_src.reserve(in_slot * NSLOT))) return rc;
  if (out_slot && (rc = e->d_yuv.reserve(out_slot * NSLOT))) return rc;
  while ((int)e->ev_in.size() < nchunks) { cudaEvent_t ev; CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); e->ev_in.push_back(ev); }
  while ((int)e->ev_done.size() < nchunks) { cudaEvent_t ev; CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)); e->ev_done.push_back(ev); }
  std::vector<cudaEvent_t> ev_read(nchunks);     // chunk k's read-back done: its output slot may be reused
  for (int k = 0; k < nchunks; k++) { CU(cudaEventCreateWithFlags(&ev_read[k], cudaEventDisableTiming)); }
  rc = B200JPEG_OK;
  for (int k = 0; k < nchunks && rc == B200JPEG_OK; k++) {
    const int i0 = k * C, nk = std::min(C, n_images - i0), slot = k % NSLOT;
    const uint8_t *src = static_cast<const uint8_t *>(pixels) + (size_t)i0 * image_stride;
    if (!pixels_on_device) {
      uint8_t *dst = e->d_src.as<uint8_t>() + slot * in_slot;
      if (k >= NSLOT) cudaStreamWaitEvent(e->s_in, e->ev_done[k - NSLOT], 0);        // the slot's previous kernel has read it
      tm.s = e->s_in; tm.mark("h2d");
      if (cudaMemcpyAsync(dst, src, image_stride * (size_t)(nk - 1) + image_bytes, cudaMemcpyHostToDevice, e->s_in) != cudaSuccess) { set_error("host->device copy failed"); rc = B200JPEG_ERR_CUDA; break; }
      tm.mark("end");
      cudaEventRecord(e->ev_in[k], e->s_in);
      cudaStreamWaitEvent(e->stream, e->ev_in[k], 0);
      src = dst;
    }
    YuvOut o = out;
    for (int ci = 0; ci < g.nc; ci++) {
      if (planes_on_device) { o.p[ci] = planes[ci] + (size_t)i0 * plane_stride[ci]; o.pitch[ci] = plane_pitch[ci]; o.stride[ci] = plane_stride[ci]; }
      else { o.p[ci] = e->d_yuv.as<uint8_t>() + slot * out_slot + out_off[ci]; o.pitch[ci] = out.pw[ci]; o.stride[ci] = (size_t)out.pw[ci] * out.ph[ci]; }
    }
    if (!planes_on_device && k >= NSLOT) cudaStreamWaitEvent(e->stream, ev_read[k - NSLOT], 0);   // the slot's previous read-back is done
    tm.s = e->stream; tm.mark("encode_yuv");
    launch_encode_yuv(g, src, o, nk, e->stream);
    tm.mark("end");
    if (cudaGetLastError() != cudaSuccess) { set_error("k_encode_yuv launch failed"); rc = B200JPEG_ERR_CUDA; break; }
    cudaEventRecord(e->ev_done[k], e->stream);
    if (!planes_on_device) {
      cudaStreamWaitEvent(e->s_out, e->ev_done[k], 0);
      tm.s = e->s_out; tm.mark("d2h");
      for (int i = 0; i < nk && rc == B200JPEG_OK; i++)
        for (int ci = 0; ci < g.nc; ci++)
          if (cudaMemcpy2DAsync(planes[ci] + (size_t)(i0 + i) * plane_stride[ci], plane_pitch[ci], o.p[ci] + (size_t)i * o.stride[ci], o.pitch[ci],
                                out.pw[ci], out.ph[ci], cudaMemcpyDeviceToHost, e->s_out) != cudaSuccess) { set_error("device->host copy failed"); rc = B200JPEG_ERR_CUDA; break; }
      tm.mark("end");
      cudaEventRecord(ev_read[k], e->s_out);
    }
  }
  cudaStreamSynchronize(e->s_in); cudaStreamSynchronize(e->stream); cudaStreamSynchronize(e->s_out);
  for (cudaEvent_t ev : ev_read) cudaEventDestroy(ev);
  if (rc) return rc;
  CU(cudaGetLastError());
  collect_stage_times(e, tm.idx);
  return B200JPEG_OK;
}

}  // namespace b200

namespace b200 {

static uint32_t *dec_words_alloc(void *ctx, size_t words)
{
  b200jpeg_encoder *e = static_cast<b200jpeg_encoder *>(ctx);
  return e->h_dec_words.reserve(words * 4) ? nullptr : e->h_dec_words.as<uint32_t>();
}

static const char *const kDecStages[6] = {"dec_h2d", "dec_sync", "dec_fix", "dec_scan", "dec_write", "dec_dc"};

// the decode stages of the last decode, appended to the stage times
static void add_decode_stage_times(b200jpeg_encoder *e)
{
  for (int k = 0; k < 6; k++) {
    float ms = 0.f; cudaEventElapsedTime(&ms, e->dec_ev[k], e->dec_ev[k + 1]);
    e->stage_names.push_back(kDecStages[k]); e->stage_ms.push_back(ms); e->stage_calls.push_back(1);
  }
}

// Entropy decode of n sequential files into e->d_dec_planes (jpeg_read_coefficients for the batch).
// first: the batch index of files[0], for the messages.
static int decode_files(b200jpeg_encoder *e, const uint8_t *const *files, const size_t *sizes, int n, int first = 0)
{
  if (!e || !files || !sizes || n <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  CU(cudaSetDevice(e->device));
  DecBatch &b = e->dec;
  int rc = build_decode_batch(files, sizes, n, b, dec_words_alloc, e, first);
  if (rc) return rc;
  size_t total = 0;
  for (int c = 0; c < b.nc; c++) { e->dec_plane_off[c] = total; total += ((size_t)n * b.wib[c] * b.hib[c] * 128 + 255) & ~(size_t)255; }
  const long long ntiles = (b.nsub + 1023) / 1024;
  if ((rc = e->d_dec_words.reserve(b.nwords * 4 + 16)) || (rc = e->d_dec_segs.reserve(b.segs.size() * sizeof(DecSeg))) ||
      (rc = e->d_dec_scans.reserve(b.scans.size() * sizeof(DecScan))) || (rc = e->d_dec_tabs.reserve(b.tabs.size() * sizeof(DecTable))) ||
      (rc = e->d_dec_out.reserve(sizeof(DecOut))) || (rc = e->d_dec_rec.reserve((size_t)b.nsub * sizeof(DecRec))) ||
      (rc = e->d_dec_pre.reserve((size_t)b.nsub * 4)) || (rc = e->d_dec_tsum.reserve((size_t)ntiles * 8)) ||
      (rc = e->d_dec_dcd.reserve((size_t)b.nblocks * 4 + 4)) || (rc = e->d_dec_planes.reserve(total)) ||
      (rc = e->d_dec_stat.reserve((size_t)n * 4 + 24)) || (rc = e->h_dec_stat.reserve((size_t)n * 4 + 24)))
    return rc;
  for (cudaEvent_t &ev : e->dec_ev) if (!ev) CU(cudaEventCreate(&ev));
  DecOut o; memset(&o, 0, sizeof o);
  for (int c = 0; c < b.nc; c++) { o.plane[c] = reinterpret_cast<int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]); o.wib[c] = b.wib[c]; o.hib[c] = b.hib[c]; }
  cudaStream_t s = e->stream;
  uint8_t *stat = e->d_dec_stat.as<uint8_t>();          // [n] status words, max rounds (int), resynchronised subsequences (u64)
  const size_t rounds_off = ((size_t)n * 4 + 7) & ~(size_t)7, stat_bytes = rounds_off + 16;
  CU(cudaEventRecord(e->dec_ev[0], s));
  CU(cudaMemcpyAsync(e->d_dec_words.p, e->h_dec_words.p, b.nwords * 4, cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_segs.p, b.segs.data(), b.segs.size() * sizeof(DecSeg), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_scans.p, b.scans.data(), b.scans.size() * sizeof(DecScan), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_tabs.p, b.tabs.data(), b.tabs.size() * sizeof(DecTable), cudaMemcpyHostToDevice, s));
  CU(cudaMemcpyAsync(e->d_dec_out.p, &o, sizeof o, cudaMemcpyHostToDevice, s));
  CU(cudaMemsetAsync(e->d_dec_planes.p, 0, total, s));
  CU(cudaMemsetAsync(stat, 0, stat_bytes, s));
  launch_decode(e->d_dec_words.as<uint32_t>(), e->d_dec_segs.as<DecSeg>(), (int)b.segs.size(), e->d_dec_scans.as<DecScan>(), e->d_dec_tabs.as<DecTable>(), b.nsub,
                e->d_dec_rec.as<DecRec>(), e->d_dec_pre.as<uint32_t>(), e->d_dec_tsum.as<unsigned long long>(), e->d_dec_dcd.as<int>(), e->d_dec_out.as<DecOut>(),
                reinterpret_cast<uint32_t *>(stat), reinterpret_cast<int *>(stat + rounds_off), reinterpret_cast<unsigned long long *>(stat + rounds_off + 8),
                e->dec_ev + 1, s);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(e->h_dec_stat.p, stat, stat_bytes, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  const uint8_t *hs = e->h_dec_stat.as<uint8_t>();
  e->dec_rounds = *reinterpret_cast<const int *>(hs + rounds_off);
  e->dec_redone = (long long)*reinterpret_cast<const unsigned long long *>(hs + rounds_off + 8);
  for (int i = 0; i < n; i++)
    if (reinterpret_cast<const uint32_t *>(hs)[i]) { set_error("image %d: corrupt entropy-coded data (an invalid Huffman code, or too few bits for a segment's MCUs)", first + i); return B200JPEG_ERR_BAD_SOURCE; }
  return B200JPEG_OK;
}

// a transform description must be the one b200jpeg_transform_setup left beside p
static int check_xform(const b200jpeg_params *p, const b200jpeg_transform_info *t)
{
  if (t->num_components != p->num_components || t->output_width != p->image_width || t->output_height != p->image_height) {
    set_error("the transform description (%d components, %dx%d) does not match the parameter block (%d components, %dx%d): run b200jpeg_transform_setup on it",
              t->num_components, t->output_width, t->output_height, p->num_components, p->image_width, p->image_height);
    return B200JPEG_ERR_PARAM;
  }
  return B200JPEG_OK;
}

// transpose_critical_parameters (transupp.c:1858-1871) on every slot of n table sets ([n][4][64], natural order)
static void transpose_qsets(uint16_t *q, int n)
{
  for (size_t s = 0; s < (size_t)n * B200JPEG_NUM_QUANT_TBLS; s++)
    for (int i = 0; i < 8; i++)
      for (int j = 0; j < i; j++) std::swap(q[s * 64 + i * 8 + j], q[s * 64 + j * 8 + i]);
}

static int encode_coefs_xform(b200jpeg_encoder *enc, const b200jpeg_params *p, const b200jpeg_transform_info *t, const int16_t *const *planes, int planes_on_device,
                              const size_t *row_pitch_blocks, const size_t *image_stride_blocks, const uint16_t *qtables, int n_images)
{
  if (!enc || !p || !t || !planes || !row_pitch_blocks || !image_stride_blocks || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  int rc = check_xform(p, t);
  if (rc) return rc;
  RawDesc rd; memset(&rd, 0, sizeof rd); rd.coefs = true; rd.xf = t;
  for (int ci = 0; ci < p->num_components && ci < 4; ci++) {
    rd.plane[ci] = reinterpret_cast<const uint8_t *>(planes[ci]); rd.pitch[ci] = row_pitch_blocks[ci] * 128; rd.stride[ci] = image_stride_blocks[ci] * 128;
  }
  std::vector<uint16_t> qt;
  if (qtables) {
    qt.assign(qtables, qtables + (size_t)n_images * B200JPEG_NUM_QUANT_TBLS * 64);
    if (t->transposed) transpose_qsets(qt.data(), n_images);
  }
  b200jpeg_params q = *p;                 // as b200jpeg_encode_batch_coefs
  q.overshoot_deringing = 0; q.smoothing_factor = 0; q.dct_method = B200JPEG_DCT_ISLOW;
  return encode_common(enc, &q, nullptr, planes_on_device, 0, 0, n_images, false, &rd, qtables ? qt.data() : nullptr);
}

// jpegtran from file bytes (b200jpeg_transcode_batch, and with a transform b200jpeg_transcode_batch_transform)
static int transcode_files(b200jpeg_encoder *e, const b200jpeg_params *p, const b200jpeg_transform_info *t, const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (!e || !p) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  e->dec.want_markers = false;
  int rc = decode_files(e, files, sizes, n_images);
  if (rc) return rc;
  const DecBatch &b = e->dec;
  // -grayscale keeps the first component of a 3-component source; every other destination has the source's components
  const bool comps_ok = p->num_components == b.nc || (t && t->force_grayscale && p->num_components == 1);
  if (!comps_ok) { set_error("the parameter block has %d components, the sources %d", p->num_components, b.nc); return B200JPEG_ERR_PARAM; }
  if (t) {
    for (int c = 0; c < p->num_components; c++)
      if (t->src_wib[c] != b.wib[c] || t->src_hib[c] != b.hib[c]) { set_error("the sources' component %d has %dx%d blocks, the transform description %dx%d", c, b.wib[c], b.hib[c], t->src_wib[c], t->src_hib[c]); return B200JPEG_ERR_PARAM; }
  }
  // each image's quantization tables: what its components latched, in the slots p assigns them; in the source's
  // orientation (p's are transposed back), encode_coefs_xform transposes them with the blocks
  std::vector<uint16_t> qt((size_t)n_images * B200JPEG_NUM_QUANT_TBLS * 64);
  for (int i = 0; i < n_images; i++) {
    uint16_t *q = qt.data() + (size_t)i * B200JPEG_NUM_QUANT_TBLS * 64;
    memcpy(q, p->quant_tbl, sizeof p->quant_tbl);
    if (t && t->transposed) transpose_qsets(q, 1);
    for (int c = 0; c < p->num_components; c++) {
      const int slot = p->comp_info[c].quant_tbl_no;
      if (slot < 0 || slot >= B200JPEG_NUM_QUANT_TBLS || !b.info[i].comp_quant_present[c]) { set_error("image %d: Quantization table 0x%02x was not defined", i, slot); return B200JPEG_ERR_PARAM; }
      memcpy(q + slot * 64, b.info[i].comp_quant[c], 128);
    }
  }
  int16_t *planes[4]; size_t pitch[4], stride[4];
  for (int c = 0; c < 4; c++) {
    planes[c] = c < b.nc ? reinterpret_cast<int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]) : nullptr;
    pitch[c] = c < b.nc ? (size_t)b.wib[c] : 0; stride[c] = c < b.nc ? (size_t)b.wib[c] * b.hib[c] : 0;
  }
  rc = t ? encode_coefs_xform(e, p, t, planes, 1, pitch, stride, qt.data(), n_images)
         : b200jpeg_encode_batch_coefs_qtables(e, p, planes, 1, pitch, stride, qt.data(), n_images);
  if (rc) return rc;
  add_decode_stage_times(e);
  return B200JPEG_OK;
}

// A source b200jpeg_decompress_batch takes: sequential, 8-bit, gray or three components with component 0 at the
// largest factors (1 or 2 each way) over 1x1 chroma; everything else is refused, never approximated.
static int check_decompress_source(const b200jpeg_source_info &s, int i)
{
  const char *why = nullptr;
  if (s.sof == 0xC2) why = "progressive (SOF2) source: only sequential files are decoded to pixels";
  else if (s.data_precision != 8) why = "12-bit source: only 8-bit files are decoded to pixels";
  else if (s.num_components != 1 && s.num_components != 3) why = "4-component (CMYK / YCCK) source: only gray and 3-component files are decoded to pixels";
  else if (s.num_components == 3 && (s.h_samp_factor[0] > 2 || s.v_samp_factor[0] > 2 || s.h_samp_factor[1] != 1 || s.v_samp_factor[1] != 1 ||
                                     s.h_samp_factor[2] != 1 || s.v_samp_factor[2] != 1))
    why = "sampling layout other than 4:4:4, 4:2:2, 4:4:0 or 4:2:0 (the reference's int_upsample and 2:1 non-fancy cases are not on the device)";
  if (why) { set_error("image %d: %s", i, why); return B200JPEG_ERR_UNSUPPORTED; }
  for (int c = 0; c < s.num_components; c++)
    if (!s.comp_quant_present[c]) { set_error("image %d: Quantization table 0x%02x was not defined", i, s.quant_tbl_no[c]); return B200JPEG_ERR_BAD_SOURCE; }
  return B200JPEG_OK;
}

// the multiplier tables of jddctmgr.c start_pass for the ifast and float IDCTs, from one quantization table
static const int kAanScales[64] = {
  16384, 22725, 21407, 19266, 16384, 12873,  8867,  4520, 22725, 31521, 29692, 26722, 22725, 17855, 12299,  6270,
  21407, 29692, 27969, 25172, 21407, 16819, 11585,  5906, 19266, 26722, 25172, 22654, 19266, 15137, 10426,  5315,
  16384, 22725, 21407, 19266, 16384, 12873,  8867,  4520, 12873, 17855, 16819, 15137, 12873, 10114,  6967,  3552,
   8867, 12299, 11585, 10426,  8867,  6967,  4799,  2446,  4520,  6270,  5906,  5315,  4520,  3552,  2446,  1247};
static const double kAanScaleFactor[8] = {1.0, 1.387039845, 1.306562965, 1.175875602, 1.0, 0.785694958, 0.541196100, 0.275899379};
static void method_table(int method, const uint16_t *q, uint32_t *out)
{
  for (int i = 0; i < 64; i++) {
    if (method == B200JPEG_DCT_IFAST) {
      const int v = (int)(((long long)q[i] * kAanScales[i] + 2048) >> 12);                 // DESCALE(.., 14 - IFAST_SCALE_BITS)
      memcpy(&out[i], &v, 4);
    } else {
      const float f = (float)((double)q[i] * kAanScaleFactor[i >> 3] * kAanScaleFactor[i & 7]);
      memcpy(&out[i], &f, 4);
    }
  }
}

// the IDCT and upsampling / colour conversion stages of one decoded chunk (e->dec) for a non-default plan: each
// needed component through the IDCT of its DCT_scaled_size into a plane of wib * size samples a row, then
// k_upsample_opts into the pixels.  qt / mt: host staging for the tables.
static int idct_upsample_opts(b200jpeg_encoder *e, const DecPlan &plan, int nk, uint8_t *pix, size_t row_pitch, size_t image_stride,
                              std::vector<uint16_t> &qt, std::vector<uint32_t> &mt)
{
  const DecBatch &b = e->dec;
  const int nc = b.nc;
  cudaStream_t s = e->stream;
  size_t off[4] = {0, 0, 0, 0}, total = 0;
  bool need_mt = false;
  for (int c = 0; c < nc; c++) {
    if (!plan.needed[c]) continue;
    off[c] = total; total += ((size_t)nk * b.hib[c] * b.wib[c] * plan.ssize[c] * plan.ssize[c] + 255) & ~(size_t)255;
    need_mt |= plan.ssize[c] == 8 && plan.method != B200JPEG_DCT_ISLOW;
  }
  int rc;
  if ((rc = e->d_dec_samples.reserve(total)) || (rc = e->d_dec_quant.reserve((size_t)nk * nc * 128)) ||
      (need_mt && (rc = e->d_dec_mtab.reserve((size_t)nk * nc * 256)))) return rc;
  qt.resize((size_t)nk * nc * 64);
  for (int i = 0; i < nk; i++)
    for (int c = 0; c < nc; c++) memcpy(&qt[((size_t)i * nc + c) * 64], b.info[i].comp_quant[c], 128);
  CU(cudaMemcpyAsync(e->d_dec_quant.p, qt.data(), qt.size() * 2, cudaMemcpyHostToDevice, s));
  if (need_mt) {
    mt.resize((size_t)nk * nc * 64);
    for (size_t t = 0; t < (size_t)nk * nc; t++) method_table(plan.method, &qt[t * 64], &mt[t * 64]);
    CU(cudaMemcpyAsync(e->d_dec_mtab.p, mt.data(), mt.size() * 4, cudaMemcpyHostToDevice, s));
  }
  CU(cudaEventRecord(e->pix_ev[0], s));
  UpsOpt u;
  memset(&u, 0, sizeof u);
  for (int c = 0; c < nc; c++) {
    if (!plan.needed[c]) continue;
    const int sz = plan.ssize[c];
    uint8_t *dst = e->d_dec_samples.as<uint8_t>() + off[c];
    const bool by_method = sz == 8 && plan.method != B200JPEG_DCT_ISLOW;
    const void *tab = by_method ? static_cast<const void *>(e->d_dec_mtab.as<uint32_t>() + c * 64) : static_cast<const void *>(e->d_dec_quant.as<uint16_t>() + c * 64);
    launch_idct_opts(sz, plan.method, reinterpret_cast<const int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]), tab, nc * 64, dst, b.wib[c], b.hib[c], nk, s);
    if (c < 3) {
      u.plane[c] = dst; u.pitch[c] = b.wib[c] * sz; u.stride[c] = (long long)b.hib[c] * sz * u.pitch[c];
      u.dw[c] = plan.dw[c]; u.dh[c] = plan.dh[c]; u.hr[c] = plan.hr[c]; u.vr[c] = plan.vr[c]; u.fancy[c] = plan.fancy[c];
    }
  }
  CU(cudaEventRecord(e->pix_ev[1], s));
  u.nin = plan.nin; u.conv = plan.conv; u.ps = plan.ps;
  for (int k = 0; k < 4; k++) u.off[k] = plan.off[k];
  launch_upsample_opts(u, pix, row_pitch, image_stride, plan.out_w, plan.out_h, nk, s);
  CU(cudaEventRecord(e->pix_ev[2], s));
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(s));
  for (int k = 0; k < 6; k++) { float ms = 0.f; cudaEventElapsedTime(&ms, e->dec_ev[k], e->dec_ev[k + 1]); e->dec_ms[k] += ms; }
  for (int k = 0; k < 2; k++) { float ms = 0.f; cudaEventElapsedTime(&ms, e->pix_ev[k], e->pix_ev[k + 1]); e->dec_ms[6 + k] += ms; }
  return B200JPEG_OK;
}

// jpeg_read_scanlines for a batch of files: entropy decode, IDCT and upsampling / colour conversion chunk by chunk
// (the coefficient and sample planes are one chunk's), into pixels on the device.
// opts: the decompress object's options (nullptr: its defaults); options that give what the defaults give take the
// default route.
static int decompress_files(b200jpeg_encoder *e, const uint8_t *const *files, const size_t *sizes, int n, uint8_t *pix, size_t row_pitch, size_t image_stride,
                            bool want_markers, const b200jpeg_decompress_options *opts = nullptr)
{
  // every refusal comes before any device work
  b200jpeg_source_info s0;
  {
    static thread_local b200jpeg_source_info s;
    for (int i = 0; i < n; i++) {
      if (!files[i]) { set_error("image %d: no file", i); return B200JPEG_ERR_PARAM; }
      int rc = b200jpeg_parse_source(files[i], sizes[i], &s);
      if (rc) { std::string m = b200jpeg_last_error(); set_error("image %d: %s", i, m.c_str()); return rc; }
      if ((rc = check_decompress_source(s, i))) return rc;
      if (i == 0) s0 = s;
      bool same = s.image_width == s0.image_width && s.image_height == s0.image_height && s.num_components == s0.num_components;
      for (int c = 0; same && c < s.num_components; c++) same = s.h_samp_factor[c] == s0.h_samp_factor[c] && s.v_samp_factor[c] == s0.v_samp_factor[c];
      if (same && s.num_components == 3) same = (s.jpeg_color_space == B200JPEG_CS_RGB) == (s0.jpeg_color_space == B200JPEG_CS_RGB);
      if (!same) { set_error("image %d: geometry (size, components, sampling, colour space) differs from image 0", i); return B200JPEG_ERR_PARAM; }
    }
  }
  const int W = s0.image_width, H = s0.image_height, nc = s0.num_components;
  const int hx = nc == 3 ? s0.h_samp_factor[0] : 1, vx = nc == 3 ? s0.v_samp_factor[0] : 1;
  DecPlan plan;
  if (opts) { int rc = plan_decompress(s0, *opts, plan); if (rc) return rc; }
  const bool def = plan.is_default;
  const int OW = def ? W : plan.out_w, OH = def ? H : plan.out_h, onc = def ? nc : plan.out_nc;
  if (row_pitch < (size_t)OW * onc || (n > 1 && image_stride < row_pitch * (size_t)(OH - 1) + (size_t)OW * onc)) { set_error("row_pitch or image_stride smaller than the decoded image (%dx%d, %d components)", OW, OH, onc); return B200JPEG_ERR_PARAM; }
  CU(cudaSetDevice(e->device));
  for (cudaEvent_t &ev : e->pix_ev) if (!ev) CU(cudaEventCreate(&ev));
  for (float &m : e->dec_ms) m = 0.f;
  e->dec.want_markers = want_markers;
  if (want_markers) e->dec_markers.assign(n, std::vector<uint8_t>());
  // chunks of about 1.6 M blocks (8 images of 3840x2160 4:2:0, 300 MB of coefficient and sample planes)
  long long per = 0;
  for (int c = 0; c < nc; c++) per += (long long)div_up((long long)W * s0.h_samp_factor[c], (nc == 3 ? hx : s0.h_samp_factor[0]) * 8) * div_up((long long)H * s0.v_samp_factor[c], (nc == 3 ? vx : s0.v_samp_factor[0]) * 8);
  const int C = std::min(n, e->chunk_images_override > 0 ? e->chunk_images_override : (int)std::max(1LL, 1600000LL / std::max(1LL, per)));
  cudaStream_t s = e->stream;
  std::vector<uint16_t> qt;
  std::vector<uint32_t> mt;
  for (int i0 = 0; i0 < n; i0 += C) {
    const int nk = std::min(C, n - i0);
    int rc = decode_files(e, files + i0, sizes + i0, nk, i0);
    if (rc) return rc;
    const DecBatch &b = e->dec;
    if (want_markers) for (int i = 0; i < nk; i++) e->dec_markers[i0 + i].swap(e->dec.markers[i]);
    if (!def) { if ((rc = idct_upsample_opts(e, plan, nk, pix + (size_t)i0 * image_stride, row_pitch, image_stride, qt, mt))) return rc; continue; }
    size_t off[4] = {0, 0, 0, 0}, total = 0;
    for (int c = 0; c < nc; c++) { off[c] = total; total += ((size_t)nk * b.hib[c] * b.wib[c] * 64 + 255) & ~(size_t)255; }
    if ((rc = e->d_dec_samples.reserve(total)) || (rc = e->d_dec_quant.reserve((size_t)nk * nc * 128))) return rc;
    qt.resize((size_t)nk * nc * 64);
    for (int i = 0; i < nk; i++)
      for (int c = 0; c < nc; c++) memcpy(&qt[((size_t)i * nc + c) * 64], b.info[i].comp_quant[c], 128);
    CU(cudaMemcpyAsync(e->d_dec_quant.p, qt.data(), qt.size() * 2, cudaMemcpyHostToDevice, s));
    CU(cudaEventRecord(e->pix_ev[0], s));
    const uint8_t *planes[4] = {nullptr, nullptr, nullptr, nullptr}; int pitch[4] = {0, 0, 0, 0}; long long stride[4] = {0, 0, 0, 0};
    for (int c = 0; c < nc; c++) {
      uint8_t *dst = e->d_dec_samples.as<uint8_t>() + off[c];
      launch_idct_islow(reinterpret_cast<const int16_t *>(e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c]), e->d_dec_quant.as<uint16_t>() + c * 64, nc * 64,
                        dst, b.wib[c], b.hib[c], nk, s);
      planes[c] = dst; pitch[c] = b.wib[c] * 8; stride[c] = (long long)b.hib[c] * 8 * pitch[c];
    }
    CU(cudaEventRecord(e->pix_ev[1], s));
    const int dw = div_up(W, hx), dh = div_up(H, vx);                    // downsampled_width / _height of the chroma (jdmaster.c)
    if (launch_upsample_color(hx, vx, nc, planes, pitch, stride, dw, dh, nc == 3 && s0.jpeg_color_space != B200JPEG_CS_RGB,
                              pix + (size_t)i0 * image_stride, row_pitch, image_stride, W, H, nk, s)) { set_error("no upsampling kernel for %dx%d sampling of %d components", hx, vx, nc); return B200JPEG_ERR_UNSUPPORTED; }
    CU(cudaEventRecord(e->pix_ev[2], s));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(s));
    for (int k = 0; k < 6; k++) { float ms = 0.f; cudaEventElapsedTime(&ms, e->dec_ev[k], e->dec_ev[k + 1]); e->dec_ms[k] += ms; }
    for (int k = 0; k < 2; k++) { float ms = 0.f; cudaEventElapsedTime(&ms, e->pix_ev[k], e->pix_ev[k + 1]); e->dec_ms[6 + k] += ms; }
  }
  return B200JPEG_OK;
}

// the stages of the last decompress, appended to the stage times
static void add_decompress_stage_times(b200jpeg_encoder *e)
{
  static const char *const extra[2] = {"idct", "upsample_color"};
  for (int k = 0; k < 8; k++) { e->stage_names.push_back(k < 6 ? kDecStages[k] : extra[k - 6]); e->stage_ms.push_back(e->dec_ms[k]); e->stage_calls.push_back(1); }
}

// b200jpeg_decompress_batch (opts nullptr) and b200jpeg_decompress_batch_opts
static int decompress_batch(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const uint8_t *const *files, const size_t *sizes, int n_images,
                            void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride)
{
  if (!e || !files || !sizes || !pixels || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  uint8_t *dst = static_cast<uint8_t *>(pixels);
  size_t dp = row_pitch, ds = image_stride;
  if (!pixels_on_device) {
    // decode into a buffer of the batch's size on the device, then copy the rows out
    b200jpeg_source_info *s = new b200jpeg_source_info;
    int rc = b200jpeg_parse_source(files[0], files[0] ? sizes[0] : 0, s);
    int ow = 0, oh = 0, ocs = 0, onc = 0;
    if (!rc) rc = opts ? b200jpeg_decompress_output_opts(s, opts, &ow, &oh, &ocs, &onc) : b200jpeg_decompress_output(s, &ow, &oh, &ocs, &onc);
    const size_t row = rc ? 0 : (size_t)ow * onc, rows = rc ? 0 : (size_t)oh;
    delete s;
    if (rc) { std::string m = b200jpeg_last_error(); set_error("image 0: %s", m.c_str()); return rc; }
    if (row_pitch < row || (n_images > 1 && image_stride < row_pitch * (rows - 1) + row)) { set_error("row_pitch or image_stride smaller than the decoded image"); return B200JPEG_ERR_PARAM; }
    dp = (row + 3) & ~(size_t)3; ds = dp * rows;
    CU(cudaSetDevice(e->device));
    if ((rc = e->d_dec_pixels.reserve(ds * (size_t)n_images))) return rc;
    dst = e->d_dec_pixels.as<uint8_t>();
    rc = decompress_files(e, files, sizes, n_images, dst, dp, ds, false, opts);
    if (rc) return rc;
    for (int i = 0; i < n_images; i++)
      CU(cudaMemcpy2DAsync(static_cast<uint8_t *>(pixels) + (size_t)i * image_stride, row_pitch, dst + (size_t)i * ds, dp, row, rows, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
  } else {
    int rc = decompress_files(e, files, sizes, n_images, dst, dp, ds, false, opts);
    if (rc) return rc;
  }
  e->pending_marks = 0;
  e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
  add_decompress_stage_times(e);
  return B200JPEG_OK;
}

// b200jpeg_recompress_batch (opts nullptr) and b200jpeg_recompress_batch_opts
static int recompress_batch(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const b200jpeg_params *p, const uint8_t *const *files,
                            const size_t *sizes, int n_images)
{
  if (!e || !p || !files || !sizes || n_images <= 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  int rc = b200jpeg_validate(p);
  if (rc) return rc;
  if (p->data_precision != 8) { set_error("the sources decode to 8-bit samples, the parameter block has data_precision %d", p->data_precision); return B200JPEG_ERR_PARAM; }
  const size_t pitch = ((size_t)p->image_width * p->input_components + 3) & ~(size_t)3, stride = pitch * (size_t)p->image_height;
  {
    b200jpeg_source_info *s = new b200jpeg_source_info;
    int w = 0, h = 0, cs = 0, nc = 0;
    rc = files[0] ? b200jpeg_parse_source(files[0], sizes[0], s) : B200JPEG_OK;
    if (!rc && files[0]) rc = opts ? b200jpeg_decompress_output_opts(s, opts, &w, &h, &cs, &nc) : b200jpeg_decompress_output(s, &w, &h, &cs, &nc);
    delete s;
    if (rc) { std::string m = b200jpeg_last_error(); set_error("image 0: %s", m.c_str()); return rc; }
    if (files[0] && (w != p->image_width || h != p->image_height || cs != p->in_color_space || nc != p->input_components)) {
      set_error("the sources decode to %dx%d pixels of %d samples in colour space %d, the parameter block describes %dx%d of %d in %d (see b200jpeg_decompress_output)",
                w, h, nc, cs, p->image_width, p->image_height, p->input_components, p->in_color_space);
      return B200JPEG_ERR_PARAM;
    }
  }
  CU(cudaSetDevice(e->device));
  if ((rc = e->d_dec_pixels.reserve(stride * (size_t)n_images))) return rc;
  if ((rc = decompress_files(e, files, sizes, n_images, e->d_dec_pixels.as<uint8_t>(), pitch, stride, true, opts))) return rc;
  if ((rc = encode_common(e, p, e->d_dec_pixels.p, 1, pitch, stride, n_images, false, nullptr, nullptr, &e->dec_markers))) return rc;
  add_decompress_stage_times(e);
  return B200JPEG_OK;
}

}  // namespace b200

extern "C" {

int b200jpeg_decompress_batch(b200jpeg_encoder *e, const uint8_t *const *files, const size_t *sizes, int n_images,
                              void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride)
{
  return b200::decompress_batch(e, nullptr, files, sizes, n_images, pixels, pixels_on_device, row_pitch, image_stride);
}

int b200jpeg_decompress_batch_opts(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const uint8_t *const *files,
                                   const size_t *sizes, int n_images, void *pixels, int pixels_on_device, size_t row_pitch, size_t image_stride)
{
  if (!opts) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return b200::decompress_batch(e, opts, files, sizes, n_images, pixels, pixels_on_device, row_pitch, image_stride);
}

int b200jpeg_recompress_batch(b200jpeg_encoder *e, const b200jpeg_params *p, const uint8_t *const *files, const size_t *sizes, int n_images)
{
  return b200::recompress_batch(e, nullptr, p, files, sizes, n_images);
}

int b200jpeg_recompress_batch_opts(b200jpeg_encoder *e, const b200jpeg_decompress_options *opts, const b200jpeg_params *p,
                                   const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (!opts) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return b200::recompress_batch(e, opts, p, files, sizes, n_images);
}

int b200jpeg_decode_coefs_batch(b200jpeg_encoder *e, const uint8_t *const *files, const size_t *sizes, int n_images,
                                int16_t *const *planes, int planes_on_device, const size_t *row_pitch_blocks, const size_t *image_stride_blocks)
{
  if (!e || !planes || !row_pitch_blocks || !image_stride_blocks) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  e->dec.want_markers = false;
  int rc = decode_files(e, files, sizes, n_images);
  if (rc) return rc;
  const DecBatch &b = e->dec;
  for (int c = 0; c < b.nc; c++) {
    const size_t wib = (size_t)b.wib[c], hib = (size_t)b.hib[c];
    if (!planes[c] || row_pitch_blocks[c] < wib || (n_images > 1 && image_stride_blocks[c] < row_pitch_blocks[c] * (hib - 1) + wib)) {
      set_error("coefficient plane %d: bad pointer, pitch or stride (needs %zu rows of %zu blocks)", c, hib, wib); return B200JPEG_ERR_PARAM;
    }
    const uint8_t *src = e->d_dec_planes.as<uint8_t>() + e->dec_plane_off[c];
    for (int i = 0; i < n_images; i++)
      CU(cudaMemcpy2DAsync(reinterpret_cast<uint8_t *>(planes[c]) + (size_t)i * image_stride_blocks[c] * 128, row_pitch_blocks[c] * 128,
                           src + (size_t)i * hib * wib * 128, wib * 128, wib * 128, hib, planes_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, e->stream));
  }
  CU(cudaStreamSynchronize(e->stream));
  e->pending_marks = 0;
  e->stage_names.clear(); e->stage_ms.clear(); e->stage_calls.clear();
  add_decode_stage_times(e);
  return B200JPEG_OK;
}

int b200jpeg_transcode_batch(b200jpeg_encoder *e, const b200jpeg_params *p, const uint8_t *const *files, const size_t *sizes, int n_images)
{
  return b200::transcode_files(e, p, nullptr, files, sizes, n_images);
}

int b200jpeg_transcode_batch_transform(b200jpeg_encoder *e, const b200jpeg_params *p, const b200jpeg_transform_info *t,
                                       const uint8_t *const *files, const size_t *sizes, int n_images)
{
  if (!t) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return b200::transcode_files(e, p, t, files, sizes, n_images);
}

int b200jpeg_last_decode_sync(const b200jpeg_encoder *e, int *max_cta_rounds, long long *resync_subsequences)
{
  if (!e) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  if (max_cta_rounds) *max_cta_rounds = e->dec_rounds;
  if (resync_subsequences) *resync_subsequences = e->dec_redone;
  return B200JPEG_OK;
}

int b200jpeg_encoder_create(b200jpeg_encoder **enc, int device)
{
  if (!enc) return B200JPEG_ERR_PARAM;
  *enc = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0) { set_error("no usable CUDA device (%s); libb200jpeg has no CPU fallback", e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"); return B200JPEG_ERR_NO_DEVICE; }
  if (device < 0 || device >= count) { set_error("device %d out of range (0..%d)", device, count - 1); return B200JPEG_ERR_PARAM; }
  CU(cudaSetDevice(device));
  b200jpeg_encoder *o = new b200jpeg_encoder();
  o->device = device;
  if ((e = cudaDeviceGetAttribute(&o->sms, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) { set_error("cudaDeviceGetAttribute failed: %s", cudaGetErrorString(e)); delete o; return B200JPEG_ERR_CUDA; }
  cudaError_t e2 = cudaStreamCreateWithFlags(&o->stream, cudaStreamNonBlocking);
  if (e2 == cudaSuccess) e2 = cudaStreamCreateWithFlags(&o->s_in, cudaStreamNonBlocking);
  if (e2 == cudaSuccess) e2 = cudaStreamCreateWithFlags(&o->s_out, cudaStreamNonBlocking);
  for (int i = 1; i < MAX_ARENAS; i++) if (e2 == cudaSuccess) e2 = cudaStreamCreateWithFlags(&o->sc[i], cudaStreamNonBlocking);
  if (e2 == cudaSuccess) e2 = cudaEventCreateWithFlags(&o->ev_fork, cudaEventDisableTiming);
  if (e2 == cudaSuccess) e2 = cudaEventCreateWithFlags(&o->ev_join, cudaEventDisableTiming);
  o->sc[0] = o->stream;
  if (e2 != cudaSuccess) { set_error("cudaStreamCreate failed: %s", cudaGetErrorString(e2)); delete o; return B200JPEG_ERR_CUDA; }
  o->launches_at_create = g_kernel_launches;
  const char *dbg = getenv("B200JPEG_KEEP_PLAIN");
  o->keep_plain = dbg && dbg[0] == '1';
  const char *ch = getenv("B200JPEG_CHUNK_IMAGES");
  if (ch) o->chunk_images_override = atoi(ch);
  const char *ns = getenv("B200JPEG_STREAMS");
  if (ns) o->n_streams = std::max(1, std::min(atoi(ns), MAX_ARENAS));
  *enc = o;
  return B200JPEG_OK;
}

void b200jpeg_encoder_destroy(b200jpeg_encoder *e)
{
  if (!e) return;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  if (e->s_in) cudaStreamSynchronize(e->s_in);
  if (e->s_out) cudaStreamSynchronize(e->s_out);
  for (int i = 1; i < MAX_ARENAS; i++) if (e->sc[i]) cudaStreamSynchronize(e->sc[i]);
  DevBuf *db[] = {&e->d_src, &e->d_yuv, &e->d_tabs_scan, &e->d_tabs_fixed, &e->d_status, &e->d_out_pos, &e->d_scan_size, &e->d_out, &e->d_qt, &e->d_tc, &e->d_best_al_all, &e->d_qimg_all, &e->d_qset};
  for (DevBuf *b : db) b->release();
  for (int i = 0; i < MAX_ARENAS; i++) e->ar[i].release();
  DevBuf *dd[] = {&e->d_dec_words, &e->d_dec_segs, &e->d_dec_scans, &e->d_dec_tabs, &e->d_dec_out, &e->d_dec_rec, &e->d_dec_pre, &e->d_dec_tsum, &e->d_dec_dcd, &e->d_dec_planes, &e->d_dec_stat,
                  &e->d_dec_samples, &e->d_dec_quant, &e->d_dec_pixels, &e->d_dec_mtab};
  for (DevBuf *b : dd) b->release();
  for (cudaEvent_t ev : e->dec_ev) if (ev) cudaEventDestroy(ev);
  for (cudaEvent_t ev : e->pix_ev) if (ev) cudaEventDestroy(ev);
  PinBuf *pb[] = {&e->h_qt, &e->h_tc, &e->h_fixed, &e->h_status, &e->h_out_pos, &e->h_scan_size, &e->h_tabs, &e->h_stage, &e->h_best_al, &e->h_qinit, &e->h_qimg, &e->h_qset, &e->h_dec_words, &e->h_dec_stat};
  for (PinBuf *b : pb) b->release();
  for (PinBuf &b : e->file_arenas) b.release();
  for (cudaEvent_t ev : e->ev) cudaEventDestroy(ev);
  for (cudaEvent_t ev : e->ev_in) cudaEventDestroy(ev);
  for (cudaEvent_t ev : e->ev_done) cudaEventDestroy(ev);
  if (e->own_stream) cudaStreamDestroy(e->stream);
  if (e->s_in) cudaStreamDestroy(e->s_in);
  if (e->s_out) cudaStreamDestroy(e->s_out);
  for (int i = 1; i < MAX_ARENAS; i++) if (e->sc[i]) cudaStreamDestroy(e->sc[i]);
  if (e->ev_fork) cudaEventDestroy(e->ev_fork);
  if (e->ev_join) cudaEventDestroy(e->ev_join);
  delete e;
}

int b200jpeg_encoder_set_streams(b200jpeg_encoder *e, int n_streams)
{
  if (!e || n_streams < 1 || n_streams > MAX_ARENAS) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  e->n_streams = n_streams;
  return B200JPEG_OK;
}

int b200jpeg_last_chunk_images(const b200jpeg_encoder *e) { return e ? e->chunk : 0; }

int b200jpeg_encoder_set_chunk_images(b200jpeg_encoder *e, int images_per_chunk)
{
  if (!e || images_per_chunk < 0) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  e->chunk_images_override = images_per_chunk;
  return B200JPEG_OK;
}

int b200jpeg_encoder_set_stream(b200jpeg_encoder *e, void *cuda_stream)
{
  if (!e) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  CU(cudaSetDevice(e->device));
  CU(cudaStreamSynchronize(e->stream));
  if (e->own_stream) cudaStreamDestroy(e->stream);
  e->stream = static_cast<cudaStream_t>(cuda_stream);
  e->sc[0] = e->stream;
  e->own_stream = false;
  return B200JPEG_OK;
}

int b200jpeg_encode_batch(b200jpeg_encoder *enc, const b200jpeg_params *p, const void *pixels, int pixels_on_device,
                          size_t row_pitch, size_t image_stride, int n_images)
{
  return encode_common(enc, p, pixels, pixels_on_device, row_pitch, image_stride, n_images, false);
}
int b200jpeg_encode_yuv_batch(b200jpeg_encoder *enc, const b200jpeg_params *p, const void *pixels, int pixels_on_device,
                              size_t row_pitch, size_t image_stride, uint8_t *const *planes, int planes_on_device,
                              const size_t *plane_pitch, const size_t *plane_stride, int n_images)
{
  return encode_yuv(enc, p, pixels, pixels_on_device, row_pitch, image_stride, planes, planes_on_device, plane_pitch, plane_stride, n_images);
}
int b200jpeg_encode_batch_device_only(b200jpeg_encoder *enc, const b200jpeg_params *p, const void *pixels_device,
                                      size_t row_pitch, size_t image_stride, int n_images)
{
  return encode_common(enc, p, pixels_device, 1, row_pitch, image_stride, n_images, true);
}

int b200jpeg_encode_batch_raw(b200jpeg_encoder *enc, const b200jpeg_params *p, const uint8_t *const *planes, int planes_on_device,
                              const size_t *row_pitch, const size_t *image_stride, int n_images)
{
  if (!enc || !p || !planes || !row_pitch || !image_stride) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  RawDesc rd; memset(&rd, 0, sizeof rd);
  for (int ci = 0; ci < p->num_components && ci < 4; ci++) { rd.plane[ci] = planes[ci]; rd.pitch[ci] = row_pitch[ci]; rd.stride[ci] = image_stride[ci]; }
  return encode_common(enc, p, nullptr, planes_on_device, 0, 0, n_images, false, &rd);
}

int b200jpeg_encode_batch_coefs(b200jpeg_encoder *enc, const b200jpeg_params *p, const int16_t *const *planes, int planes_on_device,
                                const size_t *row_pitch_blocks, const size_t *image_stride_blocks, int n_images)
{
  if (!enc || !p || !planes || !row_pitch_blocks || !image_stride_blocks) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  RawDesc rd; memset(&rd, 0, sizeof rd); rd.coefs = true;
  for (int ci = 0; ci < p->num_components && ci < 4; ci++) {
    rd.plane[ci] = reinterpret_cast<const uint8_t *>(planes[ci]); rd.pitch[ci] = row_pitch_blocks[ci] * 128; rd.stride[ci] = image_stride_blocks[ci] * 128;
  }
  // the switches of the forward stage have no meaning on this path (and must not trip its 12-bit rules: jpegtran's
  // object still carries the profile's overshoot_deringing = TRUE)
  b200jpeg_params q = *p;
  q.overshoot_deringing = 0; q.smoothing_factor = 0; q.dct_method = B200JPEG_DCT_ISLOW;
  return encode_common(enc, &q, nullptr, planes_on_device, 0, 0, n_images, false, &rd);
}

int b200jpeg_encode_batch_qtables(b200jpeg_encoder *enc, const b200jpeg_params *p, const void *pixels, int pixels_on_device,
                                  size_t row_pitch, size_t image_stride, const uint16_t *qtables, int n_images)
{
  if (!qtables) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  return encode_common(enc, p, pixels, pixels_on_device, row_pitch, image_stride, n_images, false, nullptr, qtables);
}

int b200jpeg_encode_batch_raw_qtables(b200jpeg_encoder *enc, const b200jpeg_params *p, const uint8_t *const *planes, int planes_on_device,
                                      const size_t *row_pitch, const size_t *image_stride, const uint16_t *qtables, int n_images)
{
  if (!enc || !p || !planes || !row_pitch || !image_stride || !qtables) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  RawDesc rd; memset(&rd, 0, sizeof rd);
  for (int ci = 0; ci < p->num_components && ci < 4; ci++) { rd.plane[ci] = planes[ci]; rd.pitch[ci] = row_pitch[ci]; rd.stride[ci] = image_stride[ci]; }
  return encode_common(enc, p, nullptr, planes_on_device, 0, 0, n_images, false, &rd, qtables);
}

int b200jpeg_encode_batch_coefs_qtables(b200jpeg_encoder *enc, const b200jpeg_params *p, const int16_t *const *planes, int planes_on_device,
                                        const size_t *row_pitch_blocks, const size_t *image_stride_blocks, const uint16_t *qtables, int n_images)
{
  if (!enc || !p || !planes || !row_pitch_blocks || !image_stride_blocks || !qtables) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  RawDesc rd; memset(&rd, 0, sizeof rd); rd.coefs = true;
  for (int ci = 0; ci < p->num_components && ci < 4; ci++) {
    rd.plane[ci] = reinterpret_cast<const uint8_t *>(planes[ci]); rd.pitch[ci] = row_pitch_blocks[ci] * 128; rd.stride[ci] = image_stride_blocks[ci] * 128;
  }
  b200jpeg_params q = *p;                 // as b200jpeg_encode_batch_coefs
  q.overshoot_deringing = 0; q.smoothing_factor = 0; q.dct_method = B200JPEG_DCT_ISLOW;
  return encode_common(enc, &q, nullptr, planes_on_device, 0, 0, n_images, false, &rd, qtables);
}

int b200jpeg_encode_batch_coefs_transform(b200jpeg_encoder *enc, const b200jpeg_params *p, const b200jpeg_transform_info *t,
                                          const int16_t *const *planes, int planes_on_device,
                                          const size_t *row_pitch_blocks, const size_t *image_stride_blocks, const uint16_t *qtables, int n_images)
{
  return b200::encode_coefs_xform(enc, p, t, planes, planes_on_device, row_pitch_blocks, image_stride_blocks, qtables, n_images);
}

int b200jpeg_get_output(b200jpeg_encoder *e, int i, const uint8_t **data, size_t *size)
{
  if (!e || i < 0 || i >= (int)e->files.size()) { set_error("no such output"); return B200JPEG_ERR_PARAM; }
  if (!e->files[i].first) { set_error("no such output"); return B200JPEG_ERR_STATE; }
  if (data) *data = e->files[i].first;
  if (size) *size = e->files[i].second;
  return B200JPEG_OK;
}
size_t b200jpeg_last_scan_bytes(const b200jpeg_encoder *e) { return e ? e->last_scan_bytes : 0; }
unsigned long long b200jpeg_kernel_launches(const b200jpeg_encoder *e) { return e ? g_kernel_launches - e->launches_at_create : 0; }
int b200jpeg_last_stage_times(const b200jpeg_encoder *e, const char **names, float *ms, int max)
{
  if (!e) return 0;
  if (e->pending_marks) collect_stage_times(const_cast<b200jpeg_encoder *>(e), e->pending_marks);
  int n = (int)e->stage_ms.size();
  for (int i = 0; i < n && i < max; i++) { if (names) names[i] = e->stage_names[i]; if (ms) ms[i] = e->stage_ms[i]; }
  return n < max ? n : max;
}

long b200jpeg_debug_get_coefs(b200jpeg_encoder *e, int image, int component, int plane, int16_t *dst, size_t dst_blocks,
                              int *width_in_blocks, int *height_in_blocks)
{
  if (!e || image < 0 || image >= e->n || component < 0 || component >= e->plan.g.nc) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  // intermediates are kept for the LAST chunk of the batch only (the arenas are per chunk)
  if (image < e->last_chunk_i0 || image >= e->last_chunk_i0 + e->last_chunk_n) { set_error("image %d is not in the last chunk [%d,%d) of the batch", image, e->last_chunk_i0, e->last_chunk_i0 + e->last_chunk_n); return B200JPEG_ERR_STATE; }
  image -= e->last_chunk_i0;
  const CompGeom &c = e->plan.g.c[component];
  if (width_in_blocks) *width_in_blocks = c.wpad;
  if (height_in_blocks) *height_in_blocks = c.hpad;
  size_t nb = (size_t)c.blocks_per_image;
  if (!dst) return (long)nb;
  if (dst_blocks < nb) { set_error("buffer too small"); return B200JPEG_ERR_BUFFER; }
  Arena &A = e->ar[e->last_chunk_slot];
  DevBuf *src = plane == 0 ? &A.d_coef[component] : plane == 1 ? &A.d_raw[component] : &A.d_plain[component];
  if (plane == 2 && !(e->keep_plain && e->plan.trellis)) src = &A.d_coef[component];
  if (!src->p) { set_error("plane not available"); return B200JPEG_ERR_STATE; }
  std::vector<int16_t> tmp(nb * 64);
  CU(cudaSetDevice(e->device));
  CU(cudaMemcpy(tmp.data(), src->as<int16_t>() + (size_t)image * nb * 64, nb * 128, cudaMemcpyDeviceToHost));
  for (size_t b = 0; b < nb; b++) for (int k = 0; k < 64; k++) dst[b * 64 + kZigzag[k]] = tmp[b * 64 + k];   // zigzag -> natural
  return (long)nb;
}

int b200jpeg_debug_get_huff(b200jpeg_encoder *e, int image, int scan, int is_ac, int tbl_no, b200jpeg_huff_tbl *out)
{
  if (!e || !out || image < 0 || image >= e->n || tbl_no < 0 || tbl_no > 3) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  const int nscans = (int)e->plan.scans.size();
  DevHuff h;
  CU(cudaSetDevice(e->device));
  if (scan < 0) {          // scan = -1-ci : the trellis-phase tables of component ci
    int ci = -1 - scan;
    if (ci >= e->plan.g.nc) { set_error("bad component"); return B200JPEG_ERR_PARAM; }
    if (image < e->last_chunk_i0 || image >= e->last_chunk_i0 + e->last_chunk_n) { set_error("image %d is not in the last chunk of the batch", image); return B200JPEG_ERR_STATE; }
    CU(cudaMemcpy(&h, e->ar[e->last_chunk_slot].d_tabs_trellis.as<DevHuff>() + ((size_t)(image - e->last_chunk_i0) * e->plan.g.nc + ci) * HIST_SLOTS + (is_ac ? 4 : 0) + tbl_no, sizeof h, cudaMemcpyDeviceToHost));
  } else {
    if (scan >= nscans) { set_error("bad scan"); return B200JPEG_ERR_PARAM; }
    if (e->plan.optimize) CU(cudaMemcpy(&h, e->d_tabs_scan.as<DevHuff>() + ((size_t)image * nscans + scan) * HIST_SLOTS + (is_ac ? 4 : 0) + tbl_no, sizeof h, cudaMemcpyDeviceToHost));
    else CU(cudaMemcpy(&h, e->d_tabs_fixed.as<DevHuff>() + (is_ac ? 4 : 0) + tbl_no, sizeof h, cudaMemcpyDeviceToHost));
  }
  memset(out, 0, sizeof *out);
  memcpy(out->bits, h.bits, 17); memcpy(out->huffval, h.huffval, 256); out->present = 1;
  return B200JPEG_OK;
}

// ---- streaming shim: jpeg_start_compress / jpeg_write_scanlines / jpeg_finish_compress ----
int b200jpeg_start_compress(b200jpeg_encoder *e, const b200jpeg_params *p)
{
  if (!e || !p) { set_error("bad argument"); return B200JPEG_ERR_PARAM; }
  if (e->st_state != 0) { set_error("Improper call to JPEG library in state %d", 100 + e->st_state); return B200JPEG_ERR_STATE; }   // JERR_BAD_STATE
  int rc = b200jpeg_validate(p);
  if (rc) return rc;
  size_t bytes = (size_t)p->image_width * p->input_components * p->image_height * (p->data_precision > 8 ? 2 : 1);
  if ((rc = e->h_stage.reserve(bytes))) return rc;
  e->st_params = *p; e->st_state = 1; e->st_next_row = 0;
  return B200JPEG_OK;
}
int b200jpeg_write_scanlines(b200jpeg_encoder *e, const uint8_t *const *scanlines, int num_lines)
{
  if (!e || e->st_state != 1) { set_error("Improper call to JPEG library in state %d", e ? 100 + e->st_state : -1); return B200JPEG_ERR_STATE; }
  const b200jpeg_params &p = e->st_params;
  size_t rowbytes = (size_t)p.image_width * p.input_components * (p.data_precision > 8 ? 2 : 1);      // 12-bit rows are J12SAMPLE = short (jpeg12_write_scanlines)
  int left = p.image_height - e->st_next_row;            // extra rows are ignored (jcapistd.c:120-123)
  if (num_lines > left) num_lines = left;
  for (int i = 0; i < num_lines; i++) memcpy(e->h_stage.as<uint8_t>() + (size_t)(e->st_next_row + i) * rowbytes, scanlines[i], rowbytes);
  e->st_next_row += num_lines;
  return num_lines;
}
int b200jpeg_finish_compress(b200jpeg_encoder *e, const uint8_t **jpeg, size_t *size)
{
  if (!e || e->st_state != 1) { set_error("Improper call to JPEG library in state %d", e ? 100 + e->st_state : -1); return B200JPEG_ERR_STATE; }
  const b200jpeg_params &p = e->st_params;
  if (e->st_next_row < p.image_height) { set_error("Application transferred too few scanlines"); return B200JPEG_ERR_STATE; }   // JERR_TOO_LITTLE_DATA
  size_t rowbytes = (size_t)p.image_width * p.input_components * (p.data_precision > 8 ? 2 : 1);
  e->st_state = 0;
  int rc = encode_common(e, &p, e->h_stage.p, 0, rowbytes, rowbytes * p.image_height, 1, false);
  if (rc) return rc;
  return b200jpeg_get_output(e, 0, jpeg, size);
}

}  // extern "C"
