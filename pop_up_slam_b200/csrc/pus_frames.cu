// pus_frames.cu -- the pop-up session (pus_popup_session_*): main_3d's per-frame chain (main_3d.cpp:417-454) over a batch
// of frames, device-resident.  lines -> edges -> fit on the open segments -> get_plane_equation's actual-index filter ->
// polygons on the open segments -> clouds and depth maps of the good rows.  The stage kernels are launched through
// pus_stages.cuh as the stage calls launch them; the host loops between the stage calls (scans, packing, the filter,
// plane_jobs) run here as glue kernels on the shared code of pus_frames.cuh.  Buffers only grow; a run reads back four
// small blocks of totals to size what follows.  Compiled with --fmad=false like the stages.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <type_traits>
#include <string>
#include <vector>

#include "../../include/popup_gpu.h"
#include "pus_frames.cuh"
#include "pus_stages.cuh"

namespace pus {
namespace frames {
constexpr int kScan = 1024;

// exclusive prefix sum of v(i), i < n, in one kScan-thread block: out(i, offset) per element; every thread gets the total
template <class V, class O>
__device__ long long block_scan(int n, V v, O out) {
  __shared__ long long s[kScan];
  const int t = threadIdx.x, chunk = (n + kScan - 1) / kScan;
  const int i0 = min(n, t * chunk), i1 = min(n, i0 + chunk);
  long long sum = 0;
  for (int i = i0; i < i1; i++) sum += v(i);
  s[t] = sum;
  __syncthreads();
  for (int o = 1; o < kScan; o <<= 1) {
    const long long add = t >= o ? s[t - o] : 0;
    __syncthreads();
    s[t] += add;
    __syncthreads();
  }
  long long run = s[t] - sum;
  for (int i = i0; i < i1; i++) {
    const long long x = v(i);
    out(i, run);
    run += x;
  }
  const long long total = s[kScan - 1];
  __syncthreads();
  return total;
}

// sizes[]: what a run reads back
enum { S_LINES, S_NODE, S_OBJ, S_CPT, S_IVL, S_OPEN, S_CONN, S_GOOD, S_BOUND, S_CUT, S_WORLD, S_CROWS, S_DROWS, S_N };

// lines: each frame's count as pus_popup_lines gives it, its first packed row, its line status
__global__ void __launch_bounds__(kScan) line_scan_kernel(int n, const int* lst, const int* fc, int* line_status,
                                                          int* line_counts, long long* first, long long* sizes) {
  const long long total = block_scan(
      n, [&](int f) { return (long long)(lst[f] ? 0 : fc[f]); },
      [&](int f, long long o) {
        first[f] = o;
        line_status[f] = lst[f];
        line_counts[f] = lst[f] ? 0 : fc[f];
      });
  if (threadIdx.x == 0) sizes[S_LINES] = total;
}

// status 1 where pus_popup_edges would refuse the frame's lines (more than PUS_POPUP_MAX_LINES, a coordinate not finite);
// the edge stage then gets no lines for it
__global__ void line_check_kernel(int n, const int* line_counts, const long long* first, const float* lines, int* status,
                                  int* edge_lines) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const int c = line_counts[f];
  status[f] = glue::lines_status(lines + 4 * first[f], c);
  edge_lines[f] = status[f] ? 0 : c;
}

// pus_popup_edges' scratch table, frame by frame as the stage call lays it out
__global__ void edge_table_kernel(int n, const int* seg_count, const long long* first, const int* edge_lines, long long cells,
                                  edges::Frame* fr, long long* sizes) {
  long long run[4] = {0, 0, 0, 0};
  for (int f = 0; f < n; f++) glue::edge_frame(f, seg_count[f], (int)first[f], edge_lines[f], cells, run, fr[f]);
  for (int k = 0; k < 4; k++) sizes[S_NODE + k] = run[k];
}

// edge status (-1: not run), the segment limit (status 2) and the open / connected offsets
__global__ void __launch_bounds__(kScan) edge_scan_kernel(int n, const int* eout, int* status, int* edge_status,
                                                          int* open_ptr, int* conn_ptr, long long* sizes) {
  for (int f = threadIdx.x; f < n; f += kScan) {
    edge_status[f] = status[f] == 1 ? -1 : eout[4 * f];
    status[f] = glue::edges_status(status[f], eout[4 * f + 1]);
  }
  __syncthreads();
  const long long no = block_scan(
      n, [&](int f) { return (long long)(status[f] ? 0 : eout[4 * f + 1]); }, [&](int f, long long o) { open_ptr[f] = (int)o; });
  const long long nc = block_scan(
      n, [&](int f) { return (long long)(status[f] ? 0 : eout[4 * f + 2]); }, [&](int f, long long o) { conn_ptr[f] = (int)o; });
  if (threadIdx.x == 0) {
    open_ptr[n] = (int)no;
    conn_ptr[n] = (int)nc;
    sizes[S_OPEN] = no;
    sizes[S_CONN] = nc;
  }
}

// the frames' segments from their slots to the packed lists, and the row -> frame table of the fit and the polygons
__global__ void edge_pack_kernel(int n, const long long* first, const int* open_ptr, const int* conn_ptr, const float* open_slot,
                                 const float* conn_slot, const int* inc_slot, float* open, float* conn, int* inc,
                                 int* row_frame) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const long long l0 = first[f];
  const int o0 = open_ptr[f], no = open_ptr[f + 1] - o0, c0 = conn_ptr[f], nc = conn_ptr[f + 1] - c0;
  for (int i = 0; i < 4 * no; i++) open[4LL * o0 + i] = open_slot[8 * l0 + i];
  for (int i = 0; i < no; i++) inc[o0 + i] = inc_slot[2 * l0 + i];
  for (int i = 0; i < 4 * nc; i++) conn[4LL * c0 + i] = conn_slot[16 * l0 + i];
  for (int r = o0 + f; r <= o0 + no + f; r++) row_frame[r] = f;
}

// get_plane_equation's filter of the good walls; a frame without open segments has no good planes
__global__ void filter_kernel(int n, const int* open_ptr, const int* inc, int* good, int* n_good) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const int o0 = open_ptr[f], no = open_ptr[f + 1] - o0;
  n_good[f] = no > 0 ? glue::actual_filter(inc + o0, no, good + o0 + f) : 0;
}

// good_ptr (block 0) and the packed polygons' row offsets of the bound, cut and world polygons (blocks 1-3), as
// pus_popup_polygons scans them on the host
__global__ void __launch_bounds__(kScan) row_scan_kernel(int n, int n_rows, const int* n_good, const int* counts, int* good_ptr,
                                                         long long* off, int* ptr3, long long* sizes) {
  if (blockIdx.x == 0) {
    const long long ng = block_scan(
        n, [&](int f) { return (long long)n_good[f]; }, [&](int f, long long o) { good_ptr[f] = (int)o; });
    if (threadIdx.x == 0) {
      good_ptr[n] = (int)ng;
      sizes[S_GOOD] = ng;
    }
    return;
  }
  const int k = blockIdx.x - 1;
  const int* c = counts + (size_t)k * n_rows;
  long long* o = off + (size_t)k * n_rows;
  int* p = ptr3 + (size_t)k * (n_rows + 1);
  const long long t = block_scan(
      n_rows, [&](int r) { return (long long)c[r]; },
      [&](int r, long long x) {
        o[r] = x;
        p[r] = (int)x;
      });
  if (threadIdx.x == 0) {
    p[n_rows] = (int)t;
    sizes[S_BOUND + k] = t;
  }
}

// one job (polygon box, shifted vertices) per good plane for the clouds and one for the depth map: plane_jobs on the device.
// A polygon beyond PUS_POPUP_MAX_VERTICES or PUS_POPUP_MAX_COORD is not truncated; its plane gets no points (plane_status
// bit 0) or is not drawn (bit 1).
struct JobArgs {
  int n, downsample, cloud_from_cut;
  const int *open_ptr, *good, *good_ptr;
  const float* planes_sensor;
  const float *bound, *cut;
  const int *bound_ptr, *cut_ptr;
  int *good_rows, *plane_status;
  float* planes;
  cloud::Job *cjobs, *djobs;
  int2 *cvtx, *dvtx;
};
__global__ void job_kernel(JobArgs A) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= A.n) return;
  const int r0 = A.open_ptr[f] + f, nr = A.open_ptr[f + 1] - A.open_ptr[f] + 1;
  int p = A.good_ptr[f];
  if (p == A.good_ptr[f + 1]) return;
  for (int j = 0; j < nr; j++) {
    const int r = r0 + j;
    if (!A.good[r]) continue;
    A.good_rows[p] = j;
    for (int i = 0; i < 4; i++) A.planes[4LL * p + i] = A.planes_sensor[4LL * r + i];
    int st = 0;
    for (int k = 0; k < 2; k++) {
      const bool from_cut = k == 0 && A.cloud_from_cut;
      const int* ptr = from_cut ? A.cut_ptr : A.bound_ptr;
      const float* q = (from_cut ? A.cut : A.bound) + 2LL * ptr[r];
      cloud::Job J{f, ptr[r], ptr[r + 1] - ptr[r], 0, 0, 0, 0, 0};
      if (!glue::polygon_ok(q, J.n)) {
        st |= 1 << k;
        J.n = 0;
      }
      if (J.n > 0) glue::polygon_box(q, J.n, A.downsample, J, (k == 0 ? A.cvtx : A.dvtx) + J.v0);
      (k == 0 ? A.cjobs : A.djobs)[p] = J;
    }
    A.plane_status[p] = st;
    p++;
  }
}

// the jobs' first span rows
__global__ void __launch_bounds__(kScan) job_scan_kernel(int n, const int* good_ptr, cloud::Job* cjobs, cloud::Job* djobs,
                                                         long long* sizes) {
  const int n_planes = good_ptr[n];
  const long long a = block_scan(
      n_planes, [&](int p) { return (long long)cjobs[p].bh; }, [&](int p, long long o) { cjobs[p].row0 = (int)o; });
  const long long b = block_scan(
      n_planes, [&](int p) { return (long long)djobs[p].bh; }, [&](int p, long long o) { djobs[p].row0 = (int)o; });
  if (threadIdx.x == 0) {
    sizes[S_CROWS] = a;
    sizes[S_DROWS] = b;
  }
}
}  // namespace frames

bool on_device(const void* p) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

namespace {
struct Slot {
  void* p = nullptr;
  size_t bytes = 0;
};

struct Session {
  int device = 0;
  pus_popup_config cfg{};
  cudaStream_t own = nullptr, st = nullptr;
  std::vector<Slot> dev, host;
  size_t cursor = 0, hcursor = 0;
  long long n_allocs = 0, reserved = 0;
  pus_popup_frames res{};

  ~Session() {
    if (st) cudaStreamSynchronize(st);
    for (Slot& s : dev) cudaFree(s.p);
    for (Slot& s : host) cudaFreeHost(s.p);
    if (own) cudaStreamDestroy(own);
  }
  // grow-only slot k of the device (or pinned host) buffers; slots are taken in the same order on every run
  cudaError_t slot(std::vector<Slot>& v, size_t& cur, bool pinned, void** p, size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (cur == v.size()) v.emplace_back();
    Slot& s = v[cur++];
    if (s.bytes < bytes) {
      const size_t want = std::max(bytes, s.bytes + s.bytes / 2);
      if (s.p) (pinned ? cudaFreeHost(s.p) : cudaFree(s.p));
      reserved -= (long long)s.bytes;
      s.p = nullptr;
      s.bytes = 0;
      const cudaError_t e = pinned ? cudaMallocHost(&s.p, want) : cudaMalloc(&s.p, want);
      if (e != cudaSuccess) return e;
      s.bytes = want;
      reserved += (long long)want;
      n_allocs++;
    }
    *p = s.p;
    return cudaSuccess;
  }
};

struct Arena : pus::Alloc {
  Session& S;
  explicit Arena(Session& s) : S(s) {}
  cudaError_t raw(void** p, size_t bytes) override { return S.slot(S.dev, S.cursor, false, p, bytes); }
};

bool finite9(const float* a) {
  for (int i = 0; i < 9; i++)
    if (!std::isfinite(a[i])) return false;
  return true;
}

// "" when the config is one the stage calls accept as main_3d runs them: the edges' and the lines' own rules (the edges'
// frame size first), then the session's
std::string config_error(const pus_popup_config& c) {
  const std::string why = edges::shape_error(c.width, c.height, &c.edges);
  if (!why.empty()) return why;
  if (const char* w = lines::shape_error(c.width, c.height, c.channels, c.fast_edges)) return w;
  if (!finite9(c.K) || !finite9(c.invK)) return "K and invK must be finite";
  if (c.downsample_poly && (c.want_labels || c.want_depth) && ((c.width | c.height) & 1))
    return "label images and depth maps in downsample_poly mode need an even width and height";
  if (c.want_rgb && c.channels != 3) return "want_rgb needs BGR images (channels 3)";
  return "";
}

const Call kSession{"pus_popup_session"};
}  // namespace
}  // namespace pus

using namespace pus;

extern "C" int pus_popup_session_create(int device, const pus_popup_config* cfg, pus_popup_session* out) {
  if (!cfg || !out) return kSession.refuse("config and out must be given");
  const std::string why = config_error(*cfg);
  if (!why.empty()) return kSession.refuse(why);
  if (kSession.check_device(device) < 0) return -1;
  Session* S = new Session;
  S->device = device;
  S->cfg = *cfg;
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&S->own, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete S;
    return kSession.refuse(std::string("stream: ") + cudaGetErrorString(e));
  }
  S->st = S->own;
  *out = S;
  return 0;
}

extern "C" int pus_popup_session_destroy(pus_popup_session s) {
  if (!s) return kSession.refuse("session is NULL");
  Session* S = (Session*)s;
  cudaSetDevice(S->device);
  delete S;
  return 0;
}

extern "C" int pus_popup_session_set_stream(pus_popup_session s, void* cuda_stream) {
  if (!s) return kSession.refuse("session is NULL");
  Session* S = (Session*)s;
  S->st = cuda_stream ? (cudaStream_t)cuda_stream : S->own;
  return 0;
}

extern "C" int pus_popup_session_memory(pus_popup_session s, long long* allocations, long long* reserved_bytes) {
  if (!s) return kSession.refuse("session is NULL");
  Session* S = (Session*)s;
  if (allocations) *allocations = S->n_allocs;
  if (reserved_bytes) *reserved_bytes = S->reserved;
  return 0;
}

extern "C" int pus_popup_session_run(pus_popup_session s, int n_frames, const unsigned char* images, const unsigned char* labels,
                                     const float* Ts) {
  using namespace pus::frames;
  if (!s) return kSession.refuse("session is NULL");
  if (n_frames < 0) return kSession.refuse("n_frames < 0");
  if (n_frames > 0 && (!images || !labels || !Ts)) return kSession.refuse("images, labels and Ts must be given");
  Session& S = *(Session*)s;
  const pus_popup_config& c = S.cfg;
  S.res = pus_popup_frames{};   // and so it stays until the run has succeeded
  const Call C{"pus_popup_session_run"};
  PUS_CALL_OK(C, cudaSetDevice(S.device));
  S.cursor = S.hcursor = 0;
  Arena A(S);
  cudaStream_t st = S.st;
  const int n = n_frames, W = c.width, H = c.height;
  const long long px = (long long)W * H;
  auto dev = [&](auto*& p, size_t count) { return A.get(p, count); };
  auto pinned = [&](auto*& p, size_t count) {
    void* v = nullptr;
    const cudaError_t e = S.slot(S.host, S.hcursor, true, &v, (count > 0 ? count : 1) * sizeof(*p));
    p = (std::remove_reference_t<decltype(p)>)v;
    return e;
  };
  // inputs: device pointers are read in place, host data goes through pinned staging
  auto input = [&](const auto* src, size_t count, const auto*& d) -> cudaError_t {
    using T = std::remove_const_t<std::remove_reference_t<decltype(*src)>>;
    const bool in_place = on_device(src);
    T *h = nullptr, *dd = nullptr;
    cudaError_t e;   // a device input still takes its (empty) staging slots, so the later slots keep their places
    if ((e = pinned(h, in_place ? 0 : count)) != cudaSuccess || (e = dev(dd, in_place ? 0 : count)) != cudaSuccess) return e;
    if (in_place) {
      d = src;
      return cudaSuccess;
    }
    if (n == 0) {
      d = dd;
      return cudaSuccess;
    }
    std::memcpy(h, src, count * sizeof(T));
    d = dd;
    return cudaMemcpyAsync(dd, h, count * sizeof(T), cudaMemcpyHostToDevice, st);
  };
  const unsigned char *d_img = nullptr, *d_lab = nullptr;
  const float* d_T = nullptr;
  float* d_K = nullptr;
  long long* sizes = nullptr;
  long long* h_sizes = nullptr;
  PUS_CALL_OK(C, input(images, (size_t)(n * px * c.channels), d_img));
  PUS_CALL_OK(C, input(labels, (size_t)(n * px), d_lab));
  PUS_CALL_OK(C, input(Ts, (size_t)n * 16, d_T));
  PUS_CALL_OK(C, dev(d_K, 18));
  PUS_CALL_OK(C, dev(sizes, S_N));
  PUS_CALL_OK(C, pinned(h_sizes, S_N));
  PUS_CALL_OK(C, cudaMemcpyAsync(d_K, c.K, 9 * sizeof(float), cudaMemcpyHostToDevice, st));
  PUS_CALL_OK(C, cudaMemcpyAsync(d_K + 9, c.invK, 9 * sizeof(float), cudaMemcpyHostToDevice, st));
  const float *d_Kf = d_K, *d_iK = d_K + 9;
  auto readback = [&]() {   // one host synchronisation
    cudaError_t e = cudaMemcpyAsync(h_sizes, sizes, S_N * sizeof(long long), cudaMemcpyDeviceToHost, st);
    return e != cudaSuccess ? e : cudaStreamSynchronize(st);
  };
  const unsigned fb = (unsigned)((n + 127) / 128);

  // 1. lines (fast_edges: the 0.5x image)
  const lines::Dims D = lines::make_dims(W, H, c.channels, c.fast_edges);
  lines::Work LW;
  int *line_status = nullptr, *line_counts = nullptr, *status = nullptr, *edge_lines = nullptr;
  long long* first = nullptr;
  float* d_lines = nullptr;
  PUS_CALL_OK(C, lines::detect(st, A, n, D, d_img, LW));
  PUS_CALL_OK(C, dev(line_status, n));
  PUS_CALL_OK(C, dev(line_counts, n));
  PUS_CALL_OK(C, dev(status, n));
  PUS_CALL_OK(C, dev(edge_lines, n));
  PUS_CALL_OK(C, dev(first, n));
  PUS_CALL_OK(C, dev(d_lines, 4 * (size_t)n * D.nslot));   // a frame has at most line_slots lines
  // 2. edges: label maps first, then the table from their segment counts and the lines
  edges::Maps M;
  edges::Frame* d_fr = nullptr;
  PUS_CALL_OK(C, edges::prep(st, A, n, d_lab, W, H, c.edges, M));
  PUS_CALL_OK(C, dev(d_fr, n));
  if (n > 0) {
    line_scan_kernel<<<1, kScan, 0, st>>>(n, LW.st, LW.fc, line_status, line_counts, first, sizes);
    PUS_CALL_OK(C, lines::scatter(st, n, D, LW, first, d_lines));
    line_check_kernel<<<fb, 128, 0, st>>>(n, line_counts, first, d_lines, status, edge_lines);
    edge_table_kernel<<<1, 1, 0, st>>>(n, M.seg_count, first, edge_lines, (long long)M.w * M.h, d_fr, sizes);
    PUS_CALL_OK(C, cudaGetLastError());
    PUS_CALL_OK(C, readback());   // sync 1: the line total and the edge scratch
  } else {
    std::memset(h_sizes, 0, S_N * sizeof(long long));
  }
  const long long n_lines = h_sizes[S_LINES];
  const long long tot[4] = {h_sizes[S_NODE], h_sizes[S_OBJ], h_sizes[S_CPT], h_sizes[S_IVL]};
  float *open_slot = nullptr, *conn_slot = nullptr;
  int *inc_slot = nullptr, *eout = nullptr, *edge_status = nullptr, *open_ptr = nullptr, *conn_ptr = nullptr;
  PUS_CALL_OK(C, dev(open_slot, 8 * n_lines));
  PUS_CALL_OK(C, dev(conn_slot, 16 * n_lines));
  PUS_CALL_OK(C, dev(inc_slot, 2 * n_lines));
  PUS_CALL_OK(C, dev(eout, 4 * (size_t)n));
  PUS_CALL_OK(C, dev(edge_status, n));
  PUS_CALL_OK(C, dev(open_ptr, n + 1));
  PUS_CALL_OK(C, dev(conn_ptr, n + 1));
  PUS_CALL_OK(C, edges::select(st, A, n, c.edges, W, H, M, d_fr, tot, n_lines, d_lines, open_slot, conn_slot, inc_slot, eout));
  if (n > 0) {
    edge_scan_kernel<<<1, kScan, 0, st>>>(n, eout, status, edge_status, open_ptr, conn_ptr, sizes);
    PUS_CALL_OK(C, cudaGetLastError());
    PUS_CALL_OK(C, readback());   // sync 2: the open and connected totals
  }
  const long long n_open = h_sizes[S_OPEN], n_conn = h_sizes[S_CONN];
  const int n_rows = (int)(n_open + n);
  // 3. fit on the open segments; the same launch gives the polygons their planes and world ground endpoints
  float *open = nullptr, *conn = nullptr, *pw = nullptr, *ps = nullptr, *dist = nullptr, *ends = nullptr;
  int *inc = nullptr, *row_frame = nullptr, *good = nullptr;
  PUS_CALL_OK(C, dev(open, 4 * n_open));
  PUS_CALL_OK(C, dev(conn, 4 * n_conn));
  PUS_CALL_OK(C, dev(inc, n_open));
  PUS_CALL_OK(C, dev(row_frame, n_rows));
  PUS_CALL_OK(C, dev(pw, 4 * (size_t)n_rows));
  PUS_CALL_OK(C, dev(ps, 4 * (size_t)n_rows));
  PUS_CALL_OK(C, dev(dist, n_rows));
  PUS_CALL_OK(C, dev(good, n_rows));
  PUS_CALL_OK(C, dev(ends, 6 * (size_t)n_rows));
  // 5. polygons on the open segments (their rows are the fit's)
  float *bslot = nullptr, *cslot = nullptr, *wslot = nullptr, *bound = nullptr, *cut = nullptr, *world = nullptr;
  int *pcnt = nullptr, *ptr3 = nullptr, *n_good = nullptr, *good_ptr = nullptr;
  long long* poff = nullptr;
  PUS_CALL_OK(C, dev(bslot, (size_t)n_rows * poly::kBoundSlot * 2));
  PUS_CALL_OK(C, dev(cslot, (size_t)n_rows * poly::kCutSlot * 2));
  PUS_CALL_OK(C, dev(wslot, (size_t)n_rows * poly::kCutSlot * 3));
  PUS_CALL_OK(C, dev(bound, (size_t)n_rows * poly::kBoundSlot * 2));
  PUS_CALL_OK(C, dev(cut, (size_t)n_rows * poly::kBoundSlot * 2));
  PUS_CALL_OK(C, dev(world, (size_t)n_rows * poly::kCutSlot * 3));
  PUS_CALL_OK(C, dev(pcnt, 3 * (size_t)n_rows));
  PUS_CALL_OK(C, dev(poff, 3 * (size_t)n_rows));
  PUS_CALL_OK(C, dev(ptr3, 3 * ((size_t)n_rows + 1)));
  PUS_CALL_OK(C, dev(n_good, n));
  PUS_CALL_OK(C, dev(good_ptr, n + 1));
  const poly::Params PP{open_ptr, row_frame, n_rows, open, d_Kf, d_iK, d_T, ps, ends, W, H, c.ceiling_threshold,
                        c.walllength_threshold, bslot, cslot, wslot, pcnt};
  if (n > 0) {
    edge_pack_kernel<<<fb, 128, 0, st>>>(n, first, open_ptr, conn_ptr, open_slot, conn_slot, inc_slot, open, conn, inc,
                                         row_frame);
    PUS_CALL_OK(C, cudaMemsetAsync(pw, 0, 4 * (size_t)n_rows * sizeof(float), st));
    PUS_CALL_OK(C, cudaMemsetAsync(ps, 0, 4 * (size_t)n_rows * sizeof(float), st));
    PUS_CALL_OK(C, cudaMemsetAsync(dist, 0, (size_t)n_rows * sizeof(float), st));
    PUS_CALL_OK(C, cudaMemsetAsync(good, 0, (size_t)n_rows * sizeof(int), st));
    PUS_CALL_OK(C, launch_fit(st, n, open_ptr, row_frame, n_rows, open, d_iK, d_T, c.plane_cam_dist_thre, 0, pw, ps, dist, good,
                              ends));
    PUS_CALL_OK(C, poly::launch_rows(st, PP));
    // 4. the actual-index filter, then the offsets
    filter_kernel<<<fb, 128, 0, st>>>(n, open_ptr, inc, good, n_good);
    row_scan_kernel<<<4, kScan, 0, st>>>(n, n_rows, n_good, pcnt, good_ptr, poff, ptr3, sizes);
    PUS_CALL_OK(C, poly::launch_pack(st, PP, poff, bound, cut, world));
    PUS_CALL_OK(C, cudaGetLastError());
  }
  // 6. / 7. the good rows' jobs for the clouds and the depth map
  const int vcap = n_rows * poly::kBoundSlot;
  int *good_rows = nullptr, *plane_status = nullptr;
  float* planes = nullptr;
  cloud::Job *cjobs = nullptr, *djobs = nullptr;
  int2 *cvtx = nullptr, *dvtx = nullptr;
  PUS_CALL_OK(C, dev(good_rows, n_rows));
  PUS_CALL_OK(C, dev(plane_status, n_rows));
  PUS_CALL_OK(C, dev(planes, 4 * (size_t)n_rows));
  PUS_CALL_OK(C, dev(cjobs, n_rows));
  PUS_CALL_OK(C, dev(djobs, n_rows));
  PUS_CALL_OK(C, dev(cvtx, vcap));
  PUS_CALL_OK(C, dev(dvtx, vcap));
  const int cloud_from_cut = c.walllength_threshold > 0;
  if (n > 0) {
    frames::JobArgs JA{n, c.downsample_poly ? 1 : 0, cloud_from_cut, open_ptr, good, good_ptr, ps, bound, cut,
                       ptr3, ptr3 + (n_rows + 1), good_rows, plane_status, planes, cjobs, djobs, cvtx, dvtx};
    job_kernel<<<fb, 128, 0, st>>>(JA);
    job_scan_kernel<<<1, kScan, 0, st>>>(n, good_ptr, cjobs, djobs, sizes);
    PUS_CALL_OK(C, cudaGetLastError());
    PUS_CALL_OK(C, readback());   // sync 3: good planes, vertex totals, box rows
  }
  const int n_planes = (int)h_sizes[S_GOOD];
  const long long crows = h_sizes[S_CROWS], drows = h_sizes[S_DROWS];
  // clouds
  int2* cspan = nullptr;
  int *rowcnt = nullptr, *ccount = nullptr;
  long long *rowoff = nullptr, *coff = nullptr;
  PUS_CALL_OK(C, dev(cspan, crows));
  PUS_CALL_OK(C, dev(rowcnt, crows));
  PUS_CALL_OK(C, dev(rowoff, crows + 1));
  PUS_CALL_OK(C, dev(ccount, n_planes));
  PUS_CALL_OK(C, dev(coff, n_planes));
  cloud::Params CP{cjobs, cvtx, planes, d_T, d_iK, c.want_rgb ? d_img : nullptr, W, H, c.downsample_poly ? 2 : 1, c.channels == 3 && W == 960,
                   c.depth_thre, c.ceiling_threshold, cspan, rowcnt, rowoff, nullptr, nullptr};
  long long n_points = 0;
  if (n > 0) {
    PUS_CALL_OK(C, cloud::launch_count(st, n_planes, crows, CP, rowoff, ccount, coff));
    PUS_CALL_OK(C, cudaMemcpyAsync(sizes, rowoff + crows, sizeof(long long), cudaMemcpyDeviceToDevice, st));
    PUS_CALL_OK(C, readback());   // sync 4: the point total
    n_points = h_sizes[0];
  }
  float* xyz = nullptr;
  unsigned char *rgb = nullptr, *lab = nullptr;
  float *depth = nullptr, *fill = nullptr;
  PUS_CALL_OK(C, dev(xyz, 3 * n_points));
  PUS_CALL_OK(C, dev(rgb, c.want_rgb ? 3 * n_points : 0));
  PUS_CALL_OK(C, dev(lab, c.want_labels ? (size_t)(n * px) : 0));
  const int scale = c.downsample_poly ? 2 : 1;
  PUS_CALL_OK(C, dev(depth, c.want_depth ? (size_t)(n * px) : 0));
  PUS_CALL_OK(C, dev(fill, c.want_depth && scale == 2 ? (size_t)n * (W / 2) * (H / 2) : 0));
  cloud::Edge* dedges = nullptr;
  int2* dspan = nullptr;
  PUS_CALL_OK(C, dev(dedges, c.want_depth ? vcap : 0));
  PUS_CALL_OK(C, dev(dspan, c.want_depth ? drows : 0));
  if (n > 0) {
    CP.xyz = xyz;
    CP.rgb = c.want_rgb ? rgb : nullptr;
    if (n_points > 0) PUS_CALL_OK(C, cloud::launch_write(st, n_planes, CP));
    if (c.want_labels) {
      PUS_CALL_OK(C, cudaMemsetAsync(lab, 127, (size_t)(n * px), st));
      PUS_CALL_OK(C, cloud::launch_labels(st, n, good_ptr, CP, lab));
    }
    if (c.want_depth)
      PUS_CALL_OK(C, cloud::launch_depth(st, n, n_planes, good_ptr, djobs, dvtx, dedges, dspan, planes, d_T, d_iK, W, H,
                                         c.downsample_poly, c.ceiling_threshold, scale == 2 ? fill : depth, depth));
    PUS_CALL_OK(C, cudaGetLastError());
  }
  pus_popup_frames& R = S.res;
  R.n_frames = n;
  R.n_rows = n_rows;
  R.n_good = n_planes;
  R.n_open = n_open;
  R.n_connect = n_conn;
  R.n_bound = h_sizes[S_BOUND];
  R.n_cut = h_sizes[S_CUT];
  R.n_world = h_sizes[S_WORLD];
  R.n_points = n_points;
  R.status = status; R.line_status = line_status; R.line_counts = line_counts; R.edge_status = edge_status;
  R.open_ptr = open_ptr; R.connect_ptr = conn_ptr; R.open_segs = open; R.connect_segs = conn; R.open_in_connect = inc;
  R.planes_world = pw; R.planes_sensor = ps; R.dist = dist; R.good = good;
  R.bound_ptr = ptr3; R.cut_ptr = ptr3 + (n_rows + 1); R.world_ptr = ptr3 + 2 * (n_rows + 1);
  R.bound2d = bound; R.cut2d = cut; R.world3d = world;
  R.good_ptr = good_ptr; R.good_rows = good_rows; R.plane_status = plane_status;
  R.cloud_counts = ccount; R.cloud_offsets = coff; R.xyz = xyz; R.rgb = c.want_rgb ? rgb : nullptr;
  R.labels = c.want_labels ? lab : nullptr; R.depth = c.want_depth ? depth : nullptr;
  return 0;
}

extern "C" int pus_popup_session_result(pus_popup_session s, pus_popup_frames* out) {
  if (!s || !out) return kSession.refuse("session and out must be given");
  *out = ((Session*)s)->res;
  return 0;
}

extern "C" int pus_popup_session_download(pus_popup_session s, pus_popup_frames* dst) {
  if (!s || !dst) return kSession.refuse("session and dst must be given");
  Session& S = *(Session*)s;
  const pus_popup_frames& R = S.res;
  const long long n = R.n_frames, rows = R.n_rows, g = R.n_good, px = (long long)S.cfg.width * S.cfg.height;
  struct Copy { void* d; const void* s; long long bytes; };
  const Copy copies[] = {
      {dst->status, R.status, 4 * n}, {dst->line_status, R.line_status, 4 * n}, {dst->line_counts, R.line_counts, 4 * n},
      {dst->edge_status, R.edge_status, 4 * n}, {dst->open_ptr, R.open_ptr, 4 * (n + 1)},
      {dst->connect_ptr, R.connect_ptr, 4 * (n + 1)}, {dst->open_segs, R.open_segs, 16 * R.n_open},
      {dst->connect_segs, R.connect_segs, 16 * R.n_connect}, {dst->open_in_connect, R.open_in_connect, 4 * R.n_open},
      {dst->planes_world, R.planes_world, 16 * rows}, {dst->planes_sensor, R.planes_sensor, 16 * rows},
      {dst->dist, R.dist, 4 * rows}, {dst->good, R.good, 4 * rows}, {dst->bound_ptr, R.bound_ptr, 4 * (rows + 1)},
      {dst->cut_ptr, R.cut_ptr, 4 * (rows + 1)}, {dst->world_ptr, R.world_ptr, 4 * (rows + 1)},
      {dst->bound2d, R.bound2d, 8 * R.n_bound}, {dst->cut2d, R.cut2d, 8 * R.n_cut}, {dst->world3d, R.world3d, 12 * R.n_world},
      {dst->good_ptr, R.good_ptr, 4 * (n + 1)}, {dst->good_rows, R.good_rows, 4 * g},
      {dst->plane_status, R.plane_status, 4 * g}, {dst->cloud_counts, R.cloud_counts, 4 * g},
      {dst->cloud_offsets, R.cloud_offsets, 8 * g}, {dst->xyz, R.xyz, 12 * R.n_points},
      {dst->rgb, R.rgb, 3 * R.n_points}, {dst->labels, R.labels, n * px}, {dst->depth, R.depth, 4 * n * px}};
  if (n > 0 && !R.status) return kSession.refuse("no successful run to download");
  if ((dst->rgb && !R.rgb) || (dst->labels && !R.labels) || (dst->depth && !R.depth))
    return kSession.refuse("an optional output the config does not make was asked for");
  cudaError_t e = cudaSetDevice(S.device);
  for (const Copy& c : copies)
    if (e == cudaSuccess && c.d && c.bytes > 0) e = cudaMemcpyAsync(c.d, c.s, (size_t)c.bytes, cudaMemcpyDefault, S.st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(S.st);
  if (e != cudaSuccess) return kSession.refuse(std::string("download: ") + cudaGetErrorString(e));
  return 0;
}
