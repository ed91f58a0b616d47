// pus_stages.cuh -- the pop-up stages' internal launchers: device pointers in, kernels enqueued on a stream.  The extern "C"
// stage calls (pus_popup.cu, pus_lines.cu) and the pop-up session (pus_frames.cu) launch the same kernels through these.
// Scratch comes from an Alloc: the stage calls free theirs on return (TempAlloc), the session keeps grow-only buffers.
// Also the host side every stage call shares: its error messages and device check (Call), and the seg_ptr row table.
#pragma once
#include <cuda_runtime.h>

#include <climits>
#include <new>
#include <string>
#include <vector>

#include "../../include/popup_gpu.h"

namespace pus {
extern thread_local std::string g_err;

// whether p is device (or managed) memory; anything else is taken as host memory (pus_frames.cu)
bool on_device(const void* p);

// device scratch for a launcher
struct Alloc {
  virtual ~Alloc() = default;
  virtual cudaError_t raw(void** p, size_t bytes) = 0;
  template <class T>
  cudaError_t get(T*& p, size_t n) {
    void* v = nullptr;
    const cudaError_t e = raw(&v, (n > 0 ? n : 1) * sizeof(T));
    p = (T*)v;
    return e;
  }
  // get, then a synchronous copy of h [0, n) (none when n is 0)
  template <class T>
  cudaError_t upload(T*& d, const T* h, size_t n) {
    const cudaError_t e = get(d, n);
    return e != cudaSuccess || n == 0 ? e : cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice);
  }
};
// a synchronous copy of d [0, n) into h (none when n is 0)
template <class T>
cudaError_t download(T* h, const T* d, size_t n) {
  return n == 0 ? cudaSuccess : cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost);
}
// cudaMalloc per request, everything freed on destruction
struct TempAlloc : Alloc {
  std::vector<void*> ps;
  ~TempAlloc() override {
    for (void* p : ps) cudaFree(p);
  }
  cudaError_t raw(void** p, size_t bytes) override {
    const cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) ps.push_back(*p);
    return e;
  }
};

// the messages of one extern "C" call: everything it refuses goes to g_err as "<name>: <why>"
struct Call {
  const char* name;
  int refuse(const std::string& why) const {
    g_err = std::string(name) + ": " + why;
    return -1;
  }
  // 0, or -1 refused: the library has no CPU path to fall back to
  int check_device(int device) const {
    int n = 0;
    if (cudaGetDeviceCount(&n) == cudaSuccess && device >= 0 && device < n) return 0;
    return refuse("no CUDA device usable; libpopup_gpu has no CPU fallback");
  }
  // true, with "<name>: <what>: <CUDA error>" in g_err, when e is an error
  bool failed(cudaError_t e, const char* what) const {
    if (e != cudaSuccess) refuse(std::string(what) + ": " + cudaGetErrorString(e));
    return e != cudaSuccess;
  }
};
// return -1 from the calling function when `call` fails, reported through the Call C
#define PUS_CALL_OK(C, call)                    \
  do {                                          \
    if ((C).failed((call), #call)) return -1;   \
  } while (0)

// Frame f of a CSR seg_ptr [n_frames + 1] owns the rows seg_ptr[f] + f .. seg_ptr[f + 1] + f: its ground row, then one row
// per segment.  Checks all of seg_ptr before row_frame is written: given, starting at 0, and frame by frame non-decreasing
// and, when capped, at most PUS_POPUP_MAX_SEGMENTS segments; the row count must fit an int.  Then sets each row's frame.
// Returns NULL, or why seg_ptr is refused.  n_frames >= 0.
inline const char* row_frames(int n_frames, const int* seg_ptr, std::vector<int>& row_frame, bool capped = false) {
  if (!seg_ptr || seg_ptr[0] != 0) return "seg_ptr must be given and start at 0";
  for (int f = 0; f < n_frames; f++) {
    if (seg_ptr[f + 1] < seg_ptr[f]) return "seg_ptr is not ascending";
    if (capped && seg_ptr[f + 1] - seg_ptr[f] > PUS_POPUP_MAX_SEGMENTS)
      return "a frame has more than PUS_POPUP_MAX_SEGMENTS segments";
  }
  if (seg_ptr[n_frames] > INT_MAX - n_frames) return "seg_ptr has more rows than an int can count";
  try {
    row_frame.resize((size_t)seg_ptr[n_frames] + n_frames);
  } catch (const std::bad_alloc&) {
    return "seg_ptr has more rows than host memory holds";
  }
  for (int f = 0; f < n_frames; f++)
    for (int r = seg_ptr[f] + f; r <= seg_ptr[f + 1] + f; r++) row_frame[r] = f;
  return nullptr;
}

// ---- lines (pus_lines.cu) ----
namespace lines {
struct Dims {
  int W, H, C, ds, w, h;          // input size and channels, halving, detection size
  long long N, n;                 // input and detection pixels per frame
  int plim, clim, hcap, nslot;    // pix_limit, chain_limit, half_cap, line_slots of n
};
Dims make_dims(int width, int height, int channels, int downsample);
// NULL when the detector takes frames of this shape, else why not
const char* shape_error(int width, int height, int channels, int downsample);
struct Work {   // the detector's buffers; st / fc are each frame's status and line count after detect()
  unsigned char *grey, *lut, *i8, *b8;
  unsigned short *h16, *rec;
  short *dx, *dy, *g;
  int *hist, *anc, *nanc, *p1, *p2, *s1, *s2, *cpx, *sid, *st, *nc, *cc, *fc;
  unsigned* bits;
  float* slots;
};
// grey .. per-frame counts of n_frames images (d_img [n][H][W][C])
cudaError_t detect(cudaStream_t st, Alloc& A, int n_frames, const Dims& D, const unsigned char* d_img, Work& W);
// the frames' lines packed at d_first[f] (rows) into d_out
cudaError_t scatter(cudaStream_t st, int n_frames, const Dims& D, const Work& W, const long long* d_first, float* d_out);
}  // namespace lines

// ---- ground edges (pus_popup.cu) ----
namespace edges {
struct Frame {   // one frame's scratch and output slots
  long long node, obj, cpt, line, ivl, tab;
  int node_cap, obj_cap, cpt_cap, ivl_cap, l0, n;
};
struct Maps {    // the preprocessed label maps and each frame's marching-squares segment count
  int w, h;
  unsigned char* map;
  int* seg_count;
};
// label preprocessing and segment counts of d_labels [n][height][width]
cudaError_t prep(cudaStream_t st, Alloc& A, int n_frames, const unsigned char* d_labels, int width, int height,
                 const pus_edge_params& P, Maps& M);
// the frames' selection; tot = the Frame table's node, obj, cpt, ivl totals, n_lines the rows the line slots span.
// out[4 f] = status, open count, connected count, branch bits; open / connected rows and open_in_connect go to the
// frames' slots (8, 16 and 2 values per line from Frame::l0)
cudaError_t select(cudaStream_t st, Alloc& A, int n_frames, const pus_edge_params& P, int width, int height, const Maps& M,
                   const Frame* d_fr, const long long tot[4], long long n_lines, const float* d_lines, float* d_open,
                   float* d_conn, int* d_inc, int* d_out);
}  // namespace edges

// ---- fit and polygons (pus_popup.cu) ----
// popup_kernel over n_rows rows (row_frame [n_rows]); any output may be NULL
cudaError_t launch_fit(cudaStream_t st, int n_frames, const int* d_seg_ptr, const int* d_row_frame, int n_rows,
                       const float* d_segs, const float* d_invK, const float* d_Ts, float dist_thre, int mode, float* d_pw,
                       float* d_ps, float* d_dist, int* d_good, float* d_ends);
namespace poly {
constexpr int kBoundSlot = PUS_POPUP_MAX_VERTICES;   // the ground polygon has n + 6 vertices at most, a wall's 7
constexpr int kWallMax = 7;
constexpr int kHullMax = 34;                          // 6 x 4 edge crossings + 10 corners
constexpr int kCutSlot = kHullMax + 1;
struct Params {
  const int* seg_ptr;
  const int* row_frame;
  int n_rows;
  const float* segs;
  const float* K;
  const float* invK;
  const float* Ts;
  const float* planes;   // [n_rows][4] sensor frame, from popup_kernel
  const float* ends;     // [n_rows][6] world ground endpoints of the wall rows, from popup_kernel
  int width, height;
  float ceiling, walllength;
  float* bound;          // [n_rows][kBoundSlot][2]
  float* cut;            // [n_rows][kCutSlot][2]
  float* world;          // [n_rows][kCutSlot][3]
  int* counts;           // [3][n_rows]: bound, cut, world
};
cudaError_t launch_rows(cudaStream_t st, const Params& P);
// the rows' slots packed at off [3][n_rows] (outputs may be NULL)
cudaError_t launch_pack(cudaStream_t st, const Params& P, const long long* d_off, float* ob, float* oc, float* ow);
}  // namespace poly

// ---- clouds and depth maps (pus_popup.cu) ----
namespace cloud {
struct Job { int frame, v0, n, bx, by, bw, bh, row0; };   // per plane: polygon in vtx[v0 .. v0+n), box, first span row
struct Edge { int x1, y1, major, minor, sy, vert, valid; };
struct Params {
  const Job* jobs;
  const int2* vtx;
  const float* planes;   // [n_planes][4] sensor frame
  const float* Ts;       // [n_frames][16]
  const float* invK;
  const unsigned char* images;   // uploaded only when colours are written
  int width, height, scale, border;   // border: images were given and are 960 wide (matrixToCloud's x < 4 || y < 4 rule)
  float depth_thre, ceiling;
  int2* span;            // [rows]
  int* row_count;        // [rows]
  const long long* row_off;
  float* xyz;
  unsigned char* rgb;
};
// spans and row counts, then row_off [rows + 1] and each plane's count and offset
cudaError_t launch_count(cudaStream_t st, int n_planes, long long rows, const Params& P, long long* d_row_off, int* d_counts,
                         long long* d_offsets);
cudaError_t launch_write(cudaStream_t st, int n_planes, const Params& P);
// label images (already 127 everywhere)
cudaError_t launch_labels(cudaStream_t st, int n_frames, const int* d_plane_ptr, const Params& P, unsigned char* d_labels);
// depth maps [n][height][width] into d_out (d_fill: the fill grid, which is d_out itself without downsample)
cudaError_t launch_depth(cudaStream_t st, int n_frames, int n_planes, const int* d_plane_ptr, const Job* d_jobs,
                         const int2* d_vtx, Edge* d_edges, int2* d_span, const float* d_planes, const float* d_Ts,
                         const float* d_invK, int width, int height, int downsample, float ceiling, float* d_fill,
                         float* d_out);
}  // namespace cloud
}  // namespace pus
