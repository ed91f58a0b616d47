// pus_stages.cuh -- the pop-up stages' internal launchers: device pointers in, kernels enqueued on a stream.  The extern "C"
// stage calls (pus_popup.cu, pus_lines.cu) and the pop-up session (pus_frames.cu) launch the same kernels through these.
// Scratch comes from an Alloc: the stage calls free theirs on return (TempAlloc), the session keeps grow-only buffers.
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "../../include/popup_gpu.h"

namespace pus {

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
};
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

// ---- lines (pus_lines.cu) ----
namespace lines {
struct Dims {
  int W, H, C, ds, w, h;          // input size and channels, halving, detection size
  long long N, n;                 // input and detection pixels per frame
  int plim, clim, hcap, nslot;    // pix_limit, chain_limit, half_cap, line_slots of n
};
Dims make_dims(int width, int height, int channels, int downsample);
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
