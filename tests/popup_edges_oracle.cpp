// CPU oracle of pus_popup_edges: the call restated on the host around the frame code of pus_edges.cuh, which the device
// runs one thread per frame.  The independent restatement of the stages is tools/make_popup_edge_golden.py (its fixture
// is compared with this oracle bit for bit); this file checks the device's per-pixel passes, scratch layout and packing.
// Exports orc_popup_edges (the C-ABI), orc_popup_edges_codes (per-frame branch bits), orc_edges_preprocess (stage 0) and
// orc_edges_contour (stage 1 on a preprocessed map).
#include <cstring>
#include <string>
#include <vector>

#include "../pop_up_slam_b200/csrc/pus_edges.cuh"

using namespace pus::edges;

static thread_local std::string g_orc_err;

namespace {
// stage 0: [h][w] preprocessed map of one frame
void preprocess(const unsigned char* lab, int W, int H, const pus_edge_params& P, std::vector<unsigned char>& out, int& w, int& h) {
  const int ds = P.downsample_contour ? 1 : 0;
  w = ds ? half_size(W) : W;
  h = ds ? half_size(H) : H;
  const int kd = ds ? 8 : P.dilation_distance, ke = ds ? 8 : P.erosion_distance;
  std::vector<unsigned char> a((size_t)w * h), b((size_t)w * h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) a[(size_t)y * w + x] = box_pass(lab, W, H, ds, w, h, x, y, kd, true, true);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) b[(size_t)y * w + x] = box_pass(a.data(), w, h, 0, w, h, x, y, kd, false, true);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) a[(size_t)y * w + x] = box_pass(b.data(), w, h, 0, w, h, x, y, ke, true, false);
  out.resize((size_t)w * h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) out[(size_t)y * w + x] = 255 - box_pass(a.data(), w, h, 0, w, h, x, y, ke, false, false);
}

struct AsmStore {
  std::vector<int> tab, nodes, objs;
  std::vector<unsigned char> flags;
  Asm A;
  AsmStore(const unsigned char* map, int w, int h) {
    long long ns = 0;
    for (int r = 0; r + 1 < h; r++)
      for (int c = 0; c + 1 < w; c++) ns += cell_count(map, w, r, c);
    const int nc = (int)node_cap_of(ns), oc = (int)obj_cap_of(ns);
    tab.assign(2 * (size_t)w * h, -1);
    nodes.assign(2 * (size_t)nc, 0);
    objs.assign(3 * (size_t)oc, 0);
    flags.assign(2 * (size_t)oc, 0);
    A = Asm{tab.data(), tab.data() + (size_t)w * h, nodes.data(), nodes.data() + nc, objs.data(), objs.data() + oc,
            objs.data() + 2 * oc, flags.data(), flags.data() + oc, nc, oc, 0, 0, 0u, false};
  }
};

// one frame: status, rows and bits
int frame(const unsigned char* lab, int W, int H, const float* lines, int n, const pus_edge_params& P, std::vector<float>& open,
          std::vector<float>& conn, std::vector<int>& inc, int& n_open, int& n_conn, unsigned& bits) {
  std::vector<unsigned char> map;
  int w, h;
  preprocess(lab, W, H, P, map, w, h);
  AsmStore st(map.data(), w, h);
  std::vector<float> cpts(2 * (size_t)(st.A.node_cap / 20 + 2));
  const int rc = 2 * (n > 0 ? n : 1);   // Sel::row_cap
  std::vector<Lin> rows(rc);
  std::vector<float> bounds(2 * (size_t)(n > 0 ? n : 1));
  const long long cap = ivl_cap_of(n);
  std::vector<Ivl> iv((size_t)cap), iv2((size_t)cap);
  Sel S{rows.data(), rc, iv.data(), iv2.data(), bounds.data(), (int)cap};
  open.assign(4 * (size_t)rc, 0.f);
  conn.assign(8 * (size_t)rc, 0.f);
  inc.assign(rc, 0);
  bits = 0;
  const int s = frame_edges(P, W, H, map.data(), w, h, st.A, cpts.data(), (int)cpts.size() / 2, lines, n, S, open.data(),
                            conn.data(), inc.data(), n_open, n_conn, bits);
  if (s) n_open = n_conn = 0;
  return s;
}
}  // namespace

extern "C" {
const char* orc_popup_last_error(void) { return g_orc_err.c_str(); }

int orc_popup_edges(int device, int n_frames, const unsigned char* labels, int width, int height, const int* line_ptr,
                    const float* lines, const pus_edge_params* params, int* status, int* open_counts, int* connect_counts,
                    float* open_segs, float* connect_segs, int* open_in_connect, long long open_capacity,
                    long long connect_capacity) {
  (void)device;
  const std::string why = args_error(n_frames, labels, width, height, line_ptr, lines, params, status, open_counts,
                                     connect_counts);
  if (!why.empty()) { g_orc_err = "orc_popup_edges: " + why; return -1; }
  std::vector<std::vector<float>> O(n_frames), Cn(n_frames);
  std::vector<std::vector<int>> I(n_frames);
  long long to = 0, tc = 0;
  int found = 0;
  for (int f = 0; f < n_frames; f++) {
    unsigned bits;
    status[f] = frame(labels + (size_t)f * width * height, width, height, lines + 4 * (size_t)line_ptr[f],
                      line_ptr[f + 1] - line_ptr[f], *params, O[f], Cn[f], I[f], open_counts[f], connect_counts[f], bits);
    to += open_counts[f];
    tc += connect_counts[f];
    found += status[f] == 0;
  }
  if ((open_segs && open_capacity < to) || (connect_segs && connect_capacity < tc)) {
    g_orc_err = "orc_popup_edges: a capacity is smaller than its number of segments";
    return -1;
  }
  long long po = 0, pc = 0;
  for (int f = 0; f < n_frames; f++) {
    if (open_segs) std::memcpy(open_segs + 4 * po, O[f].data(), 4 * (size_t)open_counts[f] * sizeof(float));
    if (open_segs && open_in_connect) std::memcpy(open_in_connect + po, I[f].data(), (size_t)open_counts[f] * sizeof(int));
    if (connect_segs) std::memcpy(connect_segs + 4 * pc, Cn[f].data(), 4 * (size_t)connect_counts[f] * sizeof(float));
    po += open_counts[f];
    pc += connect_counts[f];
  }
  return found;
}

// per-frame branch bits (pus_edges.cuh B_*) of the same batch; returns 0 or -1
int orc_popup_edges_codes(int n_frames, const unsigned char* labels, int width, int height, const int* line_ptr,
                          const float* lines, const pus_edge_params* params, int* bits_out) {
  for (int f = 0; f < n_frames; f++) {
    std::vector<float> o, c;
    std::vector<int> i;
    int no, nc;
    unsigned bits;
    frame(labels + (size_t)f * width * height, width, height, lines + 4 * (size_t)line_ptr[f], line_ptr[f + 1] - line_ptr[f],
          *params, o, c, i, no, nc, bits);
    bits_out[f] = (int)bits;
  }
  return 0;
}

// stage 0 of one frame into out (room for width * height); returns w << 16 | h of the preprocessed map
int orc_edges_preprocess(const unsigned char* lab, int width, int height, const pus_edge_params* params, unsigned char* out) {
  std::vector<unsigned char> m;
  int w, h;
  preprocess(lab, width, height, *params, m, w, h);
  std::memcpy(out, m.data(), m.size());
  return w << 16 | h;
}

// stage 1 on a preprocessed [h][w] map: the kept contour's points (x, y, every 20th, times scale) into pts (room for cap);
// returns their number, -1 without a contour, -2 when the assembly raises or runs out of scratch
int orc_edges_contour(const unsigned char* map, int w, int h, int scale, float* pts, int cap) {
  AsmStore st(map, w, h);
  bool raised = false;
  for (int r = 0; r + 1 < h; r++)
    for (int c = 0; c + 1 < w; c++) {
      int seg[4];
      const int ns = cell_segments(cell_case(map, w, r, c), r, c, w, map, seg);
      for (int i = 0; i < ns; i++)
        if (!assemble_one(st.A, seg[2 * i], seg[2 * i + 1], raised)) return -2;
    }
  return pick_contour(st.A, w, scale, pts, cap);
}
}
