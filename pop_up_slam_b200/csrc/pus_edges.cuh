// pus_edges.cuh -- popup_plane::edge_get_polygons (PUW/libs/select_edge.cpp:66-406) with the two Python stages it calls,
// pop_up_fun.python_get_contours and interval_tree_optimization (pop_up_python/.../pop_up_fun.py:85-205), as __host__
// __device__ code: the label preprocessing rule, the marching-squares case table, the contour assembly and the sequential
// selection passes of one frame.  pus_popup.cu runs it on the device (one thread per frame after the per-pixel kernels);
// the test oracle tests/popup_edges_oracle.cpp compiles the same code for the host.  The pins (scikit-image 0.14's
// find_contours, intervaltree 2.x, NumPy 1.x promotion, OpenCV 4.13's morphology) are stated in include/popup_gpu.h.
#pragma once
#include <math.h>
#include <limits.h>

#include <cmath>
#include <string>

#include "../../include/popup_gpu.h"

#if defined(__CUDACC__)
#define PUS_EHD __host__ __device__
#else
#define PUS_EHD
#endif

namespace pus {
namespace poly {
struct P2 { float x, y; };

// x86 cvttss2si, which the reference's (int) casts compile to: NaN or out of range gives INT_MIN (cvt.rzi saturates)
PUS_EHD inline int trunc_i(float v) {
#if defined(__CUDA_ARCH__)
  return (v >= -2147483648.f && v < 2147483648.f) ? __float2int_rz(v) : INT_MIN;
#else
  return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN;
#endif
}

// direction_hit_boundary (matrix_utils.cpp:229-270, nobottom = false); its lambdas are double expressions rounded to float
PUS_EHD inline P2 hit_boundary(P2 pt, P2 d, int w, int h) {
  if (d.y < 0) {
    const float l = (float)((0.0 - (double)pt.y) / (double)d.y);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.x) && trunc_i(q.x) <= w - 1) return q;
    }
  }
  if (d.y > 0) {
    const float l = (float)(((double)h - 1.0 - (double)pt.y) / (double)d.y);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.x) && trunc_i(q.x) <= w - 1) return q;
    }
  }
  if (d.x > 0) {
    const float l = (float)(((double)w - 1.0 - (double)pt.x) / (double)d.x);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.y) && trunc_i(q.y) <= h - 1) return q;
    }
  }
  if (d.x < 0) {
    const float l = (float)((0.0 - (double)pt.x) / (double)d.x);
    if (l >= 0) {
      const P2 q{pt.x + l * d.x, pt.y + l * d.y};
      if (0 <= trunc_i(q.y) && trunc_i(q.y) <= h - 1) return q;
    }
  }
  return P2{-1.f, -1.f};
}
}  // namespace poly

namespace edges {

// branch bits of a frame (orc_popup_edges_codes and the fixture's "codes")
enum : unsigned {
  B_JOIN_APPEND = 1u << 0,     // assembly: a later contour appended to an earlier one
  B_JOIN_PREPEND = 1u << 1,    // assembly: an earlier contour prepended to a later one
  B_CLOSE = 1u << 2,           // assembly: a contour closed
  B_STALE = 1u << 3,           // assembly: a dict entry of a joined contour was used again (a point shared by chains)
  B_MERGE_END = 1u << 4,       // step 3: seg1's end taken from seg2
  B_MERGE_BEGIN = 1u << 5,     // step 3: seg1's begin taken from seg2
  B_DELETE_COVER = 1u << 6,    // step 4: the less covering one deleted
  B_DELETE_CONTOUR = 1u << 7,  // step 4: both cover much, the one farther from the contour deleted
  B_SPLIT = 1u << 8,           // intervals: split_overlaps split something
  B_DUPLICATE = 1u << 9,       // intervals: a piece with the same bounds removed
  B_PIECE_MERGE = 1u << 10,    // intervals: adjacent pieces of one line merged
  B_REFINE = 1u << 11,         // intervals: a piece's y values refined through int()
  B_SHORT = 1u << 12,          // post: a segment shorter than post_short_thre dropped
  B_BIND = 1u << 13,           // post: two endpoints bound to their int mean
  B_POST_MERGE = 1u << 14,     // post: two successive segments merged
  B_EXTEND_KEPT = 1u << 15,    // post: an extension to the border kept
  B_EXTEND_REVERTED = 1u << 16,// post: an extension reverted (post_extend_thre)
  B_CONNECT = 1u << 17,        // post: connectors inserted
  B_MATERIALIZE = 1u << 18,    // assembly: a joined (dead) contour was written through a stale entry
};

constexpr double kPI = 3.14159265;   // select_edge.cpp:17

struct Lin { float v[4]; };
// an interval of the x-cover tree: [b, e) with the line it came from (intervaltree's Interval(begin, end, data))
struct Ivl { float b, e; Lin d; };

// the angle of a direction in degrees, normalize_to_pi'd (matrix_utils.cpp:495-503).  atan2 is taken in double and rounded
// to float: glibc's atan2f and CUDA's differ, this one definition is used on every side (at most 1 ulp from atan2f)
PUS_EHD inline float angle_deg(float dx, float dy) {
  const float a = (float)atan2((double)dy, (double)dx);
  const float ang = (float)((double)a / kPI * 180.0);
  if (ang > 90) return ang - 180;
  if (ang < -90) return ang + 180;
  return ang;
}
PUS_EHD inline float norm2(float x, float y) { return sqrtf(x * x + y * y); }
PUS_EHD inline float angle_diff(float a, float b) {
  const float d = fabsf(a - b);
  return 180.f - d < d ? 180.f - d : d;   // std::min(diff, 180 - diff)
}

// max over 10 samples of the distance to the nearest contour point (select_edge.cpp:116-122); sample_ind / 10.0 rounds to float
PUS_EHD inline float contour_dist(const Lin& l, const float* cpts, int nc) {
  float mx = 0.f;
  for (int k = 0; k < 10; k++) {
    const float s = (float)(k / 10.0);
    const float px = l.v[0] + s * (l.v[2] - l.v[0]), py = l.v[1] + s * (l.v[3] - l.v[1]);
    float mn = 0.f;
    for (int i = 0; i < nc; i++) {
      const float d = norm2(cpts[2 * i] - px, cpts[2 * i + 1] - py);
      if (i == 0 || d < mn) mn = d;
    }
    if (k == 0 || mn > mx) mx = mn;
  }
  return mx;
}

// point_distproj_to_line / point_dist_line (matrix_utils.cpp:318-350)
PUS_EHD inline void distproj(float bx, float by, float ex, float ey, float qx, float qy, float& dist, float& proj) {
  const float len = norm2(ex - bx, ey - by);
  if ((double)len < 0.001) { dist = norm2(qx - bx, qy - by); proj = -1; return; }
  float t = ((qx - bx) * (ex - bx) + (qy - by) * (ey - by)) / len / len;
  const float px = bx + t * (ex - bx), py = by + t * (ey - by);
  dist = norm2(qx - px, qy - py);
  if (t > 1) t = 1;
  if (t < 0) t = 0;
  proj = t;
}
PUS_EHD inline float dist_line(const float* b, const float* e, const float* q) {
  const float len = norm2(e[0] - b[0], e[1] - b[1]);
  if ((double)len < 0.001) return norm2(q[0] - b[0], q[1] - b[1]);
  const float t = ((q[0] - b[0]) * (e[0] - b[0]) + (q[1] - b[1]) * (e[1] - b[1])) / len / len;
  const float px = b[0] + t * (e[0] - b[0]), py = b[1] + t * (e[1] - b[1]);
  return norm2(q[0] - px, q[1] - py);
}

PUS_EHD inline void remove_row(Lin* a, int& n, int r) {
  for (int i = r; i + 1 < n; i++) a[i] = a[i + 1];
  n--;
}

// ---- stage 1: find_contours(map, 0) of scikit-image 0.14 ---------------------------------------------------------------
// On uint8 data at level 0 every crossing edge has one corner equal to 0, and _get_fraction puts the point on that corner,
// so every contour point is a pixel (key r * w + c).  Per cell the segments (from, to) of the case table with
// fully_connected = 'low'; returns their number (0..2) and writes the keys.  Bits: ul > 0 (1), ur (2), ll (4), lr (8).
PUS_EHD inline int cell_segments(int cs, int r0, int c0, int w, const unsigned char* m, int* seg) {
  if (cs == 0 || cs == 15) return 0;
  const int r1 = r0 + 1, c1 = c0 + 1;
  const bool ul0 = m[r0 * w + c0] == 0, ur0 = m[r0 * w + c1] == 0, ll0 = m[r1 * w + c0] == 0;
  const int top = ul0 ? r0 * w + c0 : r0 * w + c1;
  const int bottom = ll0 ? r1 * w + c0 : r1 * w + c1;
  const int left = ul0 ? r0 * w + c0 : r1 * w + c0;
  const int right = ur0 ? r0 * w + c1 : r1 * w + c1;
  int a[4], n = 0;
  switch (cs) {
    case 1: a[0] = top; a[1] = left; n = 1; break;
    case 2: a[0] = right; a[1] = top; n = 1; break;
    case 3: a[0] = right; a[1] = left; n = 1; break;
    case 4: a[0] = left; a[1] = bottom; n = 1; break;
    case 5: a[0] = top; a[1] = bottom; n = 1; break;
    case 6: a[0] = right; a[1] = top; a[2] = left; a[3] = bottom; n = 2; break;
    case 7: a[0] = right; a[1] = bottom; n = 1; break;
    case 8: a[0] = bottom; a[1] = right; n = 1; break;
    case 9: a[0] = top; a[1] = left; a[2] = bottom; a[3] = right; n = 2; break;
    case 10: a[0] = bottom; a[1] = top; n = 1; break;
    case 11: a[0] = bottom; a[1] = left; n = 1; break;
    case 12: a[0] = left; a[1] = right; n = 1; break;
    case 13: a[0] = top; a[1] = right; n = 1; break;
    default: a[0] = left; a[1] = top; n = 1; break;   // 14
  }
  int k = 0;
  for (int i = 0; i < n; i++)
    if (a[2 * i] != a[2 * i + 1]) { seg[2 * k] = a[2 * i]; seg[2 * k + 1] = a[2 * i + 1]; k++; }   // degenerate: skipped
  return k;
}
PUS_EHD inline int cell_case(const unsigned char* m, int w, int r, int c) {
  return (m[r * w + c] > 0) | (m[r * w + c + 1] > 0) << 1 | (m[(r + 1) * w + c] > 0) << 2 | (m[(r + 1) * w + c + 1] > 0) << 3;
}

// Scratch of one frame's assembly.  _assemble_contours keeps deques in two dicts keyed by point and never deletes an entry
// for good (a pop is always followed by a store under the same key), so a key can point at a contour that has since been
// joined into another one or closed.  Here a contour is a run [first, last] of a singly linked node list; a join splices
// the absorbed contour's nodes into the survivor, which leaves the absorbed run intact and contiguous (lists only grow at
// their ends), so a stale entry still reads the absorbed deque's contents.  A contour that no longer owns its run is copied
// into fresh nodes before it is written (B_MATERIALIZE) or spliced again.
struct Asm {
  int* starts;       // [h * w] contour id or -1
  int* ends;         // [h * w]
  int* node_pt;      // [node_cap]
  int* node_next;    // [node_cap]
  int* c_first;      // [obj_cap]
  int* c_last;
  int* c_len;
  unsigned char* c_owns;
  unsigned char* c_alive;
  int node_cap, obj_cap;
  int n_nodes, n_obj;
  unsigned bits;
  bool overflow;
};

PUS_EHD inline int new_node(Asm& A, int pt) {
  if (A.n_nodes >= A.node_cap) { A.overflow = true; return -1; }
  A.node_pt[A.n_nodes] = pt;
  A.node_next[A.n_nodes] = -1;
  return A.n_nodes++;
}
// give contour c its own copy of its run
PUS_EHD inline bool materialize(Asm& A, int c) {
  if (A.c_owns[c]) return true;
  A.bits |= B_MATERIALIZE;
  int src = A.c_first[c], prev = -1, first = -1;
  for (int i = 0; i < A.c_len[c]; i++) {
    const int nd = new_node(A, A.node_pt[src]);
    if (nd < 0) return false;
    if (prev >= 0) A.node_next[prev] = nd; else first = nd;
    prev = nd;
    src = A.node_next[src];
  }
  A.c_first[c] = first;
  A.c_last[c] = prev;
  A.c_owns[c] = 1;
  return true;
}
PUS_EHD inline bool append(Asm& A, int c, int pt) {
  if (!materialize(A, c)) return false;
  const int nd = new_node(A, pt);
  if (nd < 0) return false;
  A.node_next[A.c_last[c]] = nd;
  A.c_last[c] = nd;
  A.c_len[c]++;
  return true;
}
PUS_EHD inline bool appendleft(Asm& A, int c, int pt) {
  if (!materialize(A, c)) return false;
  const int nd = new_node(A, pt);
  if (nd < 0) return false;
  A.node_next[nd] = A.c_first[c];
  A.c_first[c] = nd;
  A.c_len[c]++;
  return true;
}
PUS_EHD inline int last_pt(const Asm& A, int c) { return A.node_pt[A.c_last[c]]; }
PUS_EHD inline int first_pt(const Asm& A, int c) { return A.node_pt[A.c_first[c]]; }

// one segment of _assemble_contours.  Returns false when the scratch overflowed or the reference raises (a dict pop of a
// key that was never stored: KeyError).
PUS_EHD inline bool assemble_one(Asm& A, int from, int to, bool& raised) {
  const int tail = A.starts[to], head = A.ends[from];
  if (tail >= 0 && head >= 0) {
    if (!A.c_alive[tail] || !A.c_alive[head] || !A.c_owns[tail] || !A.c_owns[head]) A.bits |= B_STALE;
    if (tail == head) {
      A.bits |= B_CLOSE;
      return append(A, head, to);
    }
    if (tail > head) {   // tail created second (numbers follow creation): head.extend(tail)
      A.bits |= B_JOIN_APPEND;
      if (!materialize(A, head)) return false;
      if (!A.c_owns[tail] && !materialize(A, tail)) return false;
      A.node_next[A.c_last[head]] = A.c_first[tail];
      A.c_last[head] = A.c_last[tail];
      A.c_len[head] += A.c_len[tail];
      A.c_owns[tail] = 0;
      const int tl = last_pt(A, tail);
      if (A.ends[tl] < 0) { raised = true; return false; }   // ends.pop(tail[-1])
      A.c_alive[tail] = 0;                                   // contours.pop(tail_num, None)
      A.starts[first_pt(A, head)] = head;
      A.ends[last_pt(A, head)] = head;
    } else {             // tail.extendleft(reversed(head))
      A.bits |= B_JOIN_PREPEND;
      if (!materialize(A, tail)) return false;
      if (!A.c_owns[head] && !materialize(A, head)) return false;
      A.node_next[A.c_last[head]] = A.c_first[tail];
      A.c_first[tail] = A.c_first[head];
      A.c_len[tail] += A.c_len[head];
      A.c_owns[head] = 0;
      const int hf = first_pt(A, head);
      if (A.starts[hf] < 0) { raised = true; return false; }   // starts.pop(head[0])
      A.c_alive[head] = 0;
      A.starts[first_pt(A, tail)] = tail;
      A.ends[last_pt(A, tail)] = tail;
    }
    return true;
  }
  if (tail < 0 && head < 0) {
    if (A.n_obj >= A.obj_cap) { A.overflow = true; return false; }
    const int c = A.n_obj++;
    const int n0 = new_node(A, from), n1 = new_node(A, to);
    if (n1 < 0) return false;
    A.node_next[n0] = n1;
    A.c_first[c] = n0; A.c_last[c] = n1; A.c_len[c] = 2; A.c_owns[c] = 1; A.c_alive[c] = 1;
    A.starts[from] = c;
    A.ends[to] = c;
    return true;
  }
  if (tail >= 0) {
    if (!A.c_alive[tail] || !A.c_owns[tail]) A.bits |= B_STALE;
    if (!appendleft(A, tail, from)) return false;
    A.starts[from] = tail;
    return true;
  }
  if (!A.c_alive[head] || !A.c_owns[head]) A.bits |= B_STALE;
  if (!append(A, head, to)) return false;
  A.ends[to] = head;
  return true;
}

// python_get_contours after the assembly: the live contour with the largest start-end distance (first maximum), (r, c)
// swapped to (x, y), [0:-1:20], doubled with downsample.  Returns the number of points written to pts (at most cap), or -1
// when there is no contour.
PUS_EHD inline int pick_contour(const Asm& A, int w, int scale, float* pts, int cap) {
  int best = -1;
  double bl = -1.0;
  for (int c = 0; c < A.n_obj; c++) {
    if (!A.c_alive[c]) continue;
    const int a = first_pt(A, c), b = last_pt(A, c);
    const double dr = (double)(a / w - b / w), dc = (double)(a % w - b % w);
    const double l = sqrt(dr * dr + dc * dc);
    if (best < 0 || l > bl) { best = c; bl = l; }
  }
  if (best < 0) return -1;
  int n = 0, nd = A.c_first[best];
  const int len = A.c_len[best];
  for (int i = 0; i < len - 1 && n < cap; i++, nd = A.node_next[nd])
    if (i % 20 == 0) {
      const int p = A.node_pt[nd];
      pts[2 * n] = (float)(p % w) * (float)scale;
      pts[2 * n + 1] = (float)(p / w) * (float)scale;
      n++;
    }
  return n;
}

// ---- stages 2-4 ---------------------------------------------------------------------------------------------------------
// Scratch of one frame's selection, for n input lines.  iv, iv2: interval pieces, ivl_cap = 2 n^2 + 2 each: the k <= n
// intervals of the greedy pass have at most 2 k bounds, and split_overlaps gives each of the 2 k - 1 elementary ranges
// one piece per interval containing it.  The pieces that leave the interval stage are at most 2 k - 1 <= 2 n - 1: without
// a split they are the k intervals; after one, the duplicate removal keeps exactly one piece per (begin, end) (the first
// of the longest lines wins all its pairs, every other piece loses to it), and the merges only remove pieces -- but they
// stop after 100 passes, so the pieces can outnumber the input lines.  Hence g, the work rows, and the open rows have
// row_cap = 2 n, the connected rows (at most twice the open ones, less one) 4 n.
struct Sel {
  Lin* g;          // [row_cap]
  int row_cap;
  Ivl* iv;
  Ivl* iv2;
  float* bounds;   // [2 n_lines]
  int ivl_cap;
};

PUS_EHD inline bool lin_eq(const Lin& a, const Lin& b) {
  return a.v[0] == b.v[0] && a.v[1] == b.v[1] && a.v[2] == b.v[2] && a.v[3] == b.v[3];
}
// Interval order of intervaltree 2.x: (begin, end), then the data lists compared element by element
PUS_EHD inline bool ivl_less(const Ivl& a, const Ivl& b) {
  if (a.b != b.b) return a.b < b.b;
  if (a.e != b.e) return a.e < b.e;
  for (int k = 0; k < 4; k++)
    if (a.d.v[k] != b.d.v[k]) return a.d.v[k] < b.d.v[k];
  return false;
}
PUS_EHD inline bool ivl_eq(const Ivl& a, const Ivl& b) { return a.b == b.b && a.e == b.e && lin_eq(a.d, b.d); }
PUS_EHD inline void ivl_sort(Ivl* a, int n) {
  for (int i = 1; i < n; i++) {
    const Ivl x = a[i];
    int j = i - 1;
    while (j >= 0 && ivl_less(x, a[j])) { a[j + 1] = a[j]; j--; }
    a[j + 1] = x;
  }
}
// tree.add(Interval): a set, so an equal interval is not added twice
PUS_EHD inline void ivl_add(Ivl* t, int& n, const Ivl& x) {
  for (int i = 0; i < n; i++)
    if (ivl_eq(t[i], x)) return;
  t[n++] = x;
}

// get_intersect_len_tree: the float64 sum, in sorted order, of the float32 overlaps of the half-open search
PUS_EHD inline double intersect_len(float q0, float q1, const Ivl* t, int n) {
  double s = 0.0;
  if (!(q0 < q1)) return s;   // search(begin >= end) is empty
  // t is kept sorted by the caller
  for (int i = 0; i < n; i++) {
    if (!(t[i].b < q1 && t[i].e > q0)) continue;
    float m = q1 - t[i].b;
    const float o2 = t[i].e - q0, o3 = fabsf(q1 - q0), o4 = t[i].e - t[i].b;
    if (o2 < m) m = o2;
    if (o3 < m) m = o3;
    if (o4 < m) m = o4;
    s += (double)m;
  }
  return s;
}

// The whole selection of one frame.  lines [n][4]; cpts [nc][2] the contour points (already doubled).  Writes the open
// segments to open_out ([n][4] room) and the connected ones to conn_out ([2 n][4]), open_in_conn [n].  Returns the status
// (include/popup_gpu.h) and the counts.
PUS_EHD inline int select_edges(const pus_edge_params& P, int width, int height, const float* lines, int n,
                                const float* cpts, int nc, Sel& S, float* open_out, float* conn_out, int* open_in_conn,
                                int& n_open, int& n_conn, unsigned& bits) {
  n_open = n_conn = 0;
  Lin* g = S.g;
  int m = 0;
  // step 1: length, boundary, vertical
  for (int i = 0; i < n; i++) {
    const float* l = lines + 4 * i;
    const float vx = l[2] - l[0], vy = l[3] - l[1];
    if ((double)norm2(vx, vy) < P.pre_minium_len) continue;
    const double bt = P.pre_boundary_thre;
    if (((double)l[0] < bt && (double)l[2] < bt) || ((double)l[0] > width - bt && (double)l[2] > width - bt) ||
        ((double)l[1] < bt && (double)l[3] < bt) || ((double)l[1] > height - bt && (double)l[3] > height - bt))
      continue;
    const float ang = angle_deg(vx, vy);
    if (!((double)fabsf(fabsf(ang) - 90.f) > P.pre_vertical_thre)) continue;
    // step 2: close to the contour; then x1 <= x2
    Lin L{{l[0], l[1], l[2], l[3]}};
    if (!((double)contour_dist(L, cpts, nc) < P.pre_contour_close_thre)) continue;
    if (L.v[0] > L.v[2]) L = Lin{{l[2], l[3], l[0], l[1]}};
    g[m++] = L;
  }
  // step 3: merge parallel neighbours end to begin
  for (int counter = 0; counter < 100; counter++) {
    bool hit = false;
    for (int s1 = 0; s1 < m && !hit; s1++)
      for (int s2 = s1 + 1; s2 < m; s2++) {
        const float a1 = angle_deg(g[s1].v[2] - g[s1].v[0], g[s1].v[3] - g[s1].v[1]);
        const float a2 = angle_deg(g[s2].v[2] - g[s2].v[0], g[s2].v[3] - g[s2].v[1]);
        if (!((double)angle_diff(a1, a2) < P.pre_merge_angle_thre)) continue;
        const float d12 = norm2(g[s1].v[2] - g[s2].v[0], g[s1].v[3] - g[s2].v[1]);
        const float d21 = norm2(g[s2].v[2] - g[s1].v[0], g[s2].v[3] - g[s1].v[1]);
        if ((double)d12 < P.pre_merge_dist_thre) {
          g[s1].v[2] = g[s2].v[2]; g[s1].v[3] = g[s2].v[3];
          remove_row(g, m, s2);
          bits |= B_MERGE_END;
          hit = true;
          break;
        }
        if ((double)d21 < P.pre_merge_dist_thre) {
          g[s1].v[0] = g[s2].v[0]; g[s1].v[1] = g[s2].v[1];
          remove_row(g, m, s2);
          bits |= B_MERGE_BEGIN;
          hit = true;
          break;
        }
      }
    if (!hit) break;
  }
  // step 4: delete one of two parallel, close, much-overlapping lines
  for (int counter = 0; counter < 100; counter++) {
    bool hit = false;
    for (int s1 = 0; s1 < m && !hit; s1++)
      for (int s2 = s1 + 1; s2 < m; s2++) {
        const float* a = g[s1].v;
        const float* b = g[s2].v;
        const float a1 = angle_deg(a[2] - a[0], a[3] - a[1]), a2 = angle_deg(b[2] - b[0], b[3] - b[1]);
        if (!((double)angle_diff(a1, a2) < P.pre_proj_angle_thre)) continue;
        float d1b, p1b, d1e, p1e, d2b, p2b, d2e, p2e;
        distproj(b[0], b[1], b[2], b[3], a[0], a[1], d1b, p1b);
        distproj(b[0], b[1], b[2], b[3], a[2], a[3], d1e, p1e);
        distproj(a[0], a[1], a[2], a[3], b[0], b[1], d2b, p2b);
        distproj(a[0], a[1], a[2], a[3], b[2], b[3], d2e, p2e);
        const double dt = P.pre_proj_dist_thre;
        if (!((double)d1b < dt && (double)d1e < dt && (double)d2b < dt && (double)d2e < dt)) continue;
        const float c12 = fabsf(p1b - p1e), c21 = fabsf(p2b - p2e);
        if (!((double)c12 > P.pre_proj_cover_thre || (double)c21 > P.pre_proj_cover_thre)) continue;
        int del;
        if ((double)(c21 < c12 ? c21 : c12) < P.pre_proj_cover_large_thre) {
          del = c12 > c21 ? s2 : s1;
          bits |= B_DELETE_COVER;
        } else {
          const float bd0 = contour_dist(g[s1], cpts, nc), bd1 = contour_dist(g[s2], cpts, nc);
          del = bd0 > bd1 ? s1 : s2;
          bits |= B_DELETE_CONTOUR;
        }
        remove_row(g, m, del);
        hit = true;
        break;
      }
    if (!hit) break;
  }
  if (m == 0) return 2;

  // step 5: interval_tree_optimization
  Ivl* t = S.iv;
  int nt = 0;
  {
    // greedy: longest first, then the longest of those overlapping the cover by less than interval_overlap_thre
    int* open = (int*)S.iv2;   // scratch: the open list of line indices (m ints fit in the pieces array)
    float* len = S.bounds;     // float32 lengths
    for (int i = 0; i < m; i++) { open[i] = i; len[i] = norm2(g[i].v[2] - g[i].v[0], g[i].v[3] - g[i].v[1]); }
    int no = m;
    int best = 0;
    for (int i = 1; i < no; i++)
      if (len[open[i]] > len[open[best]]) best = i;
    int cur = open[best];
    for (int i = best; i + 1 < no; i++) open[i] = open[i + 1];
    no--;
    while (true) {
      const Lin& L = g[cur];
      if (!(L.v[0] < L.v[2])) return 3;   // a null or reversed Interval
      ivl_add(t, nt, Ivl{L.v[0], L.v[2], L});
      ivl_sort(t, nt);
      if (no == 0) break;
      int bi = -1;
      for (int i = 0; i < no; i++) {
        const Lin& q = g[open[i]];
        if (intersect_len(q.v[0], q.v[2], t, nt) < P.interval_overlap_thre)
          if (bi < 0 || len[open[i]] > len[open[bi]]) bi = i;
      }
      if (bi < 0) break;
      cur = open[bi];
      for (int i = bi; i + 1 < no; i++) open[i] = open[i + 1];
      no--;
    }
  }
  const int raw_seg = nt;
  // split_overlaps: every pair of successive boundaries, every interval containing the lower one
  int nb = 0;
  for (int i = 0; i < nt; i++) {
    const float e2[2] = {t[i].b, t[i].e};
    for (int k = 0; k < 2; k++) {
      bool seen = false;
      for (int j = 0; j < nb; j++) seen |= S.bounds[j] == e2[k];
      if (!seen) S.bounds[nb++] = e2[k];
    }
  }
  if (nb > 2) {
    for (int i = 1; i < nb; i++) {
      const float x = S.bounds[i];
      int j = i - 1;
      while (j >= 0 && x < S.bounds[j]) { S.bounds[j + 1] = S.bounds[j]; j--; }
      S.bounds[j + 1] = x;
    }
    int n2 = 0;
    for (int k = 0; k + 1 < nb; k++)
      for (int i = 0; i < nt; i++)
        if (t[i].b <= S.bounds[k] && S.bounds[k] < t[i].e) {
          if (n2 >= S.ivl_cap) return 5;
          ivl_add(S.iv2, n2, Ivl{S.bounds[k], S.bounds[k + 1], t[i].d});
        }
    for (int i = 0; i < n2; i++) t[i] = S.iv2[i];
    nt = n2;
    ivl_sort(t, nt);
  }
  const bool post = nt != raw_seg;
  if (post) {
    bits |= B_SPLIT;
    // pieces with the same bounds: the one of the shorter line (x extent, in double) goes
    unsigned char* del = (unsigned char*)S.iv2;
    for (int i = 0; i < nt; i++) del[i] = 0;
    for (int i = 0; i < nt; i++)
      for (int j = i + 1; j < nt; j++)
        if (t[i].b == t[j].b && t[i].e == t[j].e) {
          if ((double)t[i].d.v[2] - (double)t[i].d.v[0] < (double)t[j].d.v[2] - (double)t[j].d.v[0]) del[i] = 1;
          else del[j] = 1;
        }
    int k = 0;
    for (int i = 0; i < nt; i++)
      if (!del[i]) t[k++] = t[i];
      else bits |= B_DUPLICATE;
    nt = k;
    // adjacent pieces of the same line
    for (int counter = 0; counter < 100; counter++) {
      bool hit = false;
      for (int i = 0; i < nt && !hit; i++)
        for (int j = i + 1; j < nt; j++)
          if ((t[i].b == t[j].e || t[i].e == t[j].b) && lin_eq(t[i].d, t[j].d)) {
            const Ivl mg{t[i].b < t[j].b ? t[i].b : t[j].b, t[i].e > t[j].e ? t[i].e : t[j].e, t[j].d};
            for (int q = j; q + 1 < nt; q++) t[q] = t[q + 1];
            nt--;
            for (int q = i; q + 1 < nt; q++) t[q] = t[q + 1];
            nt--;
            ivl_add(t, nt, mg);
            ivl_sort(t, nt);
            bits |= B_PIECE_MERGE;
            hit = true;
            break;
          }
      if (!hit) break;
    }
  }
  // refinement (float64, as NumPy 1.x promotes a float32 scalar with a Python float) and the float32 rows
  Lin* o = g;   // the selection rows are no longer needed
  int no = 0;
  if (nt > S.row_cap) return 5;   // excluded by the bound above; checked so that no row is written out of its slot
  for (int i = 0; i < nt; i++) {
    const Lin& d = t[i].d;
    if (post && (t[i].b != d.v[0] || t[i].e != d.v[2])) {
      const double dx = (double)d.v[2] - (double)d.v[0], dy = (double)d.v[3] - (double)d.v[1];
      const double f1 = ((double)t[i].b - (double)d.v[0]) / dx, f2 = ((double)t[i].e - (double)d.v[0]) / dx;
      o[no++] = Lin{{t[i].b, (float)(long long)(f1 * dy + (double)d.v[1]), t[i].e, (float)(long long)(f2 * dy + (double)d.v[1])}};
      bits |= B_REFINE;
    } else {
      o[no++] = d;
    }
  }

  // step 6: post-processing
  int k = 0;
  for (int i = 0; i < no; i++)
    if ((double)norm2(o[i].v[2] - o[i].v[0], o[i].v[3] - o[i].v[1]) > P.post_short_thre) o[k++] = o[i];
    else bits |= B_SHORT;
  no = k;
  if (no == 0) return 4;
  for (int counter = 0; counter < 100; counter++) {
    bool hit = false;
    for (int s = 0; s + 1 < no; s++)
      if (o[s].v[2] != o[s + 1].v[0] || o[s].v[3] != o[s + 1].v[1])
        if ((double)norm2(o[s].v[2] - o[s + 1].v[0], o[s].v[3] - o[s + 1].v[1]) < P.post_bind_dist_thre) {
          const int mx = poly::trunc_i((o[s].v[2] + o[s + 1].v[0]) / 2.f), my = poly::trunc_i((o[s].v[3] + o[s + 1].v[1]) / 2.f);
          o[s].v[2] = (float)mx; o[s].v[3] = (float)my;
          o[s + 1].v[0] = (float)mx; o[s + 1].v[1] = (float)my;
          bits |= B_BIND;
          hit = true;
        }
    if (!hit) break;
  }
  for (int counter = 0; counter < 100; counter++) {
    bool hit = false;
    for (int s = 0; s + 1 < no; s++) {
      const float* a = o[s].v;
      const float* b = o[s + 1].v;
      const float a1 = angle_deg(a[2] - a[0], a[3] - a[1]), a2 = angle_deg(b[2] - b[0], b[3] - b[1]);
      if (!((double)angle_diff(a1, a2) < P.post_merge_angle_thre)) continue;
      const double mt = P.post_merge_dist_thre;
      const bool c1 = (double)dist_line(b, b + 2, a) < mt, c2 = (double)dist_line(b, b + 2, a + 2) < mt;
      const bool c3 = (double)dist_line(a, a + 2, b) < mt, c4 = (double)dist_line(a, a + 2, b + 2) < mt;
      if ((c1 && c2) || (c3 && c4)) {
        o[s].v[2] = b[2]; o[s].v[3] = b[3];
        remove_row(o, no, s + 1);
        bits |= B_POST_MERGE;
        hit = true;
        break;
      }
    }
    if (!hit) break;
  }
  // extend the first and the last segment to the border, keep it only if it stays close to the contour
  {
    Lin& f = o[0];
    Lin& l = o[no - 1];
    const float os[2] = {f.v[0], f.v[1]}, oe[2] = {l.v[2], l.v[3]};
    const poly::P2 ns = poly::hit_boundary(poly::P2{f.v[2], f.v[3]}, poly::P2{f.v[0] - f.v[2], f.v[1] - f.v[3]}, width, height);
    const poly::P2 ne = poly::hit_boundary(poly::P2{l.v[0], l.v[1]}, poly::P2{l.v[2] - l.v[0], l.v[3] - l.v[1]}, width, height);
    f.v[0] = (float)poly::trunc_i(ns.x); f.v[1] = (float)poly::trunc_i(ns.y);
    l.v[2] = (float)poly::trunc_i(ne.x); l.v[3] = (float)poly::trunc_i(ne.y);
    const float bd0 = contour_dist(o[0], cpts, nc), bd1 = contour_dist(o[no - 1], cpts, nc);
    if ((double)bd0 > P.post_extend_thre) { o[0].v[0] = os[0]; o[0].v[1] = os[1]; bits |= B_EXTEND_REVERTED; }
    else bits |= B_EXTEND_KEPT;
    if ((double)bd1 > P.post_extend_thre) { o[no - 1].v[2] = oe[0]; o[no - 1].v[3] = oe[1]; bits |= B_EXTEND_REVERTED; }
    else bits |= B_EXTEND_KEPT;
  }
  // connectors between segments that do not meet
  n_open = no;
  int nc2 = 0;
  for (int s = 0; s < no; s++) {
    if (s > 0 && (o[s - 1].v[2] != o[s].v[0] || o[s - 1].v[3] != o[s].v[1])) {
      const float c[4] = {o[s - 1].v[2], o[s - 1].v[3], o[s].v[0], o[s].v[1]};
      for (int q = 0; q < 4; q++) conn_out[4 * nc2 + q] = c[q];
      nc2++;
      bits |= B_CONNECT;
    }
    for (int q = 0; q < 4; q++) { open_out[4 * s + q] = o[s].v[q]; conn_out[4 * nc2 + q] = o[s].v[q]; }
    open_in_conn[s] = nc2++;
  }
  n_conn = nc2;
  return 0;
}

// ---- stage 0 and the frame driver ---------------------------------------------------------------------------------------
// The map after the resize (source pixel min(2 x, w - 1), min(2 y, h - 1) of cv::resize 0.5x INTER_NEAREST)
PUS_EHD inline int half_size(int n) {   // cvRound(n * 0.5): half to even
  const int q = n / 2;
  return (n & 1) ? q + (q & 1) : q;
}
// one separable pass of the k x k box (anchor k / 2; pixels outside the image take no part): along x when horiz, max when
// dilate.  src is the previous pass's map, or the label map itself (with the 0.5x pick when ds) when labels != 0.
PUS_EHD inline unsigned char box_pass(const unsigned char* src, int sw, int sh, int ds, int w, int h, int x, int y, int k,
                                      bool horiz, bool dilate) {
  const int a = k / 2;
  int v = dilate ? 0 : 255;
  for (int j = 0; j < k; j++) {
    int xx = x, yy = y;
    if (horiz) xx = x + j - a; else yy = y + j - a;
    if (xx < 0 || yy < 0 || xx >= w || yy >= h) continue;
    const int sx = ds ? (2 * xx < sw - 1 ? 2 * xx : sw - 1) : xx, sy = ds ? (2 * yy < sh - 1 ? 2 * yy : sh - 1) : yy;
    const int u = src[(long long)sy * sw + sx];
    v = dilate ? (u > v ? u : v) : (u < v ? u : v);
  }
  return (unsigned char)v;
}

// Everything after the preprocessing for one frame: the marching-squares scan in row-major cell order, the assembly, the
// contour pick and the selection.  map [h][w] is the preprocessed (255 - v) map; A's tables must hold -1.  Returns the status.
PUS_EHD inline int frame_edges(const pus_edge_params& P, int width, int height, const unsigned char* map, int w, int h,
                               Asm& A, float* cpts, int cpt_cap, const float* lines, int n, Sel& S, float* open_out,
                               float* conn_out, int* open_in_conn, int& n_open, int& n_conn, unsigned& bits) {
  n_open = n_conn = 0;
  bool raised = false;
  for (int r = 0; r + 1 < h; r++)
    for (int c = 0; c + 1 < w; c++) {
      const int cs = cell_case(map, w, r, c);
      int seg[4];
      const int ns = cell_segments(cs, r, c, w, map, seg);
      for (int i = 0; i < ns; i++)
        if (!assemble_one(A, seg[2 * i], seg[2 * i + 1], raised)) { bits |= A.bits; return A.overflow ? 5 : 1; }
    }
  bits |= A.bits;
  const int nc = pick_contour(A, w, P.downsample_contour ? 2 : 1, cpts, cpt_cap);
  if (nc <= 0) return 1;
  return select_edges(P, width, height, lines, n, cpts, nc, S, open_out, conn_out, open_in_conn, n_open, n_conn, bits);
}

// marching-squares segments of a frame's cell (for the scratch size)
PUS_EHD inline int cell_count(const unsigned char* map, int w, int r, int c) {
  int seg[4];
  return cell_segments(cell_case(map, w, r, c), r, c, w, map, seg);
}
// scratch sizes of a frame with ns segments and n lines
PUS_EHD inline long long node_cap_of(long long ns) { return 4 * ns + 64; }
PUS_EHD inline long long obj_cap_of(long long ns) { return ns + 1; }
PUS_EHD inline long long cpt_cap_of(long long ns) { return node_cap_of(ns) / 20 + 2; }
PUS_EHD inline long long ivl_cap_of(long long n) { return 2 * n * n + 2; }

// the frame size and pus_edge_params rules of pus_popup_edges, shared with the pop-up session's config check; "" when they pass
inline std::string shape_error(int width, int height, const pus_edge_params* params) {
  if (width < 4 || height < 4) return "width and height must be at least 4";
  if (!params) return "params must be given";
  if (!params->downsample_contour && (params->dilation_distance < 1 || params->erosion_distance < 1))
    return "dilation_distance and erosion_distance must be at least 1";
  return "";
}
// the checks of pus_popup_edges' arguments, shared with the test oracle's restatement of the call; "" when they pass
inline std::string args_error(int n_frames, const unsigned char* labels, int width, int height, const int* line_ptr,
                            const float* lines, const pus_edge_params* params, const int* status, const int* open_counts,
                            const int* connect_counts) {
  if (n_frames < 0) return "n_frames < 0";
  if (!line_ptr || line_ptr[0] != 0) return "line_ptr must be given and start at 0";
  for (int f = 0; f < n_frames; f++) {
    const int n = line_ptr[f + 1] - line_ptr[f];
    if (n < 0) return "line_ptr is not ascending";
    if (n > PUS_POPUP_MAX_LINES) return "a frame has more than PUS_POPUP_MAX_LINES lines";
  }
  const std::string why = shape_error(width, height, params);
  if (!why.empty()) return why;
  if (n_frames > 0 && !labels) return "labels must be given";
  const int n = line_ptr[n_frames];
  if (n > 0 && !lines) return "lines must be given";
  for (long long i = 0; i < 4LL * n; i++)
    if (!std::isfinite(lines[i])) return "a line coordinate is not finite";
  if (!status || !open_counts || !connect_counts) return "status and the count arrays must be given";
  return "";
}
}  // namespace edges
}  // namespace pus
