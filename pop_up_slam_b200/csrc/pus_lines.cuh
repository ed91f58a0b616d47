// pus_lines.cuh -- the order-dependent part of line_lbd's EDLines detector (binary_descriptor.cpp:1579-2626,
// descriptor.hpp:649-844, OctaveKeyLines :1061-1140) as __host__ __device__ code: the edge-drawing walk of one frame, the
// assembly of its chains, and the line extraction, validation and orientation of one chain.  pus_lines.cu runs it on the
// device (one thread per frame for the walk, one per chain for the lines, after the per-pixel kernels); the test oracle
// tests/popup_lines_oracle.cpp compiles the same code for the host.  The pins are stated in include/popup_gpu.h.
#pragma once
#include <math.h>

#include "../../include/popup_gpu.h"

#if defined(__CUDACC__)
#define PUS_LHD __host__ __device__
#else
#define PUS_LHD
#endif

namespace pus {
namespace lines {
// EDLineDetector() defaults and binary_descriptor.cpp:58-65
constexpr int kGradThr = 80, kAnchorThr = 8, kMinLen = 15, kTryTime = 6, kSkip = 2;
constexpr double kFitErr = 1.6;
constexpr double kPi = 3.14159265358979323846;   // M_PI
enum { kUp = 1, kRight = 2, kDown = 3, kLeft = 4 };

// One record per pixel, all the walk reads in one load: the gradient's low byte (what the neighbour comparisons see
// through (unsigned char)), g > 0 (the loop condition on the full short), the direction (|dx| < |dy|: Horizontal), the
// walk's mark, and a bit for the branch record (marked by a chain that was then dropped).  After the 5 x 5 blur the
// gradient of 8-bit data is at most 237 (|dx| + |dy| <= 949), so the low byte is the value; the walk still reads it.
enum : unsigned short { kLow = 0xff, kPos = 0x100, kHoriz = 0x200, kMark = 0x400, kDropped = 0x800 };

PUS_LHD inline unsigned short pack(int g, bool horiz) {
  return (unsigned short)((g & 0xff) | (g > 0 ? kPos : 0) | (horiz ? kHoriz : 0));
}

// Branch bits of one frame (the oracle reports them; the fixture's union covers every bit).
enum : unsigned {
  B_EQUALIZED = 1u << 0,     // mean < 90: equalizeHist applied
  B_ONE_BIN = 1u << 1,       // equalizeHist on a one-value image (identity)
  B_TURN = 1u << 2,          // a walk changed between horizontal and vertical stepping
  B_BORDER = 1u << 3,        // a walk stopped at the image border
  B_SHORT = 1u << 4,         // a chain shorter than 16 pixels was dropped (its pixels stay marked)
  B_BLOCKED = 1u << 5,       // a walk stopped at a pixel of a dropped chain
  B_FIT_FAIL = 1u << 6,      // an initial fit failed its error threshold (skip 2)
  B_FIT_NAN = 1u << 7,       // an initial fit was singular (NaN fails every comparison)
  B_POPBACK = 1u << 8,       // outliers were popped back to the chain
  B_TRYCAP = 1u << 9,       // an extension stopped at TryTime while still growing
  B_BORDER_LINE = 1u << 10,  // a line rejected as an image-border line
  B_NFA_REJECT = 1u << 11,   // a line rejected by its NFA
  B_NFA_NK = 1u << 12,       // nfa with n == k
  B_NFA_ZERO = 1u << 13,     // nfa's first term almost zero
  B_ZERO_GRAD = 1u << 14,    // a line with zero mean gradient (rejected)
  B_SWAP_Q0 = 1u << 15,      // endpoints swapped, direction in [-3pi/4, -pi/4)
  B_SWAP_Q1 = 1u << 16,      //   [-pi/4, pi/4)
  B_SWAP_Q2 = 1u << 17,      //   [pi/4, 3pi/4)
  B_SWAP_Q3 = 1u << 18,      //   [3pi/4, pi) or [-pi, -3pi/4)
  B_FLOAT_PI = 1u << 19,     // |direction| rounded to float pi lies beyond M_PI: no range taken
  B_OVER_ANCHORS = 1u << 20, // status 1: more anchors than N/5
  B_OVER_CHAINS = 1u << 21,  // status 1: more chains than N/100
  B_OVER_PIXELS = 1u << 22,  // status 1: more edge pixels in a half than N/5
  B_LINE_H = 1u << 23,       // a line fitted as y = ax + b
  B_LINE_V = 1u << 24,       // a line fitted as x = ay + b
  B_MANY = 1u << 25,         // more than PUS_POPUP_MAX_LINES lines in the frame
  B_HALVED = 1u << 26,       // detected on the 0.5x image
  B_ALL = (1u << 27) - 1
};

// EdgeDrawing's limits (binary_descriptor.cpp:1585-1586) for a w x h image: anchors and edge pixels per half N / 5,
// chains (N / 5) / 20.
PUS_LHD inline long long pix_limit(long long n) { return (unsigned)n / 5u; }
PUS_LHD inline long long chain_limit(long long n) { return ((unsigned)n / 5u) / 20u; }
// The walk's scratch per half: the limit plus the 16 pixels a chain may hold while it is still short (a chain that
// reaches past this is kept, and its half has then overflowed).
PUS_LHD inline long long half_cap(long long n) { return pix_limit(n) + kMinLen + 1; }
// Line slots of a chain that starts at pixel s of its frame's chain array: a line takes at least kMinLen pixels.
PUS_LHD inline long long line_slot(long long s, int chain) { return s / kMinLen + chain; }
PUS_LHD inline long long line_slots(long long n) { return 2 * half_cap(n) / kMinLen + chain_limit(n) + 2; }

struct Walk {
  unsigned short* rec;   // [h][w] records
  int w, h;
  int* p1;               // first halves (pixel indices), half_cap entries
  int* p2;               // second halves
  int* s1;               // chain starts in p1 / p2, chain_limit + 1 entries
  int* s2;
};

// One half-walk from (x, y) (binary_descriptor.cpp:1714-1857; the four copies there differ only in the first direction).
// Returns false when the half's scratch is full (the chain is then kept and has overflowed).
PUS_LHD inline bool half_walk(const Walk& W, int x, int y, int last_dir, int& last_x, int& last_y, int* out, int& off,
                              int cap, unsigned& bits) {
  unsigned short* rec = W.rec;
  const int w = W.w, h = W.h;
  int idx = y * w + x;
  for (;;) {
    const unsigned short r = rec[idx];
    if (!(r & kPos)) break;
    if (r & kMark) {
      if (r & kDropped) bits |= B_BLOCKED;
      break;
    }
    if (off >= cap) return false;
    rec[idx] = (unsigned short)(r | kMark);
    out[off++] = idx;
    int should = 0;
    int n1, n2, n3;
    if (r & kHoriz) {
      if (last_dir == kUp || last_dir == kDown) {
        should = x > last_x ? kRight : kLeft;
        bits |= B_TURN;
      }
      last_x = x;
      last_y = y;
      if (last_dir == kRight || should == kRight) {
        if (x == w - 1 || y == 0 || y == h - 1) { bits |= B_BORDER; break; }
        n1 = idx - w + 1; n2 = idx + 1; n3 = idx + w + 1;
        last_dir = kRight;
      } else {
        if (x == 0 || y == 0 || y == h - 1) { bits |= B_BORDER; break; }
        n1 = idx - w - 1; n2 = idx - 1; n3 = idx + w - 1;
        last_dir = kLeft;
      }
    } else {
      if (last_dir == kRight || last_dir == kLeft) {
        should = y > last_y ? kDown : kUp;
        bits |= B_TURN;
      }
      last_x = x;
      last_y = y;
      if (last_dir == kDown || should == kDown) {
        if (x == 0 || x == w - 1 || y == h - 1) { bits |= B_BORDER; break; }
        n1 = idx + w + 1; n2 = idx + w; n3 = idx + w - 1;
        last_dir = kDown;
      } else {
        if (x == 0 || x == w - 1 || y == 0) { bits |= B_BORDER; break; }
        n1 = idx - w + 1; n2 = idx - w; n3 = idx - w - 1;
        last_dir = kUp;
      }
    }
    const int g1 = rec[n1] & kLow, g2 = rec[n2] & kLow, g3 = rec[n3] & kLow;
    // the pick: first neighbour (the diagonal on the up / right side of travel), else the third, else straight on
    const int pick = (g1 >= g2 && g1 >= g3) ? n1 : (g3 >= g2 && g3 >= g1) ? n3 : n2;
    idx = pick;
    x = idx % w;
    y = idx / w;
  }
  return true;
}

// EdgeDrawing's anchor loop and chain assembly (binary_descriptor.cpp:1691-2373) over the anchors in scan order.
// chain_px receives the chains (first half reversed, then the second half without its copy of the anchor), sid[0..n]
// their starts.  Returns 0, or 1 when a half's pixels or the chain count pass the reference's limits.
PUS_LHD inline int draw_edges(const Walk& W, const int* anchors, int n_anchors, int* chain_px, int* sid, int& n_chains,
                              unsigned& bits) {
  const long long n = (long long)W.w * W.h;
  const int cap = (int)half_cap(n), plim = (int)pix_limit(n), clim = (int)chain_limit(n);
  int o1 = 0, o2 = 0, ps = 0, last_x = 0, last_y = 0;
  n_chains = 0;
  for (int i = 0; i < n_anchors; i++) {
    const int a = anchors[i];
    if (W.rec[a] & kMark) continue;
    const int ax = a % W.w, ay = a / W.w;
    W.s1[ps] = o1;
    const bool horiz = (W.rec[a] & kHoriz) != 0;
    if (!half_walk(W, ax, ay, horiz ? kRight : kDown, last_x, last_y, W.p1, o1, cap, bits)) {
      bits |= B_OVER_PIXELS;
      return 1;
    }
    W.rec[a] = (unsigned short)(W.rec[a] & ~kMark);
    W.s2[ps] = o2;
    if (!half_walk(W, ax, ay, horiz ? kLeft : kUp, last_x, last_y, W.p2, o2, cap, bits)) {
      bits |= B_OVER_PIXELS;
      return 1;
    }
    if ((o1 - W.s1[ps]) + (o2 - W.s2[ps]) < kMinLen + 1) {
      bits |= B_SHORT;
      for (int k = W.s1[ps]; k < o1; k++) W.rec[W.p1[k]] |= kDropped;
      for (int k = W.s2[ps]; k < o2; k++) W.rec[W.p2[k]] |= kDropped;
      o1 = W.s1[ps];
      o2 = W.s2[ps];
    } else {
      if (o1 > plim || o2 > plim) { bits |= B_OVER_PIXELS; return 1; }
      if (++ps > clim) { bits |= B_OVER_CHAINS; return 1; }
    }
  }
  W.s1[ps] = o1;
  W.s2[ps] = o2;
  int k = 0;
  for (int c = 0; c < ps; c++) {
    sid[c] = k;
    for (int t = W.s1[c + 1] - 1; t >= W.s1[c]; t--) chain_px[k++] = W.p1[t];
    for (int t = W.s2[c] + 1; t < W.s2[c + 1]; t++) chain_px[k++] = W.p2[t];
  }
  sid[ps] = k;
  n_chains = ps;
  return 0;
}

// ---- line extraction of one chain (EDline, binary_descriptor.cpp:2421-2619) ----
// log Gamma and nfa of descriptor.hpp:694-844
PUS_LHD inline double log_gamma_lanczos(double x) {
  const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424,
                       2.50662827511};
  double a = (x + 0.5) * log(x + 5.5) - (x + 5.5);
  double b = 0.0;
  for (int n = 0; n < 7; n++) {
    a -= log(x + (double)n);
    b += q[n] * pow(x, (double)n);
  }
  return a + log(b);
}
PUS_LHD inline double log_gamma_windschitl(double x) {
  return 0.918938533204673 + (x - 0.5) * log(x) - x + 0.5 * x * log(x * sinh(1 / x) + 1 / (810.0 * pow(x, 6.0)));
}
PUS_LHD inline double log_gamma(double x) { return x > 15.0 ? log_gamma_windschitl(x) : log_gamma_lanczos(x); }
PUS_LHD inline bool double_equal(double a, double b) {
  if (a == b) return true;
  const double abs_diff = fabs(a - b), aa = fabs(a), bb = fabs(b);
  double abs_max = aa > bb ? aa : bb;
  if (abs_max < 2.2250738585072014e-308) abs_max = 2.2250738585072014e-308;
  return (abs_diff / abs_max) <= (100.0 * 2.220446049250313e-16);
}
// n >= 1 and 0 <= k <= n always hold here (n is a line's pixel count)
PUS_LHD inline double nfa(int n, int k, double p, double logNT, unsigned& bits) {
  const double tolerance = 0.1, MLN10 = 2.30258509299404568402;
  if (n == 0 || k == 0) return -logNT;
  if (n == k) {
    bits |= B_NFA_NK;
    return -logNT - (double)n * log10(p);
  }
  const double p_term = p / (1.0 - p);
  const double log1term = log_gamma((double)n + 1.0) - log_gamma((double)k + 1.0) - log_gamma((double)(n - k) + 1.0) +
                          (double)k * log(p) + (double)(n - k) * log(1.0 - p);
  double term = exp(log1term);
  if (double_equal(term, 0.0)) {
    bits |= B_NFA_ZERO;
    if ((double)k > (double)n * p) return -log1term / MLN10 - logNT;
    return -logNT;
  }
  double bin_tail = term;
  for (int i = k + 1; i <= n; i++) {
    const double bin_term = (double)(n - i + 1) / (double)i;
    const double mult_term = bin_term * p_term;
    term *= mult_term;
    bin_tail += term;
    if (bin_term < 1.0) {
      const double err = term * ((1.0 - pow(mult_term, (double)(n - i + 1))) / (1.0 - mult_term) - 1.0);
      if (err < tolerance * fabs(-log10(bin_tail) - logNT) * bin_tail) break;
    }
  }
  return -log10(bin_tail) - logNT;
}

struct Fit {   // ATA (row-major 2 x 2) and ATV of the current line, Mat_<float> as the reference keeps them
  float A[4], V[2];
  double a, b;
};

// The products fitMatT * fitMatT.t() and fitMatT * vec: OpenCV's gemm accumulates in double and rounds to float once;
// the integer terms make the double sums exact.  X is the abscissa of the fit (x for y = ax + b, y for x = ay + b).
PUS_LHD inline void gram(const int* px, int s, int e, int w, bool horiz, float* A, float* V) {
  double sxx = 0, sx = 0, sxy = 0, sy = 0;
  for (int i = s; i < e; i++) {
    const int X = horiz ? px[i] % w : px[i] / w, Y = horiz ? px[i] / w : px[i] % w;
    sxx += (double)X * (double)X;
    sx += (double)X;
    sxy += (double)X * (double)Y;
    sy += (double)Y;
  }
  A[0] = (float)sxx; A[1] = (float)sx; A[2] = (float)sx; A[3] = (float)(e - s);
  V[0] = (float)sxy; V[1] = (float)sy;
}
PUS_LHD inline void solve(Fit& F) {
  const double coef = 1.0 / ((double)F.A[0] * (double)F.A[3] - (double)F.A[1] * (double)F.A[2]);
  F.a = coef * ((double)F.A[3] * (double)F.V[0] - (double)F.A[1] * (double)F.V[1]);
  F.b = coef * ((double)F.A[0] * (double)F.V[1] - (double)F.A[2] * (double)F.V[0]);
}
// LeastSquaresLineFit_ first form (binary_descriptor.cpp:2628-2707): kMinLen pixels from s; returns the fit error
PUS_LHD inline double fit_first(const int* px, int s, int w, bool horiz, Fit& F) {
  gram(px, s, s + kMinLen, w, horiz, F.A, F.V);
  solve(F);
  double err = 0;
  for (int i = s; i < s + kMinLen; i++) {
    const int X = horiz ? px[i] % w : px[i] / w, Y = horiz ? px[i] / w : px[i] % w;
    const double c = (double)Y - (double)X * F.a - F.b;
    err += c * c;
  }
  return sqrt(err);
}
// second form (:2708-2787): ATA += the new pixels' products (a float add)
PUS_LHD inline void fit_more(const int* px, int s, int e, int w, bool horiz, Fit& F) {
  float A[4], V[2];
  gram(px, s, e, w, horiz, A, V);
  for (int i = 0; i < 4; i++) F.A[i] = F.A[i] + A[i];
  F.V[0] = F.V[0] + V[0];
  F.V[1] = F.V[1] + V[1];
  solve(F);
}

// LineValidation_ (:2789-2870); direction as the reference's float
PUS_LHD inline bool validate(const int* px, int s, int e, const short* dx, const short* dy, int w, int h, double logNT,
                             const double* eq, float& direction, unsigned& bits) {
  const int n = e - s;
  int mgx = 0, mgy = 0;
  for (int i = s; i < e; i++) {
    mgx += dx[px[i]];
    mgy += dy[px[i]];
  }
  const double ax = fabs(eq[1]), ay = fabs(eq[0]);
  if (mgx == 0 && mgy == 0) {
    bits |= B_ZERO_GRAD;
    return false;
  }
  if (mgx > 0 && mgy >= 0) direction = (float)atan2(-ay, ax);
  if (mgx <= 0 && mgy > 0) direction = (float)atan2(ay, ax);
  if (mgx < 0 && mgy <= 0) direction = (float)atan2(ay, -ax);
  if (mgx >= 0 && mgy < 0) direction = (float)atan2(-ay, -ax);
  const double ad = fabs((double)direction);
  if (ad < 0.15 || kPi - ad < 0.15) {
    if (fabs(eq[2]) < 10 || fabs((double)h - fabs(eq[2])) < 10) { bits |= B_BORDER_LINE; return false; }
  }
  if (fabs(ad - kPi * 0.5) < 0.15) {
    if (fabs(eq[2]) < 10 || fabs((double)w - fabs(eq[2])) < 10) { bits |= B_BORDER_LINE; return false; }
  }
  int k = 0;
  for (int i = s; i < e; i++) {
    const double pd = atan2(-(double)dx[px[i]], (double)dy[px[i]]);
    const double dis = fabs((double)direction - pd);
    if (fabs(2 * kPi - dis) < 0.392699 || dis < 0.392699) k++;
  }
  if (nfa(n, k, 0.125, logNT, bits) > 0) return true;
  bits |= B_NFA_REJECT;
  return false;
}

// logNT_ of EDline (:2401)
PUS_LHD inline double log_nt(int w, int h) { return 2.0 * (log10((double)w) + log10((double)h)); }

// The lines of one chain px[0..n) (EDline's loop body, :2423-2619) in the order the reference stores them, each
// oriented as OctaveKeyLines does (:1079-1137) and scaled as keylines_to_mat (scale 1 or 2).  out holds n / kMinLen
// rows; returns their number.
PUS_LHD inline int chain_lines(const int* px, int n, const unsigned short* rec, const short* dx, const short* dy, int w,
                               int h, float scale, float* out, unsigned& bits) {
  const double logNT = log_nt(w, h);
  int S = 0, nl = 0;
  double err = 0;
  Fit F;
  while (n > S + kMinLen) {
    while (n > S + kMinLen) {
      err = fit_first(px, S, w, (rec[px[S]] & kHoriz) != 0, F);
      if (err <= kFitErr) break;
      bits |= (err == err) ? B_FIT_FAIL : B_FIT_NAN;
      S += kSkip;
    }
    if (err > kFitErr || err != err) break;
    const int l0 = S;   // the line's pixels are px[l0 .. l) (the reference's copy is this run of the chain)
    const bool horiz = (rec[px[l0]] & kHoriz) != 0;
    int l = l0, new_s = l0, tries = 0;
    double coef1 = 0;
    bool first = true;
    for (;;) {
      tries++;
      if (first) {
        first = false;
        l += kMinLen;
        S += kMinLen;
      } else {
        fit_more(px, new_s, l, w, horiz, F);
      }
      coef1 = horiz ? 1 / sqrt(F.a * F.a + 1) : 1 / sqrt(1 + F.a * F.a);
      int outl = 0;
      new_s = l;
      while (n > S) {
        const double X = px[S] % w, Y = px[S] / w;
        const double d = horiz ? fabs(F.a * X - Y + F.b) * coef1 : fabs(X - F.a * Y - F.b) * coef1;
        S++;
        l++;
        if (d > kFitErr) {
          if (++outl > 3) break;
        } else {
          outl = 0;
        }
      }
      if (outl) bits |= B_POPBACK;
      l -= outl;
      S -= outl;
      if (l - new_s > 0 && tries < kTryTime) continue;
      if (l - new_s > 0) bits |= B_TRYCAP;
      break;
    }
    double eq[3];
    if (horiz) {
      eq[0] = F.a * coef1; eq[1] = -1 * coef1; eq[2] = F.b * coef1;
    } else {
      eq[0] = 1 * coef1; eq[1] = -F.a * coef1; eq[2] = -F.b * coef1;
    }
    float direction = 0;
    if (!validate(px, l0, l, dx, dy, w, h, logNT, eq, direction, bits)) continue;
    bits |= horiz ? B_LINE_H : B_LINE_V;
    const double a1 = eq[1] * eq[1], a2 = eq[0] * eq[0], a3 = eq[0] * eq[1], a4 = eq[2] * eq[0], a5 = eq[2] * eq[1];
    const double P0x = px[l0] % w, P0y = px[l0] / w, P1x = px[l - 1] % w, P1y = px[l - 1] / w;
    const float s1 = (float)(a1 * P0x - a3 * P0y - a4), s2 = (float)(a2 * P0y - a3 * P0x - a5);
    const float e1 = (float)(a1 * P1x - a3 * P1y - a4), e2 = (float)(a2 * P1y - a3 * P1x - a5);
    // OctaveKeyLines: the float direction against double multiples of M_PI
    const float ddx = e1 - s1, ddy = e2 - s2;
    const double d = direction;
    bool swap = false;
    if (d >= -0.75 * kPi && d < -0.25 * kPi && ddy > 0) { swap = true; bits |= B_SWAP_Q0; }
    if (d >= -0.25 * kPi && d < 0.25 * kPi && ddx < 0) { swap = true; bits |= B_SWAP_Q1; }
    if (d >= 0.25 * kPi && d < 0.75 * kPi && ddy < 0) { swap = true; bits |= B_SWAP_Q2; }
    if (((d >= 0.75 * kPi && d < kPi) || (d >= -kPi && d < -0.75 * kPi)) && ddx > 0) { swap = true; bits |= B_SWAP_Q3; }
    if (d >= kPi || d < -kPi) bits |= B_FLOAT_PI;
    float* o = out + 4 * nl++;
    const float one = 1.0f;   // scale[0] of OctaveKeyLines, then keylines_to_mat's scale
    o[0] = (one * (swap ? e1 : s1)) * scale;
    o[1] = (one * (swap ? e2 : s2)) * scale;
    o[2] = (one * (swap ? s1 : e1)) * scale;
    o[3] = (one * (swap ? s2 : e2)) * scale;
  }
  return nl;
}
}  // namespace lines
}  // namespace pus
