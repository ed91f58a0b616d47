// CPU oracle of pus_popup_lines: the per-pixel stages and the packing restated on the host around the frame code of
// pus_lines.cuh (the walk and the per-chain line extraction), which the device runs after its per-pixel kernels.  The
// independent restatement of every stage is tools/make_popup_line_golden.py (its fixture is compared with this oracle
// bit for bit; its per-pixel stages are live cv2).  Exports orc_popup_lines (the C-ABI), orc_popup_lines_bits (per-frame
// branch bits) and the stage entry points orc_lines_grey, orc_lines_contrast, orc_lines_halve, orc_lines_blur,
// orc_lines_gradient and orc_lines_chains.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../pop_up_slam_b200/csrc/pus_lines.cuh"

using namespace pus::lines;

static thread_local std::string g_orc_err;

namespace {
typedef unsigned char u8;
int refl(int p, int n) { return p < 0 ? -p : (p >= n ? 2 * n - 2 - p : p); }

void grey(const u8* img, int W, int H, int C, u8* out) {
  for (long long p = 0; p < (long long)W * H; p++)
    out[p] = C == 3 ? (u8)((img[3 * p] * 3735 + img[3 * p + 1] * 19235 + img[3 * p + 2] * 9798 + (1 << 14)) >> 15) : img[p];
}

// cv::mean < 90 then cv::equalizeHist (OpenCV 4.13); returns the branch bits
unsigned contrast(const u8* g, int W, int H, u8* out) {
  const long long N = (long long)W * H;
  int hist[256] = {0};
  long long sum = 0;
  for (long long p = 0; p < N; p++) hist[g[p]]++;
  for (int v = 0; v < 256; v++) sum += (long long)v * hist[v];
  u8 lut[256];
  for (int v = 0; v < 256; v++) lut[v] = (u8)v;
  unsigned bits = 0;
  if ((double)sum * (1.0 / (double)N) < 90) {
    bits |= B_EQUALIZED;
    int i = 0;
    while (!hist[i]) ++i;
    if (hist[i] == (int)N) {
      bits |= B_ONE_BIN;
    } else {
      const float scale = (256 - 1.f) / ((int)N - hist[i]);
      int s = 0;
      for (lut[i++] = 0; i < 256; ++i) {
        s += hist[i];
        lut[i] = (u8)std::nearbyint((float)s * scale);
      }
    }
  }
  for (long long p = 0; p < N; p++) out[p] = lut[g[p]];
  return bits;
}

void halve(const u8* in, int W, int H, u8* out) {
  const int w = W / 2, h = H / 2;
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const u8* r = in + (long long)(2 * y) * W + 2 * x;
      out[(long long)y * w + x] = (u8)((r[0] + r[1] + r[W] + r[W + 1] + 2) >> 2);
    }
}

void blur(const u8* in, int w, int h, u8* out) {
  static const int k[5] = {14, 62, 104, 62, 14};
  std::vector<unsigned> row((size_t)w * h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      unsigned s = 0;
      for (int j = 0; j < 5; j++) s += k[j] * in[(long long)y * w + refl(x + j - 2, w)];
      row[(size_t)y * w + x] = s;
    }
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      unsigned s = 0;
      for (int j = 0; j < 5; j++) s += k[j] * row[(size_t)refl(y + j - 2, h) * w + x];
      out[(long long)y * w + x] = (u8)((s + (1u << 15)) >> 16);
    }
}

void gradient(const u8* b, int w, int h, short* dx, short* dy, short* g, unsigned short* rec) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      auto at = [&](int yy, int xx) { return (int)b[(long long)refl(yy, h) * w + refl(xx, w)]; };
      const int gx = at(y - 1, x + 1) + 2 * at(y, x + 1) + at(y + 1, x + 1) - at(y - 1, x - 1) - 2 * at(y, x - 1) - at(y + 1, x - 1);
      const int gy = at(y + 1, x - 1) + 2 * at(y + 1, x) + at(y + 1, x + 1) - at(y - 1, x - 1) - 2 * at(y - 1, x) - at(y - 1, x + 1);
      const int s = std::abs(gx) + std::abs(gy);
      const int t = s > kGradThr + 1 ? s : 0;
      const int gv = (int)std::nearbyint((float)t * 0.25f);
      const long long i = (long long)y * w + x;
      dx[i] = (short)gx;
      dy[i] = (short)gy;
      g[i] = (short)gv;
      rec[i] = pack(gv, std::abs(gx) < std::abs(gy));
    }
}

struct Frame {   // one frame's detection state on the host
  int w, h;
  std::vector<short> dx, dy, g;
  std::vector<unsigned short> rec;
  std::vector<int> cpx, sid;
  int n_chains = 0;
};

// the anchors and the walk; returns the status
int chains(const u8* b, int w, int h, Frame& F, unsigned& bits) {
  const long long n = (long long)w * h;
  F.w = w; F.h = h;
  F.dx.resize(n); F.dy.resize(n); F.g.resize(n); F.rec.resize(n);
  gradient(b, w, h, F.dx.data(), F.dy.data(), F.g.data(), F.rec.data());
  std::vector<int> anchors;
  for (int x = 1; x < w - 1; x += 2)
    for (int y = 1; y < h - 1; y += 2) {
      const int i = y * w + x, v = F.g[i];
      const bool a = (F.rec[i] & kHoriz) ? (v >= F.g[i - w] + kAnchorThr && v >= F.g[i + w] + kAnchorThr)
                                         : (v >= F.g[i - 1] + kAnchorThr && v >= F.g[i + 1] + kAnchorThr);
      if (a) anchors.push_back(i);
    }
  F.n_chains = 0;
  if ((long long)anchors.size() > pix_limit(n)) { bits |= B_OVER_ANCHORS; return 1; }
  const long long hc = half_cap(n), sc = chain_limit(n) + 2;
  std::vector<int> p1(hc), p2(hc), s1(sc), s2(sc);
  F.cpx.assign(2 * hc, 0);
  F.sid.assign(sc, 0);
  Walk W{F.rec.data(), w, h, p1.data(), p2.data(), s1.data(), s2.data()};
  const int st = draw_edges(W, anchors.data(), (int)anchors.size(), F.cpx.data(), F.sid.data(), F.n_chains, bits);
  if (st) F.n_chains = 0;
  return st;
}

// one frame end to end: status, its lines appended to out
int frame(const u8* img, int W, int H, int C, int ds, std::vector<float>& out, unsigned& bits) {
  const long long N = (long long)W * H;
  std::vector<u8> g(N), c(N);
  grey(img, W, H, C, g.data());
  bits |= contrast(g.data(), W, H, c.data());
  int w = W, h = H;
  std::vector<u8> s;
  if (ds) {
    bits |= B_HALVED;
    w = W / 2; h = H / 2;
    s.resize((size_t)w * h);
    halve(c.data(), W, H, s.data());
  } else {
    s.swap(c);
  }
  std::vector<u8> b((size_t)w * h);
  blur(s.data(), w, h, b.data());
  Frame F;
  const int st = chains(b.data(), w, h, F, bits);
  if (st) return st;
  const size_t before = out.size();
  for (int k = 0; k < F.n_chains; k++) {
    const int a = F.sid[k], e = F.sid[k + 1];
    std::vector<float> rows(4 * (size_t)((e - a) / kMinLen + 1));
    const int nl = chain_lines(F.cpx.data() + a, e - a, F.rec.data(), F.dx.data(), F.dy.data(), w, h, ds ? 2.0f : 1.0f,
                               rows.data(), bits);
    out.insert(out.end(), rows.begin(), rows.begin() + 4 * nl);
  }
  if ((out.size() - before) / 4 > PUS_POPUP_MAX_LINES) bits |= B_MANY;
  return 0;
}
}  // namespace

extern "C" {
const char* orc_popup_last_error(void) { return g_orc_err.c_str(); }

// the C-ABI of pus_popup_lines on the host (same refusals)
long long orc_popup_lines(int device, int n_frames, const u8* images, int width, int height, int channels, int downsample,
                          int* status, int* counts, float* lines, long long capacity) {
  (void)device;
  auto refuse = [](const char* why) { g_orc_err = std::string("orc_popup_lines: ") + why; return -1LL; };
  if (n_frames < 0) return refuse("n_frames < 0");
  if (!images && n_frames > 0) return refuse("images is NULL");
  if (!status || !counts) return refuse("status and counts are required");
  if (channels != 1 && channels != 3) return refuse("channels must be 1 (grey) or 3 (BGR)");
  if (downsample && ((width & 1) || (height & 1))) return refuse("downsample needs even width and height");
  const int w = downsample ? width / 2 : width, h = downsample ? height / 2 : height;
  if (w < 3 || h < 3) return refuse("the detection image (after the optional halving) must be at least 3 x 3");
  if ((long long)width * height > PUS_POPUP_LINES_MAX_PIXELS) return refuse("a frame has more than 2^28 pixels");
  std::vector<float> all;
  const long long per = (long long)width * height * channels;
  for (int f = 0; f < n_frames; f++) {
    unsigned bits = 0;
    const size_t before = all.size();
    status[f] = frame(images + per * f, width, height, channels, downsample, all, bits);
    counts[f] = (int)((all.size() - before) / 4);
  }
  const long long total = (long long)all.size() / 4;
  if (!lines) return total;
  if (capacity < total) return refuse("capacity is smaller than the number of lines");
  if (total) std::memcpy(lines, all.data(), all.size() * sizeof(float));
  return total;
}

void orc_popup_lines_bits(int n_frames, const u8* images, int width, int height, int channels, int downsample,
                          unsigned* bits) {
  const long long per = (long long)width * height * channels;
  for (int f = 0; f < n_frames; f++) {
    std::vector<float> out;
    bits[f] = 0;
    frame(images + per * f, width, height, channels, downsample, out, bits[f]);
  }
}

void orc_lines_grey(const u8* img, int W, int H, int C, u8* out) { grey(img, W, H, C, out); }
int orc_lines_contrast(const u8* g, int W, int H, u8* out) { return (int)contrast(g, W, H, out); }
void orc_lines_halve(const u8* in, int W, int H, u8* out) { halve(in, W, H, out); }
void orc_lines_blur(const u8* in, int w, int h, u8* out) { blur(in, w, h, out); }
void orc_lines_gradient(const u8* b, int w, int h, short* dx, short* dy, short* g, u8* dir) {
  std::vector<unsigned short> rec((size_t)w * h);
  gradient(b, w, h, dx, dy, g, rec.data());
  for (size_t i = 0; i < rec.size(); i++) dir[i] = (rec[i] & kHoriz) ? 255 : 0;
}
// the chains of a blurred image: pixel indices into px (capacity cap), starts into sid (n_chains + 1); returns the
// number of chains, -1 for status 1, -2 when a capacity is short
int orc_lines_chains(const u8* b, int w, int h, int* px, long long cap, int* sid, long long sid_cap) {
  Frame F;
  unsigned bits = 0;
  if (chains(b, w, h, F, bits)) return -1;
  if (F.n_chains + 1 > sid_cap || F.sid[F.n_chains] > cap) return -2;
  std::memcpy(sid, F.sid.data(), (F.n_chains + 1) * sizeof(int));
  std::memcpy(px, F.cpx.data(), F.sid[F.n_chains] * sizeof(int));
  return F.n_chains;
}
}
