// pus_lines.cu -- popup_plane::get_ground_edges' line detection (popup_plane.cpp:753-770 and line_lbd's EDLines,
// binary_descriptor.cpp:483-585, 792-1144, 1579-2870) batched over frames on the device, behind pus_popup_lines.
// Per-pixel kernels make the grey image, the per-frame histogram and LUT, the optional 0.5x image, the 5 x 5 blur,
// the Sobel maps and one packed record per pixel; one block per frame compacts the anchors in the reference's
// column-major scan order; one thread per frame replays the order-dependent walk (pus_lines.cuh); one thread per chain
// extracts its lines; a per-frame prefix sum over the chains and a scatter pack them in frame and chain order.
// Compiled with --fmad=false so the double arithmetic of the fits rounds like the reference's scalar code.
#include <cuda_runtime.h>

#include <climits>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/popup_gpu.h"
#include "pus_lines.cuh"
#include "pus_stages.cuh"

namespace pus {
namespace lines {

__device__ __forceinline__ int refl(int p, int n) { return p < 0 ? -p : (p >= n ? 2 * n - 2 - p : p); }

// cvtColor BGR2GRAY on 8U (OpenCV's fixed point, 15 fractional bits) or a copy; the frame's histogram in shared memory
__global__ void grey_hist_kernel(Dims D, const unsigned char* __restrict__ img, unsigned char* __restrict__ grey,
                                 int* __restrict__ hist) {
  __shared__ int sh[256];
  const int f = blockIdx.y;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < D.N) {
    const long long q = (long long)f * D.N + p;
    int v;
    if (D.C == 3) {
      const unsigned char* s = img + 3 * q;
      v = (s[0] * 3735 + s[1] * 19235 + s[2] * 9798 + (1 << 14)) >> 15;
    } else {
      v = img[q];
    }
    grey[q] = (unsigned char)v;
    atomicAdd(&sh[v], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[256 * f + i], sh[i]);
}

// cv::mean < 90 (the integer sum times 1.0 / N in double) decides equalizeHist; its LUT, or the identity
__global__ void lut_kernel(int n_frames, Dims D, const int* __restrict__ hist, unsigned char* __restrict__ lut,
                           unsigned* __restrict__ bits) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  const int* hf = hist + 256 * f;
  unsigned char* L = lut + 256 * f;
  long long sum = 0;
  for (int v = 0; v < 256; v++) sum += (long long)v * hf[v];
  unsigned b = D.ds ? B_HALVED : 0;
  for (int v = 0; v < 256; v++) L[v] = (unsigned char)v;
  if ((double)sum * (1.0 / (double)D.N) < 90) {
    b |= B_EQUALIZED;
    int i = 0;
    while (!hf[i]) ++i;
    const int total = (int)D.N;
    if (hf[i] == total) {
      b |= B_ONE_BIN;
    } else {
      const float scale = (256 - 1.f) / (total - hf[i]);
      int s = 0;
      for (L[i++] = 0; i < 256; ++i) {
        s += hf[i];
        L[i] = (unsigned char)__float2int_rn((float)s * scale);   // <= 255: s <= total - hf[first]
      }
    }
  }
  bits[f] = b;
}

// the LUT, then with downsample OpenCV's 0.5x INTER_LINEAR on 8U (its area fast path: (a + b + c + d + 2) >> 2)
__global__ void prep_kernel(int n_frames, Dims D, const unsigned char* __restrict__ grey,
                            const unsigned char* __restrict__ lut, unsigned char* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.n * n_frames) return;
  const int f = (int)(i / D.n), p = (int)(i % D.n);
  const unsigned char* L = lut + 256 * f;
  const unsigned char* g = grey + (long long)f * D.N;
  if (D.ds) {
    const int x = p % D.w, y = p / D.w;
    const unsigned char* r0 = g + (long long)(2 * y) * D.W + 2 * x;
    out[i] = (unsigned char)((L[r0[0]] + L[r0[1]] + L[r0[D.W]] + L[r0[D.W + 1]] + 2) >> 2);
  } else {
    out[i] = L[g[p]];
  }
}

// GaussianBlur 5 x 5, sigma 1 on 8U: OpenCV 4.13's bit-exact separable filter (kernel 14 62 104 62 14 / 256, the row
// pass kept with 8 fractional bits, the column pass rounded from 16), BORDER_REFLECT_101
__constant__ int c_gk[5] = {14, 62, 104, 62, 14};
__global__ void blur_row_kernel(int n_frames, Dims D, const unsigned char* __restrict__ in, unsigned short* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.n * n_frames) return;
  const int p = (int)(i % D.n), x = p % D.w;
  const unsigned char* row = in + (i - x);
  int s = 0;
  for (int j = 0; j < 5; j++) s += c_gk[j] * row[refl(x + j - 2, D.w)];
  out[i] = (unsigned short)s;
}
__global__ void blur_col_kernel(int n_frames, Dims D, const unsigned short* __restrict__ in, unsigned char* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.n * n_frames) return;
  const long long f0 = i - i % D.n;
  const int p = (int)(i % D.n), x = p % D.w, y = p / D.w;
  unsigned s = 0;
  for (int j = 0; j < 5; j++) s += (unsigned)c_gk[j] * in[f0 + (long long)refl(y + j - 2, D.h) * D.w + x];
  out[i] = (unsigned char)((s + (1u << 15)) >> 16);
}

// Sobel 3 x 3 to 16S (BORDER_REFLECT_101), |dx| + |dy|, THRESH_TOZERO at 81, / 4 (saturate_cast<short> of v * 0.25f:
// round half to even), the direction |dx| < |dy|, and the packed record
__global__ void grad_kernel(int n_frames, Dims D, const unsigned char* __restrict__ b, short* __restrict__ dx,
                            short* __restrict__ dy, short* __restrict__ g, unsigned short* __restrict__ rec) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.n * n_frames) return;
  const long long f0 = i - i % D.n;
  const int p = (int)(i % D.n), x = p % D.w, y = p / D.w;
  const int xm = refl(x - 1, D.w), xp = refl(x + 1, D.w);
  const unsigned char* rm = b + f0 + (long long)refl(y - 1, D.h) * D.w;
  const unsigned char* r0 = b + f0 + (long long)y * D.w;
  const unsigned char* rp = b + f0 + (long long)refl(y + 1, D.h) * D.w;
  const int gx = (rm[xp] + 2 * r0[xp] + rp[xp]) - (rm[xm] + 2 * r0[xm] + rp[xm]);
  const int gy = (rp[xm] + 2 * rp[x] + rp[xp]) - (rm[xm] + 2 * rm[x] + rm[xp]);
  const int ax = gx < 0 ? -gx : gx, ay = gy < 0 ? -gy : gy;
  const int t = ax + ay > kGradThr + 1 ? ax + ay : 0;
  const int q = t >> 2, r = t & 3;
  const int gv = r < 2 ? q : (r > 2 ? q + 1 : q + (q & 1));
  dx[i] = (short)gx;
  dy[i] = (short)gy;
  g[i] = (short)gv;
  rec[i] = pack(gv, ax < ay);
}

// The anchors of one frame (binary_descriptor.cpp:1640-1666: w outer, h inner, both from 1 in steps of 2) compacted in
// that order by a block-wide prefix sum; one block per frame.  n_anchor receives the full count, anchors the first plim.
__global__ void __launch_bounds__(1024) anchor_kernel(Dims D, const short* __restrict__ g, const unsigned short* __restrict__ rec,
                                                      int* __restrict__ anchors, int* __restrict__ n_anchor) {
  __shared__ int warp_sum[32];
  __shared__ int carry_s;
  const int f = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const short* gf = g + (long long)f * D.n;
  const unsigned short* rf = rec + (long long)f * D.n;
  int* af = anchors + (long long)f * D.plim;
  const int nh = (D.h - 1) / 2, nw = (D.w - 1) / 2, npos = nw * nh;
  if (t == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < npos; base += 1024) {
    const int k = base + t;
    int flag = 0, idx = 0;
    if (k < npos) {
      const int x = 1 + 2 * (k / nh), y = 1 + 2 * (k % nh);
      idx = y * D.w + x;
      const int v = gf[idx];
      if (rf[idx] & kHoriz) flag = v >= gf[idx - D.w] + kAnchorThr && v >= gf[idx + D.w] + kAnchorThr;
      else flag = v >= gf[idx - 1] + kAnchorThr && v >= gf[idx + 1] + kAnchorThr;
    }
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_sum[wid] = __popc(m);
    __syncthreads();
    if (wid == 0) {
      int v = warp_sum[lane], s = v;
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += u;
      }
      warp_sum[lane] = s - v;   // exclusive
    }
    __syncthreads();
    const int carry = carry_s;
    if (flag) {
      const int pos = carry + warp_sum[wid] + __popc(m & ((1u << lane) - 1));
      if (pos < D.plim) af[pos] = idx;
    }
    __syncthreads();
    if (t == 1023) carry_s = carry + warp_sum[31] + __popc(m);
    __syncthreads();
  }
  if (t == 0) n_anchor[f] = carry_s;
}

// The walk of each frame, one thread in a block of its own (the frames' walks diverge; a warp would serialise them)
__global__ void walk_kernel(int n_frames, Dims D, unsigned short* rec, const int* __restrict__ anchors,
                            const int* __restrict__ n_anchor, int* p1, int* p2, int* s1, int* s2, int* chain_px, int* sid,
                            int* __restrict__ status, int* __restrict__ n_chains) {
  const int f = blockIdx.x;
  if (f >= n_frames || threadIdx.x) return;
  unsigned bits = 0;
  n_chains[f] = 0;
  if (n_anchor[f] > D.plim) { status[f] = 1; return; }
  const long long hc = D.hcap, sc = D.clim + 2;
  Walk W{rec + (long long)f * D.n, D.w, D.h, p1 + f * hc, p2 + f * hc, s1 + f * sc, s2 + f * sc};
  int nc = 0;
  status[f] = draw_edges(W, anchors + (long long)f * D.plim, n_anchor[f], chain_px + 2 * hc * f, sid + sc * f, nc, bits);
  n_chains[f] = status[f] ? 0 : nc;
}

// one thread per (frame, chain): the chain's lines into its slots
__global__ void chain_kernel(int n_frames, Dims D, const unsigned short* __restrict__ rec, const short* __restrict__ dx,
                             const short* __restrict__ dy, const int* __restrict__ chain_px, const int* __restrict__ sid,
                             const int* __restrict__ n_chains, float* __restrict__ slots, int* __restrict__ chain_count) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per = D.clim + 1;
  if (i >= per * n_frames) return;
  const int f = (int)(i / per), c = (int)(i % per);
  if (c >= n_chains[f]) return;
  const long long sc = D.clim + 2, off = (long long)f * D.n;
  const int* sf = sid + sc * f;
  const int s = sf[c], e = sf[c + 1];
  unsigned bits = 0;
  chain_count[i] = chain_lines(chain_px + 2 * D.hcap * f + s, e - s, rec + off, dx + off, dy + off, D.w, D.h,
                               D.ds ? 2.0f : 1.0f, slots + 4 * ((long long)D.nslot * f + line_slot(s, c)), bits);
}

// per frame: the chains' first rows (prefix sum in chain order) and the frame's count
__global__ void count_kernel(int n_frames, Dims D, const int* __restrict__ n_chains, int* __restrict__ chain_count,
                             int* __restrict__ frame_count) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n_frames) return;
  int* cc = chain_count + (long long)(D.clim + 1) * f;
  int s = 0;
  for (int c = 0; c < n_chains[f]; c++) {
    const int v = cc[c];
    cc[c] = s;
    s += v;
  }
  cc[n_chains[f]] = s;
  frame_count[f] = s;
}

// one thread per (frame, chain): its rows to the packed output
__global__ void scatter_kernel(int n_frames, Dims D, const int* __restrict__ sid, const int* __restrict__ n_chains,
                               const int* __restrict__ chain_first, const long long* __restrict__ frame_first,
                               const float* __restrict__ slots, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per = D.clim + 1;
  if (i >= per * n_frames) return;
  const int f = (int)(i / per), c = (int)(i % per);
  if (c >= n_chains[f]) return;
  const int r0 = chain_first[i], r1 = chain_first[i + 1];
  const float4* src = (const float4*)(slots + 4 * ((long long)D.nslot * f + line_slot(sid[(D.clim + 2) * f + c], c)));
  float4* dst = (float4*)(out + 4 * (frame_first[f] + r0));
  for (int r = 0; r < r1 - r0; r++) dst[r] = src[r];
}

Dims make_dims(int width, int height, int channels, int downsample) {
  Dims D;
  D.W = width; D.H = height; D.C = channels; D.ds = downsample ? 1 : 0;
  D.w = downsample ? width / 2 : width; D.h = downsample ? height / 2 : height;
  D.N = (long long)width * height; D.n = (long long)D.w * D.h;
  D.plim = (int)pix_limit(D.n); D.clim = (int)chain_limit(D.n); D.hcap = (int)half_cap(D.n); D.nslot = (int)line_slots(D.n);
  return D;
}

const char* shape_error(int width, int height, int channels, int downsample) {
  if (channels != 1 && channels != 3) return "channels must be 1 (grey) or 3 (BGR)";
  if (downsample && ((width & 1) || (height & 1))) return "downsample needs even width and height";
  const int w = downsample ? width / 2 : width, h = downsample ? height / 2 : height;
  if (w < 3 || h < 3) return "the detection image (after the optional halving) must be at least 3 x 3";
  if ((long long)width * height > PUS_POPUP_LINES_MAX_PIXELS) return "a frame has more than 2^28 pixels";
  return nullptr;
}

#define WCHK(call)                        \
  do {                                    \
    const cudaError_t e__ = (call);       \
    if (e__ != cudaSuccess) return e__;   \
  } while (0)

cudaError_t detect(cudaStream_t st, Alloc& A, int n_frames, const Dims& D, const unsigned char* d_img, Work& W) {
  const long long F = n_frames, nn = F * D.n, per = D.clim + 1;
  WCHK(A.get(W.grey, F * D.N));
  WCHK(A.get(W.hist, 256 * F));
  WCHK(A.get(W.lut, 256 * F));
  WCHK(A.get(W.bits, F));
  WCHK(A.get(W.i8, nn));
  WCHK(A.get(W.h16, nn));
  WCHK(A.get(W.b8, nn));
  WCHK(A.get(W.dx, nn));
  WCHK(A.get(W.dy, nn));
  WCHK(A.get(W.g, nn));
  WCHK(A.get(W.rec, nn));
  WCHK(A.get(W.anc, F * D.plim));
  WCHK(A.get(W.nanc, F));
  WCHK(A.get(W.p1, F * D.hcap));
  WCHK(A.get(W.p2, F * D.hcap));
  WCHK(A.get(W.s1, F * (D.clim + 2)));
  WCHK(A.get(W.s2, F * (D.clim + 2)));
  WCHK(A.get(W.cpx, 2 * F * D.hcap));
  WCHK(A.get(W.sid, F * (D.clim + 2)));
  WCHK(A.get(W.st, F));
  WCHK(A.get(W.nc, F));
  WCHK(A.get(W.cc, F * per));
  WCHK(A.get(W.fc, F));
  WCHK(A.get(W.slots, 4 * F * D.nslot));
  if (n_frames == 0) return cudaSuccess;
  WCHK(cudaMemsetAsync(W.hist, 0, 256 * F * sizeof(int), st));
  grey_hist_kernel<<<dim3((unsigned)((D.N + 255) / 256), (unsigned)F), 256, 0, st>>>(D, d_img, W.grey, W.hist);
  lut_kernel<<<(unsigned)((F + 63) / 64), 64, 0, st>>>(n_frames, D, W.hist, W.lut, W.bits);
  const unsigned gb = (unsigned)((nn + 255) / 256);
  prep_kernel<<<gb, 256, 0, st>>>(n_frames, D, W.grey, W.lut, W.i8);
  blur_row_kernel<<<gb, 256, 0, st>>>(n_frames, D, W.i8, W.h16);
  blur_col_kernel<<<gb, 256, 0, st>>>(n_frames, D, W.h16, W.b8);
  grad_kernel<<<gb, 256, 0, st>>>(n_frames, D, W.b8, W.dx, W.dy, W.g, W.rec);
  anchor_kernel<<<(unsigned)F, 1024, 0, st>>>(D, W.g, W.rec, W.anc, W.nanc);
  walk_kernel<<<(unsigned)F, 1, 0, st>>>(n_frames, D, W.rec, W.anc, W.nanc, W.p1, W.p2, W.s1, W.s2, W.cpx, W.sid, W.st, W.nc);
  const unsigned gc = (unsigned)((F * per + 127) / 128);
  chain_kernel<<<gc, 128, 0, st>>>(n_frames, D, W.rec, W.dx, W.dy, W.cpx, W.sid, W.nc, W.slots, W.cc);
  count_kernel<<<(unsigned)((F + 63) / 64), 64, 0, st>>>(n_frames, D, W.nc, W.cc, W.fc);
  return cudaGetLastError();
}

cudaError_t scatter(cudaStream_t st, int n_frames, const Dims& D, const Work& W, const long long* d_first, float* d_out) {
  if (n_frames == 0) return cudaSuccess;
  const unsigned gc = (unsigned)(((long long)n_frames * (D.clim + 1) + 127) / 128);
  scatter_kernel<<<gc, 128, 0, st>>>(n_frames, D, W.sid, W.nc, W.cc, d_first, W.slots, d_out);
  return cudaGetLastError();
}
#undef WCHK
}  // namespace lines
}  // namespace pus

extern "C" long long pus_popup_lines(int device, int n_frames, const unsigned char* images, int width, int height,
                                     int channels, int downsample, int* status, int* counts, float* lines,
                                     long long capacity) {
  using namespace pus;
  using namespace pus::lines;
  const Call C{"pus_popup_lines"};
  if (n_frames < 0) return C.refuse("n_frames < 0");
  if (!images && n_frames > 0) return C.refuse("images is NULL");
  if (!status || !counts) return C.refuse("status and counts are required");
  if (const char* why = shape_error(width, height, channels, downsample)) return C.refuse(why);
  if (C.check_device(device) < 0) return -1;
  if (n_frames == 0) return 0;
  PUS_CALL_OK(C, cudaSetDevice(device));
  const Dims D = make_dims(width, height, channels, downsample);
  const long long F = n_frames;
  TempAlloc A;
  Work W;
  unsigned char* d_img = nullptr;
  PUS_CALL_OK(C, A.upload(d_img, images, (size_t)(F * D.N * channels)));
  PUS_CALL_OK(C, detect(0, A, n_frames, D, d_img, W));
  std::vector<int> st(F), fc(F);
  PUS_CALL_OK(C, download(st.data(), W.st, F));
  PUS_CALL_OK(C, download(fc.data(), W.fc, F));
  std::vector<long long> ff(F);
  long long total = 0;
  for (int f = 0; f < n_frames; f++) {
    status[f] = st[f];
    counts[f] = st[f] ? 0 : fc[f];
    ff[f] = total;
    total += counts[f];
  }
  if (!lines) return total;   // size query
  if (capacity < total) return C.refuse("capacity is smaller than the number of lines");
  if (total == 0) return 0;
  long long* d_ff = nullptr;
  float* d_out = nullptr;
  PUS_CALL_OK(C, A.upload(d_ff, ff.data(), F));
  PUS_CALL_OK(C, A.get(d_out, 4 * total));
  PUS_CALL_OK(C, scatter(0, n_frames, D, W, d_ff, d_out));
  PUS_CALL_OK(C, download(lines, d_out, 4 * total));
  return total;
}
