// Tiled inference under a workspace budget (option "workspace_mb", DESIGN.md section 3): a large image runs as a
// sequence of batches of overlapping windows.  Every window is Th x Tw LR pixels, clamped inside its image, and carries
// at least `halo` pixels of context around its core wherever the core edge is not the image edge, so its core is
// computed from exactly the inputs the whole-image forward reads.
//   * tile_gather_kernel : copies a batch of LR windows out of x [n,H,W] and the matching HR windows out of x2 into
//                          contiguous batch buffers;
//   * tile_stitch_kernel : writes the HR core of every window of the batch output into y.
// Window origins come from the by-value geometry below, so a tiled forward needs no table upload and no host
// synchronisation.
#pragma once
#include <cstdint>

namespace dcscn {

struct TileGeom {
  int n_img, H, W;      // LR image
  int scale;
  int th, tw;           // window (LR pixels)
  int halo;             // LR pixels of context a core edge needs inside its window
  int my, mx;           // windows per image along y / x
  long long first;      // index of the batch's first window (image-major, then row, then column)
  int count;            // windows in this batch
};

// Core [c0, c1) and window origin o of window i (of m) along an axis of D pixels with windows of T pixels.  The first
// window starts at the image edge and its core ends `halo` pixels before the window does; every later core advances by
// T - 2 halo with `halo` pixels on both sides; the last window ends at the image edge and its core runs to it.  Origins
// are clamped into [0, D - T], which only moves the last window.
__host__ __device__ __forceinline__ void tile_axis(int i, int m, int T, int r, int D, int* c0, int* c1, int* o) {
  const int S = T - 2 * r;
  *c0 = i == 0 ? 0 : (T - r) + (i - 1) * S;
  *c1 = i == m - 1 ? D : (T - r) + i * S;
  int org = *c0 - r;
  if (org > D - T) org = D - T;
  if (org < 0) org = 0;
  *o = org;
}

// Windows along an axis of D pixels: one when the window spans it, else the first, as many full interior cores as it
// takes for the last core to start at least `halo` pixels inside the last window (D - T + halo), and the last.
__host__ __device__ __forceinline__ int tile_count(int D, int T, int r) {
  if (T >= D) return 1;
  const int S = T - 2 * r, rest = D - 2 * T + 2 * r;
  return 2 + (rest > 0 ? (rest + S - 1) / S : 0);
}

__device__ __forceinline__ void tile_window(const TileGeom& g, long long v, int* img, int* oy, int* ox, int* cy0,
                                            int* cy1, int* cx0, int* cx1) {
  const long long w = g.first + v;
  const long long per = (long long)g.my * g.mx;
  *img = (int)(w / per);
  const int rem = (int)(w - (long long)*img * per);
  const int wy = rem / g.mx, wx = rem - wy * g.mx;
  tile_axis(wy, g.my, g.th, g.halo, g.H, cy0, cy1, oy);
  tile_axis(wx, g.mx, g.tw, g.halo, g.W, cx0, cx1, ox);
}

// xb [count, th, tw] <- the batch's LR windows of x; x2b [count, s*th, s*tw] <- the matching HR windows of x2.
__global__ void __launch_bounds__(256) tile_gather_kernel(const TileGeom g, const float* __restrict__ x,
                                                          const float* __restrict__ x2, float* __restrict__ xb,
                                                          float* __restrict__ x2b) {
  const int s = g.scale;
  const long long lr_per = (long long)g.th * g.tw, hr_per = lr_per * s * s;
  const long long lr_total = lr_per * g.count, total = lr_total + hr_per * g.count;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const bool lr = e < lr_total;
    const long long f = lr ? e : e - lr_total;
    const long long per = lr ? lr_per : hr_per;
    const int ww = lr ? g.tw : s * g.tw;
    const long long v = f / per;
    const int r = (int)(f - v * per);
    const int yy = r / ww, xx = r - yy * ww;
    int img, oy, ox, cy0, cy1, cx0, cx1;
    tile_window(g, v, &img, &oy, &ox, &cy0, &cy1, &cx0, &cx1);
    if (lr) {
      xb[e] = __ldg(x + ((long long)img * g.H + oy + yy) * g.W + ox + xx);
    } else {
      const long long HW = (long long)s * g.W;
      x2b[f] = __ldg(x2 + ((long long)img * s * g.H + (long long)s * oy + yy) * HW + (long long)s * ox + xx);
    }
  }
}

// y <- the HR core of every window of yb [count, s*th, s*tw].
__global__ void __launch_bounds__(256) tile_stitch_kernel(const TileGeom g, const float* __restrict__ yb, float* __restrict__ y) {
  const int s = g.scale, hw = s * g.tw;
  const long long per = (long long)s * g.th * hw, total = per * g.count;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long v = e / per;
    const int r = (int)(e - v * per);
    const int yy = r / hw, xx = r - yy * hw;
    int img, oy, ox, cy0, cy1, cx0, cx1;
    tile_window(g, v, &img, &oy, &ox, &cy0, &cy1, &cx0, &cx1);
    const int Y = s * oy + yy, X = s * ox + xx;          // HR position in the image
    if (Y < s * cy0 || Y >= s * cy1 || X < s * cx0 || X >= s * cx1) continue;
    y[((long long)img * s * g.H + Y) * ((long long)s * g.W) + X] = __ldg(yb + e);
  }
}

}  // namespace dcscn
