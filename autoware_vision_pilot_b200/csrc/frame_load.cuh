// frame_load.cuh — one source pixel of a camera frame in any VPB_PIX_* layout, converted to 3 bytes: the per-format
// loads the pre-process (preprocess.cu) and the rectification (rectify.cu) share.
#pragma once
#include "common.cuh"

namespace vpb {

struct PreImg {          // one image of the call (blockIdx.z); images of one call may differ in every field
  const uint8_t* src;   // [h][stride] bytes, 3 interleaved channels
  const int* xb; const int* xk;   // horizontal bounds / coeffs (xks per output column)
  const int* yb; const int* yk;   // vertical
  int h, w, stride, xks, yks;
  int OH, OW, out_x0, out_y0;     // resized size and its paste offset in the output canvas
};
// The format fields of a non-packed image (the pre-process keeps them apart from PreImg: see PreParamsCvt)
struct PreCvt {
  const uint8_t* uv;    // NV12: the interleaved U,V plane [h/2][uv_stride]
  int fmt, uv_stride;   // VPB_PIX_*
  int bgr;              // 1: a non-packed image converts to B, G, R (the BGR conventions), 0: to R, G, B
};

// OpenCV's YUV -> RGB of COLOR_YUV2RGB_NV12 / _UYVY / _YUYV (BT.601 limited range, 20-bit fixed point): y' = max(Y -
// 16, 0) * 1220542 + 2^19, R = (y' + 1673527 v) >> 20, G = (y' - 852492 v - 409993 u) >> 20, B = (y' + 2116026 u) >> 20,
// u = U - 128, v = V - 128, each clipped to [0, 255].  No term overflows 32 bits.
__device__ __forceinline__ void yuv_px(int Y, int U, int V, int bgr, int (&o)[3]) {
  const int y = max(Y - 16, 0) * 1220542 + (1 << 19);
  const int u = U - 128, v = V - 128;
  const int r = min(max((y + 1673527 * v) >> 20, 0), 255);
  const int g = min(max((y - 852492 * v - 409993 * u) >> 20, 0), 255);
  const int b = min(max((y + 2116026 * u) >> 20, 0), 255);
  o[0] = bgr ? b : r; o[1] = g; o[2] = bgr ? r : b;
}

// Source pixel (x, y) of a YUV image, converted: chroma of the 2x2 block (NV12) or the horizontal pair (UYVY, YUYV)
__device__ __forceinline__ void yuv_load(const PreImg& im, const PreCvt& yv, int y, int x, int (&o)[3]) {
  const uint8_t* row = im.src + static_cast<size_t>(y) * im.stride;
  if (yv.fmt == VPB_PIX_NV12) {
    const uint8_t* c = yv.uv + static_cast<size_t>(y >> 1) * yv.uv_stride + (x & ~1);
    yuv_px(__ldg(row + x), __ldg(c), __ldg(c + 1), yv.bgr, o);
  } else {
    const uint8_t* m = row + (x & ~1) * 2;        // macropixel: U Y0 V Y1 (UYVY) or Y0 U Y1 V (YUYV)
    if (yv.fmt == VPB_PIX_UYVY) yuv_px(__ldg(m + 1 + ((x & 1) << 1)), __ldg(m), __ldg(m + 2), yv.bgr, o);
    else yuv_px(__ldg(m + ((x & 1) << 1)), __ldg(m + 1), __ldg(m + 3), yv.bgr, o);
  }
}

// OpenCV's bilinear demosaic (COLOR_Bayer**2RGB): pixel (x, y) of a Bayer image, with the border rule folded in: x, y
// are clamped to the interior [1, w-2] x [1, h-2] (OpenCV copies column 1 to 0 and w-2 to w-1, then row 1 to 0 and h-2
// to h-1), so only the 3x3 neighbourhood of an interior pixel is read, never a byte outside the descriptor.  At an R
// or B site: G = (4 neighbours + 2) >> 2, the other colour = (4 diagonals + 2) >> 2; at a G site, the colour of its
// row's R/B neighbours = (left + right + 1) >> 1 and the other = (up + down + 1) >> 1.
__device__ __forceinline__ void bayer_load(const PreImg& im, const PreCvt& cv, int y, int x, int (&o)[3]) {
  x = min(max(x, 1), im.w - 2);
  y = min(max(y, 1), im.h - 2);
  // red's site in the 2x2 block at (0, 0): RGGB (0, 0), BGGR (1, 1), GBRG (0, 1), GRBG (1, 0)
  const int rx = cv.fmt == VPB_PIX_BAYER_BGGR || cv.fmt == VPB_PIX_BAYER_GRBG;
  const int ry = cv.fmt == VPB_PIX_BAYER_BGGR || cv.fmt == VPB_PIX_BAYER_GBRG;
  const uint8_t* m = im.src + static_cast<size_t>(y) * im.stride + x;
  const uint8_t* u = m - im.stride;
  const uint8_t* d = m + im.stride;
  const int c = __ldg(m), l = __ldg(m - 1), r = __ldg(m + 1), up = __ldg(u), dn = __ldg(d);
  const int px = (x ^ rx) & 1, py = (y ^ ry) & 1;        // (0, 0): an R site, (1, 1): a B site, else G
  int R, G, B;
  if (px == py) {
    const int diag = (__ldg(u - 1) + __ldg(u + 1) + __ldg(d - 1) + __ldg(d + 1) + 2) >> 2;
    G = (l + r + up + dn + 2) >> 2;
    R = px ? diag : c;
    B = px ? c : diag;
  } else {
    const int hz = (l + r + 1) >> 1, vt = (up + dn + 1) >> 1;
    G = c;
    R = py ? vt : hz;                                     // py == 0: a G site on a row of R sites
    B = py ? hz : vt;
  }
  o[0] = cv.bgr ? B : R; o[1] = G; o[2] = cv.bgr ? R : B;
}

// Source pixel (x, y) of a non-packed image as 3 bytes in the convention's order: YUV converted, BGRA / RGBA without
// alpha, Bayer demosaiced
__device__ __forceinline__ void cvt_load(const PreImg& im, const PreCvt& cv, int y, int x, int (&o)[3]) {
  if (cv.fmt >= VPB_PIX_BAYER_RGGB) {
    bayer_load(im, cv, y, x, o);
  } else if (cv.fmt >= VPB_PIX_BGRA) {
    const uint8_t* q = im.src + static_cast<size_t>(y) * im.stride + 4 * x;
    const bool rev = (cv.fmt == VPB_PIX_BGRA) != (cv.bgr != 0);   // stored order differs from the wanted one
    const int a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2);
    o[0] = rev ? c : a; o[1] = b; o[2] = rev ? a : c;
  } else {
    yuv_load(im, cv, y, x, o);
  }
}

}  // namespace vpb
