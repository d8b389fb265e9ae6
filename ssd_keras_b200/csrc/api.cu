// Context, error reporting and host-side anchor generation for libssdk.so.
#include "common.cuh"
#include <cmath>
#include <vector>

namespace ssdk {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace ssdk

using namespace ssdk;

extern "C" int ssdk_version(void) { return SSDK_VERSION; }
extern "C" const char* ssdk_last_error(void) { return ssdk::g_err; }

extern "C" int ssdk_ctx_create(int device, ssdk_ctx** out) {
  SSDK_REQUIRE(out != nullptr, "ssdk_ctx_create: out is NULL");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("ssdk_ctx_create: no CUDA device available (%s); libssdk has no CPU fallback",
              e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    return SSDK_ERR_CUDA;
  }
  SSDK_REQUIRE(device >= 0 && device < n, "ssdk_ctx_create: device %d out of range [0,%d)", device, n);
  SSDK_CHECK_CUDA(cudaSetDevice(device));
  ssdk_ctx* c = new ssdk_ctx();
  c->device = device;
  SSDK_CHECK_CUDA(cudaGetDeviceProperties(&c->prop, device));
  c->sm_count = c->prop.multiProcessorCount;
  *out = c;
  return SSDK_OK;
}

extern "C" int ssdk_ctx_destroy(ssdk_ctx* ctx) {
  if (!ctx) return SSDK_OK;
  for (auto& w : ctx->ws) w.release();
  for (auto& s : ctx->img_stage) {
    if (s.done) { cudaEventSynchronize(s.done); cudaEventDestroy(s.done); }
    if (s.ptr) cudaFreeHost(s.ptr);
  }
  delete ctx;
  return SSDK_OK;
}

extern "C" int64_t ssdk_ctx_launch_count(const ssdk_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ------------------------------------------------------------------------------------------------
// Anchors: float64 host arithmetic, operation for operation what NumPy does in
// ssd_input_encoder.py:456-543 (no FMA contraction: this file is compiled with -ffp-contract=off).
// ------------------------------------------------------------------------------------------------
static int validate_anchor_cfg(const ssdk_anchor_cfg* c) {
  SSDK_REQUIRE(c != nullptr, "anchor cfg is NULL");
  SSDK_REQUIRE(c->n_layers > 0 && c->fm_height && c->fm_width && c->scales && c->n_aspect_ratios && c->aspect_ratios,
               "anchor cfg: missing arrays");
  SSDK_REQUIRE(c->img_height > 0 && c->img_width > 0, "anchor cfg: bad image size");
  SSDK_REQUIRE(c->coords >= 0 && c->coords <= 2, "Unexpected value for `coords`. Supported values are 'minmax', 'corners' and 'centroids'.");
  return SSDK_OK;
}

static int boxes_in_layer(const ssdk_anchor_cfg* c, int layer, int ar_off) {
  int n = c->n_aspect_ratios[layer];
  bool has1 = false;
  for (int i = 0; i < n; ++i) has1 |= (c->aspect_ratios[ar_off + i] == 1.0);
  return n + ((has1 && c->two_boxes_for_ar1) ? 1 : 0);
}

extern "C" int ssdk_anchors_count(const ssdk_anchor_cfg* c, int* out_P, int* out_n_boxes) {
  int rc = validate_anchor_cfg(c);
  if (rc) return rc;
  long long P = 0;
  int off = 0;
  for (int l = 0; l < c->n_layers; ++l) {
    int nb = boxes_in_layer(c, l, off);
    if (out_n_boxes) out_n_boxes[l] = nb;
    P += (long long)c->fm_height[l] * c->fm_width[l] * nb;
    off += c->n_aspect_ratios[l];
  }
  SSDK_REQUIRE(P < (1ll << 31), "too many anchors");
  if (out_P) *out_P = (int)P;
  return SSDK_OK;
}

// numpy.linspace(start, stop, num): y[i] = i*step + start (two roundings), y[num-1] = stop.
static void np_linspace(double start, double stop, int num, std::vector<double>& y) {
  y.resize(num);
  if (num == 1) { y[0] = 0.0 * (stop - start) + start; return; }
  double delta = stop - start;
  double step = delta / (double)(num - 1);
  for (int i = 0; i < num; ++i) {
    double t = (step == 0.0) ? ((double)i / (double)(num - 1)) * delta : (double)i * step;
    y[i] = t + start;
  }
  y[num - 1] = stop;
}

extern "C" int ssdk_anchors_generate(const ssdk_anchor_cfg* c, double* out, float* out32) {
  int rc = validate_anchor_cfg(c);
  if (rc) return rc;
  SSDK_REQUIRE(out != nullptr, "ssdk_anchors_generate: out_f64 is NULL");
  const double size = (double)(c->img_height < c->img_width ? c->img_height : c->img_width);
  const double W = (double)c->img_width, H = (double)c->img_height;
  size_t o = 0;
  int ar_off = 0;
  std::vector<double> cx, cy, bw, bh;
  for (int l = 0; l < c->n_layers; ++l) {
    const int fh = c->fm_height[l], fw = c->fm_width[l];
    const double s0 = c->scales[l], s1 = c->scales[l + 1];
    bw.clear(); bh.clear();
    for (int i = 0; i < c->n_aspect_ratios[l]; ++i) {
      double ar = c->aspect_ratios[ar_off + i];
      if (ar == 1.0) {
        double s = s0 * size;
        bw.push_back(s); bh.push_back(s);
        if (c->two_boxes_for_ar1) {
          double p = s0 * s1;
          double q = std::sqrt((double)p) * size;
          bw.push_back(q); bh.push_back(q);
        }
      } else {
        double s = s0 * size;
        double r = std::sqrt(ar);
        double w_ = s * r;
        double h_ = s / r;
        bw.push_back(w_); bh.push_back(h_);
      }
    }
    ar_off += c->n_aspect_ratios[l];
    const int nb = (int)bw.size();
    double step_h, step_w, off_h = 0.5, off_w = 0.5;
    if (c->steps_h && !std::isnan(c->steps_h[l])) { step_h = c->steps_h[l]; step_w = c->steps_w ? c->steps_w[l] : c->steps_h[l]; }
    else { step_h = H / (double)fh; step_w = W / (double)fw; }
    if (c->offsets_h && !std::isnan(c->offsets_h[l])) { off_h = c->offsets_h[l]; off_w = c->offsets_w ? c->offsets_w[l] : c->offsets_h[l]; }
    {
      double a0 = off_h * step_h, a1 = (off_h + (double)fh - 1.0) * step_h;
      np_linspace(a0, a1, fh, cy);
      double b0 = off_w * step_w, b1 = (off_w + (double)fw - 1.0) * step_w;
      np_linspace(b0, b1, fw, cx);
    }
    for (int y = 0; y < fh; ++y)
      for (int x = 0; x < fw; ++x)
        for (int b = 0; b < nb; ++b) {
          double hw = bw[b] / 2.0, hh = bh[b] / 2.0;
          double x0 = cx[x] - hw, y0 = cy[y] - hh, x1 = cx[x] + hw, y1 = cy[y] + hh;
          if (c->clip_boxes) {
            if (x0 >= W) x0 = W - 1; if (x0 < 0) x0 = 0;
            if (x1 >= W) x1 = W - 1; if (x1 < 0) x1 = 0;
            if (y0 >= H) y0 = H - 1; if (y0 < 0) y0 = 0;
            if (y1 >= H) y1 = H - 1; if (y1 < 0) y1 = 0;
          }
          if (c->normalize_coords) { x0 = x0 / W; x1 = x1 / W; y0 = y0 / H; y1 = y1 / H; }
          double* r = out + o;
          if (c->coords == SSDK_COORDS_CENTROIDS) {
            double sx = x0 + x1, sy = y0 + y1;
            r[0] = sx / 2.0; r[1] = sy / 2.0; r[2] = x1 - x0; r[3] = y1 - y0;
          } else if (c->coords == SSDK_COORDS_MINMAX) {
            r[0] = x0; r[1] = x1; r[2] = y0; r[3] = y1;
          } else {
            r[0] = x0; r[1] = y0; r[2] = x1; r[3] = y1;
          }
          o += 4;
        }
  }
  if (out32)
    for (size_t i = 0; i < o; ++i) out32[i] = (float)out[i];
  return SSDK_OK;
}
