/* oracle/t360_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.  See t360_oracle.h.
 *
 * Scalar, single-threaded, written for legibility against the reference, not speed.
 * Compile with -ffp-contract=off and no -march/-ffast-math: every float expression below
 * must round exactly where the reference's C++ rounds (SURVEY.md Appendix C ledger).
 * "ref" = the reference's Transform360/Library/VideoFrameTransform.cpp.
 */
#define _GNU_SOURCE
#include "t360_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

static const double kEps = 1e-9;              /* ref:33 */
static const double kFovDefault = 0.5333 * M_PI; /* ref:35 */

/* ------------------------------------------------------------------------------------------
 * Geometry
 * ---------------------------------------------------------------------------------------- */

/* ref:53-75 intersectSphereOffset */
static float sphere_offset_hit(float x, float y, float z, float ox, float oy, float oz) {
  float loc = x * -ox + y * -oy + z * -oz;
  float odot = ox * ox + oy * oy + oz * oz;
  float root = (float)((double)(loc * loc - odot) + 1.0);
  if (root <= 0.0f) return 0.0f;
  root = sqrtf(root);
  if (root < loc) return 0.0f;
  return root - loc;
}

/* ref:101-123 normalize_equirectangular */
static void wrap_equirect(float x, float y, float* xo, float* yo) {
  if (y >= 1.0f) {
    y = 2.0f - y;
    x += 0.5f;
  } else if (y < 0.0f) {
    y = -y;
    x += 0.5f;
  }
  if (x >= 1.0f) {
    int ip = (int)x;
    x -= (float)ip;
  } else if (x < 0.0f) {
    int ip = (int)(-x);
    x += (float)(ip + 1);
  }
  *xo = x;
  *yo = y;
}

/* ref:796-861 transformCubeFacePos: unit vector -> position in a 3x2 cubemap INPUT */
static void cube_input_pos(const T360OContext* c, float tx, float ty, float tz, float* ox, float* oy) {
  const float e = c->input_expand_coef;
  float x, y;
  if (tz <= -0.5f) {
    x = tx / tz; y = ty / tz;
    if (x >= -1.0 && x <= 1.0 && y >= -1.0 && y <= 1.0) { *ox = (5.0f + x / e) / 6.0f; *oy = (3.0f + y / e) / 4.0f; return; }
  }
  if (tz >= 0.5f) {
    x = tx / tz; y = ty / tz;
    if (x >= -1.0 && x <= 1.0 && y >= -1.0 && y <= 1.0) { *ox = (3.0f + x / e) / 6.0f; *oy = (3.0f - y / e) / 4.0f; return; }
  }
  if (tx <= -0.5f) {
    x = tz / tx; y = ty / tx;
    if (x >= -1.0 && x <= 1.0 && y >= -1.0 && y <= 1.0) { *ox = (3.0f - x / e) / 6.0f; *oy = (1.0f + y / e) / 4.0f; return; }
  }
  if (tx >= 0.5f) {
    x = tz / tx; y = ty / tx;
    if (x >= -1.0 && x <= 1.0 && y >= -1.0 && y <= 1.0) { *ox = (1.0f - x / e) / 6.0f; *oy = (1.0f - y / e) / 4.0f; return; }
  }
  if (ty <= -0.5f) {
    x = tx / ty; y = tz / ty;
    if (x >= -1.0 && x <= 1.0 && y >= -1.0 && y <= 1.0) { *ox = (1.0f - x / e) / 6.0f; *oy = (3.0f + y / e) / 4.0f; return; }
  }
  if (ty >= 0.5f) {
    x = tx / ty; y = tz / ty;
    if (x >= -1.0 && x <= 1.0 && y >= -1.0 && y <= 1.0) { *ox = (5.0f + x / e) / 6.0f; *oy = (1.0f + y / e) / 4.0f; return; }
  }
  *ox = -1.0f;
  *oy = 0.0f;
}

/* ref:863-891 transformInputPos */
static void input_pos(const T360OContext* c, float tx, float ty, float tz, float inputPixelWidth, float* ox, float* oy) {
  float d = sqrtf(tx * tx + ty * ty + tz * tz);
  if (c->input_layout == T360O_CUBEMAP_32) {
    cube_input_pos(c, tx / d, ty / d, tz / d, ox, oy);
    return;
  }
  float lon = -atan2f(-tx / d, tz / d);
  float X = (float)((double)lon / (M_PI * 2.0f) + 0.5f);
  if (c->output_layout == T360O_BARREL || c->output_layout == T360O_BARREL_SPLIT) {
    float hi = 1.0f - inputPixelWidth * 0.5f, lo = inputPixelWidth * 0.5f;
    X = X < hi ? X : hi; /* std::min(a,b): b<a ? b : a */
    X = X < lo ? lo : X; /* std::max(a,b): a<b ? b : a */
  }
  *ox = X;
  *oy = (float)((double)asinf(-ty / d) / M_PI + 0.5f);
}

/* cube basis (ref:38-49, 1118-1185): origin point p, and unit steps vx, vy, per face */
static void face_basis(int layout, int face, float p[3], float vx[3], float vy[3]) {
  static const float P0[3] = {-0.5f, -0.5f, -0.5f}, P1[3] = {0.5f, -0.5f, -0.5f}, P3[3] = {0.5f, 0.5f, -0.5f},
                     P4[3] = {-0.5f, -0.5f, 0.5f}, P5[3] = {0.5f, -0.5f, 0.5f}, P6[3] = {-0.5f, 0.5f, 0.5f};
  static const float PX[3] = {1, 0, 0}, PY[3] = {0, 1, 0}, PZ[3] = {0, 0, 1}, NX[3] = {-1, 0, 0}, NZ[3] = {0, 0, -1};
  const float *pp, *a, *b;
  if (layout == T360O_CUBEMAP_23_OFFCENTER) { /* ref:1119-1151 */
    switch (face) {
      case 0: pp = P4; a = PY; b = NZ; break;
      case 1: pp = P3; a = NX; b = PZ; break;
      case 2: pp = P5; a = PY; b = NX; break;
      case 3: pp = P1; a = NX; b = PY; break;
      case 4: pp = P1; a = PY; b = PZ; break;
      default: pp = P5; a = NX; b = NZ; break;
    }
  } else { /* ref:1153-1184 */
    switch (face) {
      case 0: pp = P5; a = NZ; b = PY; break; /* RIGHT  */
      case 1: pp = P0; a = PZ; b = PY; break; /* LEFT   */
      case 2: pp = P6; a = PX; b = NZ; break; /* TOP    */
      case 3: pp = P0; a = PX; b = PZ; break; /* BOTTOM */
      case 4: pp = P4; a = PX; b = PY; break; /* FRONT  */
      default: pp = P1; a = NX; b = PY; break; /* BACK  */
    }
  }
  memcpy(p, pp, 12); memcpy(vx, a, 12); memcpy(vy, b, 12);
}

int t360o_scaled_dims(const T360OContext* c, int outW, int outH, int* sW, int* sH) {
  *sW = (int)((double)(c->width_scale_factor * (float)outW) + 0.5);  /* ref:524 */
  *sH = (int)((double)(c->height_scale_factor * (float)outH) + 0.5); /* ref:525-526 */
  return *sW > 0 && *sH > 0;
}

/* ref:893-1316 transformPos */
int t360o_transform_pos(const T360OContext* c, float x, float y, float inputPixelWidth, float* outX, float* outY) {
  int isRight = 0;
  if (c->input_stereo_format != T360O_MONO) { /* ref:903-931 */
    if (c->output_stereo_format == T360O_LR) {
      if (x > 0.5f) { x = (x - 0.5f) / 0.5f; isRight = 1; } else { x = x / 0.5f; }
    } else if (c->output_stereo_format == T360O_TB) {
      if (y > 0.5f) {
        y = (y - 0.5f) / 0.5f;
        if (c->vflip) y = 1.0f - y;
        isRight = 1;
      } else {
        y = y / 0.5f;
      }
    }
  }

  float qx = 0, qy = 0, qz = 0, yaw = 0, pitch = 0;
  int hasMapping = 1, face = 0, vFace, hFace;
  const int L = c->output_layout;
  if (L != T360O_FLAT_FIXED) y = 1.0f - y; /* ref:936-938 */

  switch (L) { /* ref:942-1083 */
    case T360O_CUBEMAP_32:
      vFace = (int)(y * 2); hFace = (int)(x * 3);
      x = x * 3.0f - (float)hFace; y = y * 2.0f - (float)vFace;
      face = hFace + (1 - vFace) * 3;
      break;
    case T360O_CUBEMAP_23_OFFCENTER:
      vFace = (int)(y * 3); hFace = (int)(x * 2);
      x = x * 2.0f - (float)hFace; y = y * 3.0f - (float)vFace;
      face = hFace + (2 - vFace) * 2;
      break;
    case T360O_FLAT_FIXED:
      break;
    case T360O_EQUIRECT:
      yaw = (float)((double)(2.0f * x - 1.0f) * M_PI);
      pitch = (float)((double)(y - 0.5f) * M_PI);
      break;
    case T360O_BARREL:
      if (x <= 0.8f) {
        yaw = (float)((double)((2.5f * x - 1.0f) * c->expand_coef) * M_PI);
        pitch = (float)((double)((y * 0.5f - 0.25f) * c->expand_coef) * M_PI);
        face = -1;
      } else {
        vFace = (int)(y * 2);
        face = (vFace == 1) ? 2 : 3;
        x = x * 5.0f - 4.0f;
        y = y * 2.0f - (float)vFace;
      }
      break;
    case T360O_BARREL_SPLIT:
      if (3.0f * x <= 2.0f) {
        vFace = (int)(y * 2);
        yaw = (float)((double)(((3.0f / 2.0f * x - 0.5f) * c->expand_coef - (float)vFace) + 1.0f) * M_PI);
        pitch = (float)((double)(((y - 0.25f) - 0.5f * (float)vFace) * c->expand_coef) * M_PI);
        face = -1;
      } else {
        int q4 = (int)(y * 4);
        face = (q4 == 1 || q4 == 3) ? 2 : 3;
        x = x * 3.0f - 2.0f;
        switch (q4) {
          case 0: y = y * 2.0f; x = 1.0f - x; y = (0.5f - y) * c->expand_coef; break;
          case 1: y = y * 2.0f; x = 1.0f - x; y = 1.0f - c->expand_coef * (y - 0.5f); break;
          case 2: y = y * 2.0f - 0.5f; y = 1.0f - c->expand_coef * (1.0f - y); break;
          case 3: y = y * 2.0f - 1.5f; y = y * c->expand_coef; break;
          default: break;
        }
      }
      break;
    case T360O_EAC_32:
      vFace = (int)(y * 2); hFace = (int)(x * 3);
      x = x * 3.0f - (float)hFace; y = y * 2.0f - (float)vFace;
      x = (float)(tan((double)(x - 0.5f) * M_PI * 0.5f) * 0.5f + 0.5f);
      y = (float)(tan((double)(y - 0.5f) * M_PI * 0.5f) * 0.5f + 0.5f);
      face = hFace + (1 - vFace) * 3;
      break;
    default:
      return 0;
  }

  if (L == T360O_FLAT_FIXED) { /* ref:1265-1271 */
    float X = ((x - 0.5f) * c->fixed_hfov + c->fixed_yaw) / 360.0f + 0.5f;
    float Y = ((y - 0.5f) * c->fixed_vfov - c->fixed_pitch) / 180.0f + 0.5f;
    wrap_equirect(X, Y, outX, outY);
  } else {
    if (L == T360O_EQUIRECT || ((L == T360O_BARREL || L == T360O_BARREL_SPLIT) && face < 0)) { /* ref:1092-1101 */
      float sy = sinf(yaw), sp = sinf(pitch), cy = cosf(yaw), cp = cosf(pitch);
      qx = sy * cp; qy = sp; qz = cy * cp;
    } else {
      if (L == T360O_BARREL || L == T360O_BARREL_SPLIT) { /* ref:1106-1113 */
        float r2 = (x - 0.5f) * (x - 0.5f) + (y - 0.5f) * (y - 0.5f);
        if (r2 > 0.25f * c->expand_coef * c->expand_coef) hasMapping = 0;
      }
      if (hasMapping) {
        float p[3], vx[3], vy[3];
        x = (x - 0.5f) * c->expand_coef + 0.5f; /* ref:1115-1116 */
        y = (y - 0.5f) * c->expand_coef + 0.5f;
        face_basis(L, face, p, vx, vy);
        qx = p[0] + vx[0] * x + vy[0] * y; /* ref:1187-1189 */
        qy = p[1] + vx[1] * x + vy[1] * y;
        qz = p[2] + vx[2] * x + vy[2] * y;
      }
    }
    if (hasMapping) {
      const float ox = c->fixed_cube_offcenter_x, oy = c->fixed_cube_offcenter_y, oz = c->fixed_cube_offcenter_z;
      if (fabsf(ox) > kEps || fabsf(oy) > kEps || fabsf(oz) > kEps) { /* ref:1192-1230 */
        float d = sqrtf(qx * qx + qy * qy + qz * qz), dist;
        qx = qx / d; qy = qy / d; qz = qz / d;
        if (c->is_horizontal_offset) {
          d = sqrtf(qx * qx + qz * qz);
          qx = qx / d; qy = qy / d; qz = qz / d;
          dist = sphere_offset_hit(qx, 0, qz, ox, 0, oz);
          if (dist > 0.0f) { qx = qx * dist - ox; qz = qz * dist - oz; }
        } else {
          dist = sphere_offset_hit(qx, qy, qz, ox, oy, oz);
          if (dist > 0.0f) { qx = qx * dist - ox; qy = qy * dist - oy; qz = qz * dist - oz; }
        }
      }
      /* ref:1233-1246: trig in double, stored to float */
      float s1 = (float)sin((double)c->fixed_yaw * M_PI / 180.0f), s2 = (float)sin((double)c->fixed_pitch * M_PI / 180.0f),
            s3 = (float)sin((double)c->fixed_roll * M_PI / 180.0f), c1 = (float)cos((double)c->fixed_yaw * M_PI / 180.0f),
            c2 = (float)cos((double)c->fixed_pitch * M_PI / 180.0f), c3 = (float)cos((double)c->fixed_roll * M_PI / 180.0f);
      float tx = qx * (c1 * c3 + s1 * s2 * s3) - qy * (c3 * s1 * s2 - c1 * s3) + qz * (c2 * s1);
      float ty = qx * (c2 * s3) - qy * (c2 * c3) + qz * (-s2);
      float tz = qx * (c1 * s2 * s3 - c3 * s1) - qy * (c1 * c3 * s2 + s1 * s3) + qz * (c1 * c2);
      ty = -ty;
      input_pos(c, tx, ty, tz, inputPixelWidth, outX, outY);
    }
  }

  if (hasMapping) { /* ref:1278-1300 */
    if (c->input_stereo_format == T360O_TB) {
      *outY = isRight ? *outY * 0.5f + 0.5f : *outY * 0.5f;
    } else if (c->input_stereo_format == T360O_LR) {
      *outX = isRight ? *outX * 0.5f + 0.5f : *outX * 0.5f;
    }
  } else {
    *outX = -1;
    *outY = 0;
  }
  return 1;
}

/* ref:504-556 generateMapForPlane (map part) */
int t360o_generate_map(const T360OContext* c, int inW, int inH, int outW, int outH, float* map) {
  int sW, sH;
  if (!t360o_scaled_dims(c, outW, outH, &sW, &sH)) return 0;
  float ipw = 1.0f / (float)inW;
  if (c->input_stereo_format == T360O_LR) ipw *= 2;
  for (int i = 0; i < sH; ++i) {
    for (int j = 0; j < sW; ++j) {
      float y = ((float)i + 0.5f) / (float)sH, x = ((float)j + 0.5f) / (float)sW, ox, oy;
      if (!t360o_transform_pos(c, x, y, ipw, &ox, &oy)) return 0;
      map[((size_t)i * sW + j) * 2 + 0] = ox * (float)inW - 0.5f;
      map[((size_t)i * sW + j) * 2 + 1] = oy * (float)inH - 0.5f;
    }
  }
  return 1;
}

/* ------------------------------------------------------------------------------------------
 * Low-pass plan
 * ---------------------------------------------------------------------------------------- */

/* ref:78-94 calculateKernel; returns tap count, writes taps[] */
static int gauss_taps(float sigma, float* taps, int maxTaps) {
  int half = (int)(sigma * 2);
  int n = half * 2 + 1;
  if (n > maxTaps || n < 1) return -1;
  float sum = 0;
  float comp = fabsf(sigma) < kEps ? 0 : (float)(0.5 / (double)(sigma * sigma));
  for (int u = -half; u <= half; ++u) {
    float v = expf(-((float)(u * u) * comp));
    taps[u + half] = v;
    sum += v;
  }
  const float inv = (float)(1.0 / (double)sum); /* cv::Mat /= : convertTo(-1, 1./s) in float */
  for (int i = 0; i < n; ++i) taps[i] = taps[i] * inv;
  return n;
}

/* ref:126-170 */
static double ang_dist(double yaw1, double pitch1, double yaw2, double pitch2) {
  return acos(sin(pitch1) * sin(pitch2) + cos(pitch1) * cos(pitch2) * cos(yaw1 - yaw2));
}
static double sampling_arc(double offset, double arc) {
  return M_PI - 2 * atan2(cos(0.5 * arc) - offset, sin(0.5 * arc));
}
static double sph_area(double angle) { return (1 - cos(0.5 * angle)) * 2 * M_PI; }
static double effective_ratio(double ad, double offset) {
  const double fov = kFovDefault;
  double major;
  if (ad - kEps > fov / 2) {
    if (ad + fov / 2 > M_PI) {
      double e1 = sampling_arc(offset, (2 * M_PI - ad - fov / 2) * 2) / 2;
      double e2 = sampling_arc(offset, (ad - fov / 2) * 2) / 2;
      major = (2 * M_PI - e1 - e2) / fov;
    } else {
      major = (sampling_arc(offset, 2 * ad + fov) - sampling_arc(offset, 2 * ad - fov)) / 2 / fov;
    }
  } else {
    major = (sampling_arc(offset, 2 * ad + fov) + sampling_arc(offset, fov - 2 * ad)) / 2 / fov;
  }
  double cov = ang_dist(ad, 0.5 * fov, 0.0, 0.0);
  double minor = sampling_arc(offset, cov * 2) / (cov * 2);
  double r = major * minor * sph_area(fov) / (4 * M_PI);
  return r < 1.0 ? r : 1.0;
}

typedef struct {
  const T360OContext* c;
  T360OSegment* segs;
  int maxSegs, nsegs;
  float* taps;
  int maxTaps, ntaps;
  int failed;
} PlanOut;

static int push_taps(PlanOut* o, float sigma) {
  int off = o->ntaps;
  int n = gauss_taps(sigma, o->taps + off, o->maxTaps - off);
  if (n < 0) { o->failed = 1; return -1; }
  o->ntaps += n;
  return off;
}

/* ref:210-297 generateKernelAndFilteringConfig */
static void plan_band(PlanOut* o, int top, int bottom, float angle, float sigmaY, int kyOff, int nky, int inW, int inH) {
  const T360OContext* c = o->c;
  double sxd = (double)sigmaY / ((double)cosf(angle) + kEps);
  float sigmaX = (float)(0.5 * inW < sxd ? 0.5 * inW : sxd);
  int kxOff = push_taps(o, sigmaX);
  if (kxOff < 0) return;
  int nkx = o->ntaps - kxOff;
  int nH = c->adjust_kernel ? c->num_horizontal_segments : 1;
  int segW = (int)ceil(1.0 * inW / nH);
  double baseRatio = effective_ratio(0.0, 0.0);
  for (int i = 0; i < nH && i * segW < inW; ++i) {
    if (o->nsegs >= o->maxSegs) { o->failed = 1; return; }
    T360OSegment* s = &o->segs[o->nsegs++];
    int w = segW < inW - i * segW ? segW : inW - i * segW;
    s->left = i * segW; s->top = top; s->width = w; s->height = bottom - top + 1;
    if (c->adjust_kernel) {
      float avgYaw = (float)(2 * M_PI * ((i * segW + 0.5 * w) - 0.5 * inW) / inW);
      float avgPitch = (float)(0.5 * M_PI * (inH - top - bottom) / inH);
      float yaw = (float)((double)c->fixed_yaw * M_PI / 180.0f);
      float pitch = (float)((double)c->fixed_pitch * M_PI / 180.0f);
      float offset = fabsf(c->fixed_cube_offcenter_z);
      if (fabsf(yaw) < kEps && fabsf(pitch) < kEps &&
          (fabsf(c->fixed_cube_offcenter_x) > kEps || fabsf(c->fixed_cube_offcenter_y) > kEps ||
           c->fixed_cube_offcenter_z > kEps)) {
        offset = sqrtf(c->fixed_cube_offcenter_x * c->fixed_cube_offcenter_x +
                       c->fixed_cube_offcenter_y * c->fixed_cube_offcenter_y +
                       c->fixed_cube_offcenter_z * c->fixed_cube_offcenter_z);
        yaw = atan2f(-c->fixed_cube_offcenter_x / offset, -c->fixed_cube_offcenter_z / offset);
        pitch = asinf(-c->fixed_cube_offcenter_y / offset);
      }
      double dist = ang_dist(yaw, pitch, avgYaw, avgPitch);
      double ratio = effective_ratio(dist, offset);
      double scale = (double)c->kernel_adjust_factor * baseRatio / ratio;
      s->kx_off = push_taps(o, (float)(scale * (double)sigmaX));
      if (s->kx_off < 0) return;
      s->nkx = o->ntaps - s->kx_off;
      s->ky_off = push_taps(o, (float)(scale * (double)sigmaY));
      if (s->ky_off < 0) return;
      s->nky = o->ntaps - s->ky_off;
    } else {
      s->kx_off = kxOff; s->nkx = nkx; s->ky_off = kyOff; s->nky = nky;
    }
  }
}

/* ref:318-364 generateKernelsAndFilteringConfigs */
static void plan_halves(PlanOut* o, int startTop, int startBottom, float sigmaY, int kyOff, int nky, int base, int inW, int inH) {
  for (int bottom = startBottom; bottom >= 0; bottom -= base) {
    int top = bottom - base + 1 > 0 ? bottom - base + 1 : 0;
    float angle = (float)(0.5 * M_PI * (inH - top - bottom) / inH);
    plan_band(o, top, bottom, angle, sigmaY, kyOff, nky, inW, inH);
  }
  for (int top = startTop; top < inH; top += base) {
    int bottom = top + base - 1 < inH - 1 ? top + base - 1 : inH - 1;
    float angle = (float)(0.5 * M_PI * (top + bottom - inH) / inH);
    plan_band(o, top, bottom, angle, sigmaY, kyOff, nky, inW, inH);
  }
}

/* ref:367-501 calcualteFilteringConfig */
int t360o_filter_plan(const T360OContext* c, int inW, int inH, int outW, int outH, T360OSegment* segs, int maxSegs,
                      float* taps, int maxTaps, int* ntaps) {
  if (c->input_stereo_format == T360O_LR) inW = (int)(inW * 0.5);
  else if (c->input_stereo_format == T360O_TB) inH = (int)(inH * 0.5);
  if (c->output_stereo_format == T360O_LR) outW = (int)(outW * 0.5);
  else if (c->output_stereo_format == T360O_TB) outH = (int)(outH * 0.5);

  float hFov, vFov;
  switch (c->output_layout) {
    case T360O_CUBEMAP_32: hFov = 270.0f; vFov = 180.0f; break;
    case T360O_CUBEMAP_23_OFFCENTER: hFov = 180.0f; vFov = 270.0f; break;
    case T360O_FLAT_FIXED: hFov = c->fixed_hfov; vFov = c->fixed_vfov; break;
    case T360O_EQUIRECT: hFov = 360.0f; vFov = 180.0f; break;
    case T360O_BARREL:
    case T360O_BARREL_SPLIT: hFov = 450.0f; vFov = 90.0f; break;
    case T360O_EAC_32: hFov = 270.0f; vFov = 180.0f; break;
    default: *ntaps = 0; return 0;
  }
  float a = (float)inW / 360.0f, b = (float)inH / 180.0f;
  float inRes = b < a ? b : a;
  float p = (float)outW / hFov, q = (float)outH / vFov;
  float outRes = p < q ? q : p;
  float v = c->kernel_height_scale_factor * inRes / outRes;
  v = c->min_kernel_half_height < v ? v : c->min_kernel_half_height; /* std::max(min_khh, v) */
  v = v < c->max_kernel_half_height ? v : c->max_kernel_half_height; /* std::min(max_khh, v) */
  float sigmaY = 0.5f * v;

  PlanOut o = {c, segs, maxSegs, 0, taps, maxTaps, 0, 0};
  int kyOff = push_taps(&o, sigmaY);
  if (kyOff < 0) return -1;
  int nky = o.ntaps - kyOff;
  int base = (int)ceil(1.0 * inH / c->num_vertical_segments);
  if (c->num_vertical_segments % 2 == 0) {
    plan_halves(&o, (int)(0.5 * inH), (int)(0.5 * inH - 1), sigmaY, kyOff, nky, base, inW, inH);
  } else {
    int top = (int)(0.5 * (inH - base));
    int bottom = top + base - 1;
    plan_band(&o, top, bottom, 0, sigmaY, kyOff, nky, inW, inH);
    plan_halves(&o, bottom + 1, top - 1, sigmaY, kyOff, nky, base, inW, inH);
  }
  if (o.failed) return -1;
  *ntaps = o.ntaps;
  return o.nsegs;
}

/* ------------------------------------------------------------------------------------------
 * cv::remap arithmetic (OpenCV 4.x imgproc/imgwarp.cpp; SURVEY.md Appendix A)
 * ---------------------------------------------------------------------------------------- */

int t360o_remap_ksize(int interp) {
  switch (interp) {
    case T360O_NEAREST: return 1;
    case T360O_LINEAR: return 2;
    case T360O_CUBIC: return 4;
    case T360O_LANCZOS4: return 8;
    default: return 0;
  }
}

static void coeffs_1d(int interp, float x, float* w) {
  if (interp == T360O_LINEAR) {
    w[0] = 1.f - x;
    w[1] = x;
  } else if (interp == T360O_CUBIC) {
    const float A = -0.75f;
    w[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
    w[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
    w[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
    w[3] = 1.f - w[0] - w[1] - w[2];
  } else { /* Lanczos4 */
    static const double s45 = 0.70710678118654752440084436210485;
    static const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
    if (x < FLT_EPSILON) {
      for (int i = 0; i < 8; i++) w[i] = 0;
      w[3] = 1;
      return;
    }
    float sum = 0;
    double y0 = -(x + 3) * M_PI * 0.25, s0 = sin(y0), c0 = cos(y0);
    for (int i = 0; i < 8; i++) {
      double y = -(x + 3 - i) * M_PI * 0.25;
      w[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
      sum += w[i];
    }
    sum = 1.f / sum;
    for (int i = 0; i < 8; i++) w[i] *= sum;
  }
}

static int16_t sat_i16_round(float v) {
  long r = lrintf(v); /* round-half-even under the default rounding mode, like cvRound */
  return (int16_t)(r < -32768 ? -32768 : (r > 32767 ? 32767 : r));
}

void t360o_build_itab(int interp, int16_t* itab) {
  const int k = t360o_remap_ksize(interp);
  if (k < 2) return;
  float t1[32 * 8];
  const float scale = 1.f / 32;
  for (int i = 0; i < 32; i++) coeffs_1d(interp, (float)i * scale, t1 + i * k);
  for (int i = 0; i < 32; i++) {
    for (int j = 0; j < 32; j++) {
      int16_t* it = itab + (size_t)(i * 32 + j) * k * k;
      int isum = 0;
      for (int k1 = 0; k1 < k; k1++) {
        float vy = t1[i * k + k1];
        for (int k2 = 0; k2 < k; k2++) {
          float v = vy * t1[j * k + k2];
          isum += it[k1 * k + k2] = sat_i16_round(v * 32768.0f);
        }
      }
      if (isum != 32768 && k == 2) {
        /* only phase (0,0): 1.0*32768 saturates to 32767.  OpenCV's fix-up scans [1,3)x[1,3), i.e. entry
         * (1,1) of this phase and three not-yet-written entries of the next one (static zeros), so the
         * missing 1 lands on entry (1,1).  The interpolated value is unaffected (|b-a| < 16384). */
        it[3] = (int16_t)(it[3] - (isum - 32768));
      }
      if (isum != 32768 && k > 2) {
        int diff = isum - 32768, h = k / 2, Mk1 = h, Mk2 = h, mk1 = h, mk2 = h;
        for (int k1 = h; k1 < h + 2; k1++)
          for (int k2 = h; k2 < h + 2; k2++) {
            if (it[k1 * k + k2] < it[mk1 * k + mk2]) { mk1 = k1; mk2 = k2; }
            else if (it[k1 * k + k2] > it[Mk1 * k + Mk2]) { Mk1 = k1; Mk2 = k2; }
          }
        if (diff < 0) it[Mk1 * k + Mk2] = (int16_t)(it[Mk1 * k + Mk2] - diff);
        else it[mk1 * k + mk2] = (int16_t)(it[mk1 * k + mk2] - diff);
      }
    }
  }
}

static int wrap_idx(int p, int n) { /* cv::borderInterpolate(BORDER_WRAP) */
  if (p < 0) p -= ((p - n + 1) / n) * n;
  if (p >= n) p %= n;
  return p;
}

static int border_idx(int p, int n, int border) {
  if ((unsigned)p < (unsigned)n) return p;
  if (border == T360O_BORDER_REPLICATE) return p < 0 ? 0 : n - 1;
  if (border == T360O_BORDER_WRAP) return wrap_idx(p, n);
  if (border == T360O_BORDER_TRANSPARENT) { /* borderType1 = REFLECT_101 inside remap */
    if (n == 1) return 0;
    do {
      if (p < 0) p = -p;
      else p = n - 1 - (p - n) - 1;
    } while ((unsigned)p >= (unsigned)n);
    return p;
  }
  return -1; /* constant */
}

/* cvRound(float) as OpenCV computes it on x86 (cvtss2si / cvtps2dq, also in its SIMD paths): round half to even, and
 * the "integer indefinite" value INT_MIN for NaN and for values outside the int range.  It matters: an off-centre
 * projection with is_horizontal_offset divides by zero at the poles (ref:1203-1206), the map holds NaN there, and
 * cv::remap then samples column/row sat16(INT_MIN >> 5) = -32768 under BORDER_WRAP (pinned against cv2 in
 * tests/test_oracle_pin.py). */
static int cv_round_f32(float v) {
  if (!(v >= -2147483648.0f && v < 2147483648.0f)) return (-2147483647 - 1);
  return (int)lrintf(v);
}

static int sat_i16(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

void t360o_remap_u8(const uint8_t* src, int sw, int sh, size_t spitch, uint8_t* dst, int dw, int dh, size_t dpitch,
                    const float* mapxy, int interp, int border) {
  const int k = t360o_remap_ksize(interp);
  int16_t* itab = NULL;
  if (k >= 2) {
    itab = (int16_t*)malloc((size_t)1024 * k * k * sizeof(int16_t));
    t360o_build_itab(interp, itab);
  }
  for (int dy = 0; dy < dh; dy++) {
    uint8_t* D = dst + (size_t)dy * dpitch;
    const float* M = mapxy + (size_t)dy * dw * 2;
    for (int dx = 0; dx < dw; dx++) {
      float fx = M[dx * 2], fy = M[dx * 2 + 1];
      if (k == 1) {
        int sx = sat_i16(cv_round_f32(fx)), sy = sat_i16(cv_round_f32(fy));
        if ((unsigned)sx < (unsigned)sw && (unsigned)sy < (unsigned)sh) {
          D[dx] = src[(size_t)sy * spitch + sx];
        } else if (border == T360O_BORDER_TRANSPARENT) {
          continue;
        } else if (border == T360O_BORDER_CONSTANT) {
          D[dx] = 0;
        } else {
          sx = border_idx(sx, sw, border);
          sy = border_idx(sy, sh, border);
          D[dx] = src[(size_t)sy * spitch + sx];
        }
        continue;
      }
      int X = cv_round_f32(fx * 32.0f), Y = cv_round_f32(fy * 32.0f);
      int a = (Y & 31) * 32 + (X & 31);
      int sx = sat_i16(X >> 5) - (k / 2 - 1), sy = sat_i16(Y >> 5) - (k / 2 - 1);
      const int16_t* w = itab + (size_t)a * k * k;
      int inlier = sx >= 0 && sy >= 0 && sx + k <= sw && sy + k <= sh;
      int acc = 0;
      if (inlier) {
        for (int r = 0; r < k; r++) {
          const uint8_t* S = src + (size_t)(sy + r) * spitch + sx;
          for (int c = 0; c < k; c++) acc += S[c] * w[r * k + c];
        }
      } else {
        if (border == T360O_BORDER_TRANSPARENT) {
          /* every interpolator leaves the pixel alone when its anchor sample lies outside the source */
          int ax = sx + (k / 2 - 1), ay = sy + (k / 2 - 1);
          if ((unsigned)ax >= (unsigned)sw || (unsigned)ay >= (unsigned)sh) continue;
          if (k == 2) {
            /* cv2 4.13 remapBilinear: anchor inside but the 2x2 window sticks out (last row / column): blend the
             * taps that exist and renormalise by their weight, rounding half up (pinned against cv2 on 12 000
             * edge samples, tests/test_oracle_pin.py) */
            long num = 0, den = 0;
            for (int r = 0; r < 2; r++)
              for (int c = 0; c < 2; c++)
                if (sx + c < sw && sy + r < sh) {
                  num += (long)w[r * 2 + c] * src[(size_t)(sy + r) * spitch + sx + c];
                  den += w[r * 2 + c];
                }
            if (den > 0) D[dx] = (uint8_t)((2 * num + den) / (2 * den));
            continue;
          }
        }
        if (border == T360O_BORDER_CONSTANT && (sx >= sw || sx + k <= 0 || sy >= sh || sy + k <= 0)) {
          D[dx] = 0;
          continue;
        }
        for (int r = 0; r < k; r++) {
          int yy = border_idx(sy + r, sh, border);
          if (yy < 0) continue;
          for (int c = 0; c < k; c++) {
            int xx = border_idx(sx + c, sw, border);
            if (xx >= 0) acc += src[(size_t)yy * spitch + xx] * w[r * k + c];
          }
        }
      }
      int v = (acc + (1 << 14)) >> 15;
      D[dx] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
  }
  free(itab);
}

/* ------------------------------------------------------------------------------------------
 * cv::sepFilter2D arithmetic for u8 -> u8 with float32 symmetric kernels, BORDER_REPLICATE,
 * on a NON-ISOLATED roi (OpenCV 4.x filter.simd.hpp RowFilter / SymmColumnFilter; Appendix B)
 * ---------------------------------------------------------------------------------------- */
static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* cv2 4.13.0 runs this through its AVX2/AVX512-dispatched build of filter.simd.hpp, where the
 * compiler has contracted "s += f*S[k]" into fused multiply-adds: the model that reproduces it
 * bit-for-bit (0 mismatches on 4 x 1 Mpx noise planes, tests/test_oracle_pin.py) is
 *   row:    s = kx[0]*p[0];            s = fma(kx[i], p[i], s)              i = 1..n-1
 *   column: s = ky[h]*R[y];            s = fma(ky[h+i], R[y+i] + R[y-i], s) i = 1..h
 *   dst = saturate_u8(rint(s))  (half-even)
 * (SURVEY.md Appendix B modelled the same order without the fusion; that differs in ~4 px per
 * million on noise, always at a rounding tie.)  Requires a CPU with FMA, like the dispatch it models. */
__attribute__((target("fma")))
void t360o_sepfilter_roi_u8(const uint8_t* parent, int pw, int ph, size_t ppitch, int rx, int ry, int rw, int rh,
                            uint8_t* dstParent, size_t dpitch, const float* kx, int nkx, const float* ky, int nky) {
  const int hx = nkx / 2, hy = nky / 2;
  const int rows = rh + 2 * hy;
  float* R = (float*)malloc((size_t)rows * rw * sizeof(float));
  for (int r = 0; r < rows; r++) {
    const uint8_t* S = parent + (size_t)clampi(ry - hy + r, 0, ph - 1) * ppitch;
    float* Rr = R + (size_t)r * rw;
    for (int x = 0; x < rw; x++) {
      float s = kx[0] * (float)S[clampi(rx + x - hx, 0, pw - 1)];
      for (int i = 1; i < nkx; i++) s = __builtin_fmaf(kx[i], (float)S[clampi(rx + x - hx + i, 0, pw - 1)], s);
      Rr[x] = s;
    }
  }
  for (int y = 0; y < rh; y++) {
    uint8_t* D = dstParent + (size_t)(ry + y) * dpitch + rx;
    const float* Rc = R + (size_t)(y + hy) * rw;
    for (int x = 0; x < rw; x++) {
      float s = ky[hy] * Rc[x];
      for (int i = 1; i <= hy; i++) s = __builtin_fmaf(ky[hy + i], Rc[x + (size_t)i * rw] + Rc[x - (ptrdiff_t)i * rw], s);
      long v = lrintf(s);
      D[x] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
  }
  free(R);
}

/* ref:579-704 runFiltering + filterPlane: dst starts as zeros; tiles applied at offset 0 and, for LR/TB
 * input, again at the half-plane offset. */
void t360o_filter_plane(const T360OContext* c, const uint8_t* src, int w, int h, size_t spitch, uint8_t* dst,
                        size_t dpitch, const T360OSegment* segs, int nsegs, const float* taps) {
  for (int y = 0; y < h; y++) memset(dst + (size_t)y * dpitch, 0, (size_t)w);
  int passes = 1, offX[2] = {0, 0}, offY[2] = {0, 0};
  if (c->input_stereo_format == T360O_LR) { passes = 2; offX[1] = (int)(0.5 * w); }
  else if (c->input_stereo_format == T360O_TB) { passes = 2; offY[1] = (int)(0.5 * h); }
  for (int p = 0; p < passes; p++)
    for (int i = 0; i < nsegs; i++) {
      const T360OSegment* s = &segs[i];
      int left = s->left + offX[p], top = s->top + offY[p];
      if (left < 0 || top < 0 || left + s->width > w || top + s->height > h) continue; /* cv::Mat roi throws; ref:198 swallows */
      t360o_sepfilter_roi_u8(src, w, h, spitch, left, top, s->width, s->height, dst, dpitch, taps + s->kx_off, s->nkx,
                             taps + s->ky_off, s->nky);
    }
}

/* ------------------------------------------------------------------------------------------
 * cv::resize(INTER_AREA), 8-bit, one channel, shrinking (OpenCV 4.x imgproc/resize.cpp)
 * ---------------------------------------------------------------------------------------- */
typedef struct { int di, si; float alpha; } AreaTap;

/* computeResizeAreaTab */
static int area_tab(int ssize, int dsize, double scale, AreaTap* tab) {
  int k = 0;
  for (int dx = 0; dx < dsize; dx++) {
    double fsx1 = dx * scale, fsx2 = fsx1 + scale;
    double cell = scale < ssize - fsx1 ? scale : ssize - fsx1;
    int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
    if (sx2 > ssize - 1) sx2 = ssize - 1;
    if (sx1 > sx2) sx1 = sx2;
    if (sx1 - fsx1 > 1e-3) { tab[k].di = dx; tab[k].si = sx1 - 1; tab[k++].alpha = (float)((sx1 - fsx1) / cell); }
    for (int sx = sx1; sx < sx2; sx++) { tab[k].di = dx; tab[k].si = sx; tab[k++].alpha = (float)(1.0 / cell); }
    if (fsx2 - sx2 > 1e-3) {
      double a = fsx2 - sx2;
      if (a > 1.0) a = 1.0;
      if (a > cell) a = cell;
      tab[k].di = dx; tab[k].si = sx2; tab[k++].alpha = (float)(a / cell);
    }
  }
  return k;
}

/* cv::resize(INTER_AREA) when at least one axis ENLARGES (scale < 1): OpenCV 4.x imgproc/resize.cpp emulates it with its
 * 8-bit fixed-point bilinear kernel and "area mode" coefficients on BOTH axes:
 *   sx = floor(dx * scale);  fx = (float)((dx + 1) - (sx + 1) * inv_scale);  fx = fx <= 0 ? 0 : fx - floor(fx)
 *   (clamped at the last source sample; dx >= xmax copies S[sx] * 2048), coefficients = cvRound({1 - fx, fx} * 2048),
 *   rows:    H[dx] = S[sx] * a0 + S[sx + 1] * a1                                  (HResizeLinear, int)
 *   columns: dst   = (((b0 * (H0 >> 4)) >> 16) + ((b1 * (H1 >> 4)) >> 16) + 2) >> 2   (VResizeLinear<uchar> specialisation)
 * Pinned bit-exact against cv2 4.13 in tests/test_oracle_pin.py (the reference reaches it with *_scale_factor < 1,
 * ref:755-777). */
static void area_linear_axis(int dn, int sn, double scale, double inv, int* ofs, short* coef, int* dmax) {
  *dmax = dn;
  for (int d = 0; d < dn; d++) {
    int s = (int)floor(d * scale);
    float f = (float)((d + 1) - (s + 1) * inv);
    f = f <= 0 ? 0.f : f - (float)floor(f);
    if (s < 0) { f = 0; s = 0; }
    if (s + 1 >= sn) {
      if (d < *dmax) *dmax = d;
      if (s >= sn - 1) { f = 0; s = sn - 1; }
    }
    ofs[d] = s;
    long c0 = lrintf((1.f - f) * 2048.f), c1 = lrintf(f * 2048.f);
    coef[2 * d] = (short)(c0 > 32767 ? 32767 : c0);
    coef[2 * d + 1] = (short)(c1 > 32767 ? 32767 : c1);
  }
}

static int resize_area_enlarge_u8(const uint8_t* src, int sw, int sh, size_t spitch, uint8_t* dst, int dw, int dh, size_t dpitch) {
  const double inv_x = (double)dw / sw, inv_y = (double)dh / sh, scale_x = 1.0 / inv_x, scale_y = 1.0 / inv_y;
  int* xofs = (int*)malloc(sizeof(int) * ((size_t)dw + dh));
  int* yofs = xofs + dw;
  short* xa = (short*)malloc(sizeof(short) * 2 * ((size_t)dw + dh));
  short* yb = xa + 2 * (size_t)dw;
  int* rows = (int*)malloc(sizeof(int) * 2 * (size_t)dw);
  int xmax, ymax;
  area_linear_axis(dw, sw, scale_x, inv_x, xofs, xa, &xmax);
  area_linear_axis(dh, sh, scale_y, inv_y, yofs, yb, &ymax);
  for (int dy = 0; dy < dh; dy++) {
    for (int k = 0; k < 2; k++) {
      int sy = yofs[dy] + k;
      sy = sy < 0 ? 0 : (sy > sh - 1 ? sh - 1 : sy);
      const uint8_t* S = src + (size_t)sy * spitch;
      int* H = rows + (size_t)k * dw;
      for (int dx = 0; dx < dw; dx++) {
        const int sx = xofs[dx];
        H[dx] = dx < xmax ? S[sx] * xa[2 * dx] + S[sx + 1] * xa[2 * dx + 1] : S[sx] * 2048;
      }
    }
    const int b0 = yb[2 * dy], b1 = yb[2 * dy + 1];
    for (int dx = 0; dx < dw; dx++) {
      const int v = (((b0 * (rows[dx] >> 4)) >> 16) + ((b1 * (rows[dw + dx] >> 4)) >> 16) + 2) >> 2;
      dst[(size_t)dy * dpitch + dx] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
  }
  free(rows); free(xa); free(xofs);
  return 1;
}

int t360o_resize_area_u8(const uint8_t* src, int sw, int sh, size_t spitch, uint8_t* dst, int dw, int dh, size_t dpitch) {
  const double scale_x = 1.0 / ((double)dw / sw), scale_y = 1.0 / ((double)dh / sh); /* cv::resize: 1./inv_scale */
  if (scale_x < 1.0 || scale_y < 1.0) return resize_area_enlarge_u8(src, sw, sh, spitch, dst, dw, dh, dpitch);
  const int isx = (int)lrint(scale_x), isy = (int)lrint(scale_y);
  if (fabs(scale_x - isx) < DBL_EPSILON && fabs(scale_y - isy) < DBL_EPSILON) { /* resizeAreaFast_ */
    const int area = isx * isy;
    const float scale = 1.f / area;
    for (int dy = 0; dy < dh; dy++)
      for (int dx = 0; dx < dw; dx++) {
        int sum = 0;
        for (int y = 0; y < isy; y++)
          for (int x = 0; x < isx; x++) sum += src[(size_t)(dy * isy + y) * spitch + dx * isx + x];
        int v;
        if (isx == 2 && isy == 2) v = (sum + 2) >> 2;
        else v = (int)lrintf((float)sum * scale);
        dst[(size_t)dy * dpitch + dx] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
      }
    return 1;
  }
  AreaTap* xt = (AreaTap*)malloc(sizeof(AreaTap) * ((size_t)sw * 2 + dw * 2));
  AreaTap* yt = (AreaTap*)malloc(sizeof(AreaTap) * ((size_t)sh * 2 + dh * 2));
  const int nx = area_tab(sw, dw, scale_x, xt), ny = area_tab(sh, dh, scale_y, yt);
  float* buf = (float*)malloc(sizeof(float) * dw * 2);
  float* sum = buf + dw;
  int prev = yt[0].di;
  for (int dx = 0; dx < dw; dx++) sum[dx] = 0;
  for (int j = 0; j < ny; j++) { /* ResizeArea_Invoker */
    const uint8_t* S = src + (size_t)yt[j].si * spitch;
    const float beta = yt[j].alpha;
    for (int dx = 0; dx < dw; dx++) buf[dx] = 0;
    for (int k = 0; k < nx; k++) buf[xt[k].di] += (float)S[xt[k].si] * xt[k].alpha;
    if (yt[j].di != prev) {
      for (int dx = 0; dx < dw; dx++) {
        long v = lrintf(sum[dx]);
        dst[(size_t)prev * dpitch + dx] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
        sum[dx] = beta * buf[dx];
      }
      prev = yt[j].di;
    } else {
      for (int dx = 0; dx < dw; dx++) sum[dx] += beta * buf[dx];
    }
  }
  for (int dx = 0; dx < dw; dx++) {
    long v = lrintf(sum[dx]);
    dst[(size_t)prev * dpitch + dx] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
  }
  free(buf); free(xt); free(yt);
  return 1;
}

/* ref:707-794 transformPlane, both branches */
int t360o_transform_plane(const T360OContext* c, const uint8_t* src, int inW, int inH, size_t spitch, uint8_t* dst,
                          int outW, int outH, size_t dpitch, const float* map, int mapW, int mapH, int mapIndex,
                          const T360OSegment* segs, int nsegs, const float* taps) {
  int interp = c->interpolation_alg;
  if (t360o_remap_ksize(interp) == 0) return 1; /* ref:780-784: prints, still returns true */
  const int needResize = outW != mapW || outH != mapH; /* ref:735-737 */
  const int barrel = c->output_layout == T360O_BARREL || c->output_layout == T360O_BARREL_SPLIT;
  int border = barrel ? T360O_BORDER_TRANSPARENT : T360O_BORDER_WRAP;
  const uint8_t* in = src;
  size_t inPitch = spitch;
  uint8_t* blurred = NULL;
  if (c->enable_low_pass_filter) {
    blurred = (uint8_t*)malloc((size_t)inW * inH);
    t360o_filter_plane(c, src, inW, inH, spitch, blurred, (size_t)inW, segs, nsegs, taps);
    in = blurred;
    inPitch = (size_t)inW;
  }
  if (!needResize) {
    if (mapIndex && barrel)
      for (int y = 0; y < outH; y++) memset(dst + (size_t)y * dpitch, 128, (size_t)outW);
    t360o_remap_u8(in, inW, inH, inPitch, dst, outW, outH, dpitch, map, interp, border);
  } else { /* ref:755-777: render at the map's size into a 0 / 128 plane, then INTER_AREA down */
    uint8_t* big = (uint8_t*)malloc((size_t)mapW * mapH);
    memset(big, mapIndex ? 128 : 0, (size_t)mapW * mapH);
    t360o_remap_u8(in, inW, inH, inPitch, big, mapW, mapH, (size_t)mapW, map, interp, border);
    t360o_resize_area_u8(big, mapW, mapH, (size_t)mapW, dst, outW, outH, dpitch);
    free(big);
  }
  free(blurred);
  return 1;
}

/* ------------------------------------------------------------------------------------------
 * Synthetic input + hashes
 * ---------------------------------------------------------------------------------------- */
static uint32_t fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}

void t360o_noise_plane(uint8_t* dst, int w, int h, size_t pitch, uint32_t plane, uint32_t frame) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      uint32_t idx = (uint32_t)x + (uint32_t)y * (uint32_t)w + plane * (uint32_t)w * (uint32_t)h + frame * 0x9E3779B9u;
      dst[(size_t)y * pitch + x] = (uint8_t)(fmix32(idx) >> 24);
    }
}

uint64_t t360o_fnv1a64(const void* p, size_t n) {
  const uint8_t* b = (const uint8_t*)p;
  uint64_t h = 0xcbf29ce484222325ull;
  for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 0x100000001b3ull; }
  return h;
}
