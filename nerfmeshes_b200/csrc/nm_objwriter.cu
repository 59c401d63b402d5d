// Host-only: the OBJ writer of export_obj (src/nerf/nerf_helpers.py:86-111) with byte-identical text.  The reference
// formats every number with python's "{}".format(float32 scalar): the value widened to double, then repr() — the
// shortest digit string that round-trips, fixed notation for 1e-4 <= |x| < 1e16, otherwise d.ddde+XX with at least two
// exponent digits.  std::to_chars yields the same shortest digits; the layout rules are re-applied here.  A million
// vertices take about a second instead of the reference's minutes of per-line python writes (SURVEY 8f rank 3).
#include <charconv>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "nm_common.h"

namespace {

char* py_repr(double x, char* out) {
  if (std::isnan(x)) { memcpy(out, "nan", 3); return out + 3; }
  if (std::isinf(x)) { if (x < 0) *out++ = '-'; memcpy(out, "inf", 3); return out + 3; }
  char buf[48];
  auto res = std::to_chars(buf, buf + sizeof(buf), x, std::chars_format::scientific);   // [-]d[.ddd]e[+-]XX, shortest
  const char* p = buf;
  if (*p == '-') { *out++ = '-'; ++p; }
  char digits[24];
  int nd = 0;
  for (; *p != 'e'; ++p)
    if (*p != '.') digits[nd++] = *p;
  ++p;                                               // 'e'
  int e = 0;
  const bool eneg = (*p == '-');
  ++p;
  for (; p < res.ptr; ++p) e = e * 10 + (*p - '0');
  if (eneg) e = -e;
  const int decpt = e + 1;                           // position of the decimal point relative to the digit string
  if (decpt <= -4 || decpt > 16) {                   // float_repr_style 'short', format code 'r'
    *out++ = digits[0];
    if (nd > 1) { *out++ = '.'; memcpy(out, digits + 1, nd - 1); out += nd - 1; }
    *out++ = 'e';
    int ex = decpt - 1;
    *out++ = ex < 0 ? '-' : '+';
    if (ex < 0) ex = -ex;
    char eb[8];
    int ne = 0;
    do { eb[ne++] = (char)('0' + ex % 10); ex /= 10; } while (ex);
    if (ne < 2) eb[ne++] = '0';
    while (ne) *out++ = eb[--ne];
    return out;
  }
  if (decpt <= 0) {
    *out++ = '0'; *out++ = '.';
    for (int i = 0; i < -decpt; ++i) *out++ = '0';
    memcpy(out, digits, nd);
    return out + nd;
  }
  if (decpt >= nd) {
    memcpy(out, digits, nd); out += nd;
    for (int i = 0; i < decpt - nd; ++i) *out++ = '0';
    *out++ = '.'; *out++ = '0';
    return out;
  }
  memcpy(out, digits, decpt); out += decpt;
  *out++ = '.';
  memcpy(out, digits + decpt, nd - decpt);
  return out + (nd - decpt);
}

char* put_int(long long v, char* out) {
  char b[24];
  int n = 0;
  if (v < 0) { *out++ = '-'; v = -v; }
  do { b[n++] = (char)('0' + v % 10); v /= 10; } while (v);
  while (n) *out++ = b[--n];
  return out;
}

// nm_export_obj's text, or with uv != nullptr its textured variant (include/nerfmeshes_b200.h): the v and vn lines are
// written by the same code in both
int write_obj(const char* path, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces, const float* diffuse,
              int64_t n_diffuse, const float* normals, int64_t n_normals, const float* uv, const char* mtl_name) {
  NM_CHECK(path && (verts || n_verts == 0) && (faces || n_faces == 0) && (normals || n_normals == 0), "null argument");
  FILE* f = fopen(path, "wb");
  NM_CHECK(f != nullptr, "cannot open '%s' for writing", path);
  std::vector<char> buf(1 << 22);
  char* p = buf.data();
  char* const lim = buf.data() + buf.size() - 512;
  bool ok = true;
  auto flush = [&]() { ok = ok && fwrite(buf.data(), 1, (size_t)(p - buf.data()), f) == (size_t)(p - buf.data()); p = buf.data(); };
  auto triple = [&](const float* a) {
    for (int c = 0; c < 3; ++c) { *p++ = ' '; p = py_repr((double)a[c], p); }
  };
  auto text = [&](const char* s) { flush(); ok = ok && fputs(s, f) >= 0; };
  if (uv) { text("mtllib "); text(mtl_name); text("\n"); }
  for (int64_t i = 0; i < n_verts; ++i) {
    *p++ = 'v';
    triple(verts + 3 * i);
    if (diffuse && i < n_diffuse) triple(diffuse + 3 * i);
    *p++ = '\n';
    if (p > lim) flush();
  }
  for (int64_t i = 0; uv && i < 3 * n_faces; ++i) {
    *p++ = 'v'; *p++ = 't';
    for (int c = 0; c < 2; ++c) { *p++ = ' '; p = py_repr((double)uv[2 * i + c], p); }
    *p++ = '\n';
    if (p > lim) flush();
  }
  for (int64_t i = 0; i < n_normals; ++i) {
    *p++ = 'v'; *p++ = 'n';
    triple(normals + 3 * i);
    *p++ = '\n';
    if (p > lim) flush();
  }
  if (uv) text("usemtl texture\n");
  for (int64_t i = 0; i < n_faces; ++i) {
    *p++ = 'f';
    for (int c = 0; c < 3; ++c) {
      const long long idx = (long long)faces[3 * i + c] + 1;
      *p++ = ' ';
      p = put_int(idx, p);
      *p++ = '/';
      if (uv) p = put_int(3 * i + c + 1, p);
      *p++ = '/';
      p = put_int(idx, p);
    }
    *p++ = '\n';
    if (p > lim) flush();
  }
  flush();
  ok = (fclose(f) == 0) && ok;
  NM_CHECK(ok, "short write to '%s'", path);
  return 0;
}

// trunc(fl32(c*255)) clamped to [0, 255], NaN to 0
uint8_t ply_colour(float c) {
  const float v = c * 255.0f;
  if (!(v > 0.f)) return 0;
  return v >= 255.f ? 255 : (uint8_t)v;
}

}  // namespace

extern "C" int nm_export_ply(const char* path, const float* points, const float* colors, const float* normals, int64_t n,
                             int binary) {
  NM_CHECK(path && n >= 0 && (n == 0 || (points && colors && normals)), "null argument or negative count");
  NM_CHECK(binary == 0 || binary == 1, "binary must be 0 or 1");
  FILE* f = fopen(path, "wb");
  NM_CHECK(f != nullptr, "cannot open '%s' for writing", path);
  bool ok = fprintf(f,
                    "ply\nformat %s 1.0\nelement vertex %lld\nproperty float x\nproperty float y\nproperty float z\n"
                    "property float nx\nproperty float ny\nproperty float nz\nproperty uchar red\nproperty uchar green\n"
                    "property uchar blue\nend_header\n",
                    binary ? "binary_little_endian" : "ascii", (long long)n) > 0;
  std::vector<char> buf(1 << 22);
  char* p = buf.data();
  char* const lim = buf.data() + buf.size() - 512;
  auto flush = [&]() { ok = ok && fwrite(buf.data(), 1, (size_t)(p - buf.data()), f) == (size_t)(p - buf.data()); p = buf.data(); };
  for (int64_t i = 0; i < n; ++i) {
    const float* src[2] = {points + 3 * i, normals + 3 * i};
    uint8_t q[3];
    for (int c = 0; c < 3; ++c) q[c] = ply_colour(colors[3 * i + c]);
    if (binary) {                                  // x86-64 and aarch64 hosts are little-endian, as the format is
      for (int k = 0; k < 2; ++k) { memcpy(p, src[k], 12); p += 12; }
      memcpy(p, q, 3); p += 3;
    } else {
      for (int k = 0; k < 2; ++k)
        for (int c = 0; c < 3; ++c) {
          p = std::to_chars(p, lim + 512, (double)src[k][c], std::chars_format::general, 18).ptr;   // printf's %.18g
          *p++ = ' ';
        }
      for (int c = 0; c < 3; ++c) { p = put_int(q[c], p); *p++ = c < 2 ? ' ' : '\n'; }
    }
    if (p > lim) flush();
  }
  flush();
  ok = (fclose(f) == 0) && ok;
  NM_CHECK(ok, "short write to '%s'", path);
  return 0;
}

extern "C" int nm_export_obj(const char* path, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces,
                             const float* diffuse, int64_t n_diffuse, const float* normals, int64_t n_normals) {
  return write_obj(path, verts, n_verts, faces, n_faces, diffuse, n_diffuse, normals, n_normals, nullptr, nullptr);
}

extern "C" int nm_export_obj_textured(const char* path, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces,
                                      const float* diffuse, int64_t n_diffuse, const float* normals, int64_t n_normals,
                                      const float* uv, const char* mtl_name) {
  NM_CHECK(uv || n_faces == 0, "null uv pointer");
  NM_CHECK(mtl_name && *mtl_name && !strpbrk(mtl_name, "\r\n"), "the material file name must be one non-empty line");
  static const float kNoUv[2] = {0.f, 0.f};            // a face-less mesh still gets its mtllib / usemtl lines
  return write_obj(path, verts, n_verts, faces, n_faces, diffuse, n_diffuse, normals, n_normals, uv ? uv : kNoUv, mtl_name);
}
