// model.cpp -- data model, file formats and small image utilities behind lib_python.
// Reference behaviour cited per function; see model.h.
#include "model.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <iostream>
#include <limits>
#include <sstream>
#include <stdexcept>
#include <sys/stat.h>
#include <zlib.h>

namespace rcvdh {
namespace fs = std::filesystem;

static bool g_logStdout = false;
void setLogToStdout(bool v) { g_logStdout = v; }
void logInfo(const std::string& s) { (g_logStdout ? std::cout : std::cerr) << s << std::endl; }
static bool fileExists(const std::string& f) { struct stat st; return stat(f.c_str(), &st) == 0; }
static void makeDirs(const std::string& dir) {   // mkdir -p
  for (size_t pos = 1; pos <= dir.size(); ++pos)
    if (pos == dir.size() || dir[pos] == '/') { const std::string sub = dir.substr(0, pos); if (!fileExists(sub)) ::mkdir(sub.c_str(), 0777); }
}
static std::string fmtInt6(int v) { char b[32]; snprintf(b, sizeof(b), "%06d", v); return b; }

// Eigen::Quaternion::_transformVector: v + 2w (q x v) + 2 q x (q x v), float arithmetic
Vec3f Quatf::rotate(const Vec3f& v) const {
  float ux = y * v.z - z * v.y, uy = z * v.x - x * v.z, uz = x * v.y - y * v.x;
  ux += ux; uy += uy; uz += uz;
  return {v.x + w * ux + (y * uz - z * uy), v.y + w * uy + (z * ux - x * uz), v.z + w * uz + (x * uy - y * ux)};
}

// --- .raw images: i32 rows, i32 cols, i32 cvType, u64 elemSize, rows*cols*elemSize bytes (lib/core/CvUtil.cpp:25-42) ---
void freadim(const std::string& fileName, Image& dst) {
  FILE* f = fopen(fileName.c_str(), "rb");
  if (!f) throw std::runtime_error("Could not open image file '" + fileName + "'.");
  int32_t hdr[3]; uint64_t es = 0;
  if (fread(hdr, 4, 3, f) != 3 || fread(&es, 8, 1, f) != 1) { fclose(f); throw std::runtime_error("Truncated raw image header."); }
  dst.create(hdr[0], hdr[1], hdr[2]);
  if (es != dst.elemSize()) { fclose(f); throw std::runtime_error("Raw image element size mismatch."); }
  const size_t n = dst.data.size();
  if (n && fread(dst.data.data(), 1, n, f) != n) { fclose(f); throw std::runtime_error("Truncated raw image data."); }
  fclose(f);
}
void fwriteim(const std::string& fileName, const Image& src) {
  FILE* f = fopen(fileName.c_str(), "wb");
  if (!f) throw std::runtime_error("Could not write image file '" + fileName + "'.");
  int32_t hdr[3] = {src.rows, src.cols, src.type}; uint64_t es = src.elemSize();
  fwrite(hdr, 4, 3, f); fwrite(&es, 8, 1, f); fwrite(src.data.data(), 1, src.data.size(), f);
  fclose(f);
}

// --- 8-bit non-interlaced PNG decoder (cv::imread(IMREAD_GRAYSCALE / IMREAD_COLOR) for the mask streams) ---
Image imreadPng(const std::string& fileName, bool grayscale) {
  std::ifstream is(fileName, std::ios::binary);
  Image out;
  if (!is) return out;
  std::vector<uint8_t> buf((std::istreambuf_iterator<char>(is)), std::istreambuf_iterator<char>());
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  if (buf.size() < 8 || memcmp(buf.data(), sig, 8)) return out;
  auto be32 = [&](size_t o) { return (uint32_t(buf[o]) << 24) | (uint32_t(buf[o + 1]) << 16) | (uint32_t(buf[o + 2]) << 8) | buf[o + 3]; };
  uint32_t w = 0, h = 0; int bitDepth = 0, colorType = 0, interlace = 0;
  std::vector<uint8_t> idat, plte;
  for (size_t o = 8; o + 12 <= buf.size();) {
    const uint32_t len = be32(o); const std::string typ(reinterpret_cast<char*>(&buf[o + 4]), 4);
    if (o + 12 + len > buf.size()) break;
    const uint8_t* d = &buf[o + 8];
    if (typ == "IHDR") { w = be32(o + 8); h = be32(o + 12); bitDepth = d[8]; colorType = d[9]; interlace = d[12]; }
    else if (typ == "PLTE") plte.assign(d, d + len);
    else if (typ == "IDAT") idat.insert(idat.end(), d, d + len);
    else if (typ == "IEND") break;
    o += 12 + len;
  }
  if (!w || !h || bitDepth != 8 || interlace) throw std::runtime_error("Unsupported PNG (need 8-bit, non-interlaced): " + fileName);
  const int ch = colorType == 0 ? 1 : colorType == 2 ? 3 : colorType == 3 ? 1 : colorType == 4 ? 2 : 4;
  const size_t stride = size_t(w) * ch;
  std::vector<uint8_t> raw((stride + 1) * h);
  uLongf rawLen = raw.size();
  if (uncompress(raw.data(), &rawLen, idat.data(), idat.size()) != Z_OK || rawLen != raw.size()) throw std::runtime_error("PNG inflate failed: " + fileName);
  std::vector<uint8_t> pix(stride * h);
  for (uint32_t y = 0; y < h; ++y) {
    const uint8_t ft = raw[y * (stride + 1)]; const uint8_t* s = &raw[y * (stride + 1) + 1];
    uint8_t* d = &pix[y * stride]; const uint8_t* up = y ? &pix[(y - 1) * stride] : nullptr;
    for (size_t i = 0; i < stride; ++i) {
      const int a = i >= size_t(ch) ? d[i - ch] : 0, b = up ? up[i] : 0, c = (up && i >= size_t(ch)) ? up[i - ch] : 0;
      int v = s[i];
      switch (ft) {
        case 1: v += a; break; case 2: v += b; break; case 3: v += (a + b) / 2; break;
        case 4: { const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c); v += (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c); break; }
        default: break;
      }
      d[i] = uint8_t(v);
    }
  }
  out.create(int(h), int(w), cvMakeType(CV_8U, grayscale ? 1 : 3));
  for (size_t i = 0; i < size_t(w) * h; ++i) {
    int r, g, b;
    const uint8_t* p = &pix[i * ch];
    if (colorType == 0 || colorType == 4) r = g = b = p[0];
    else if (colorType == 3) { r = plte[p[0] * 3]; g = plte[p[0] * 3 + 1]; b = plte[p[0] * 3 + 2]; }
    else { r = p[0]; g = p[1]; b = p[2]; }
    if (grayscale) out.data[i] = (colorType == 0 || colorType == 4) ? uint8_t(r) : uint8_t((r * 4899 + g * 9617 + b * 1868 + 8192) >> 14);
    else { out.data[i * 3] = uint8_t(b); out.data[i * 3 + 1] = uint8_t(g); out.data[i * 3 + 2] = uint8_t(r); }
  }
  return out;
}

// --- FrameRange ---
static std::vector<std::string> explode(const std::string& s, char sep) {
  std::vector<std::string> out; std::string cur; std::istringstream is(s);
  while (std::getline(is, cur, sep)) out.push_back(cur);
  return out;
}
static void trim(std::string& s) {
  const size_t a = s.find_first_not_of(" \t"), b = s.find_last_not_of(" \t");
  s = (a == std::string::npos) ? "" : s.substr(a, b - a + 1);
}
void FrameRange::fromString(const std::string& str) {
  frames.clear();
  for (const std::string& piece : explode(str, ',')) {
    std::vector<std::string> sub = explode(piece, '-');
    if (sub.size() < 1 || sub.size() > 2) throw std::runtime_error("Malformed range piece.");
    const int start = std::stoi(sub[0]); const int end = sub.size() > 1 ? std::stoi(sub[1]) : start;
    for (int f = start; f <= end; ++f) frames.insert(f);
  }
}
std::string FrameRange::toString() const {
  if (isEmpty()) return "";
  std::string res; auto it = frames.begin(); int start = *it, last = start; ++it;
  auto add = [&]() { if (!res.empty()) res += ","; res += (last == start) ? std::to_string(start) : std::to_string(start) + "-" + std::to_string(last); };
  for (; it != frames.end(); ++it) { if (*it - last > 1) { add(); start = *it; } last = *it; }
  add();
  return res;
}
void FrameRange::resolve(int numFrames, bool clip) {
  if (clip) { std::set<int> c; for (int f : frames) if (f >= 0 && f < numFrames) c.insert(f); frames = c; }
  if (frames.empty()) for (int f = 0; f < numFrames; ++f) frames.insert(f);
  if (firstFrame() < 0 || lastFrame() >= numFrames) throw std::runtime_error("Frame range contains out-of-range frame indices.");
}
void FrameRange::checkEmpty() const { if (frames.empty()) throw std::runtime_error("Frame range is empty."); }
int FrameRange::firstFrame() const { checkEmpty(); return *frames.begin(); }
int FrameRange::lastFrame() const { checkEmpty(); return *frames.rbegin(); }
bool FrameRange::isConsecutive() const { return (lastFrame() - firstFrame() + 1) == int(frames.size()); }

// --- XformDescriptor (lib/DepthMapTransform.cpp:106-265) ---
static const char* kValueStr[] = {"None", "Scale", "ScaleShift"};
static const char* kDepthStr[] = {"None", "Identity", "Global", "Grid"};
static const char* kSpatialStr[] = {"None", "Identity", "VerticalLinear", "CornersBilinear", "BilinearGrid", "BicubicGrid"};
template <class E, size_t N> static void parseEnum(E& out, const std::string& s, const char* (&tab)[N]) {
  for (size_t i = 0; i < N; ++i) if (s == tab[i]) { out = E(int(i)); return; }
  throw std::runtime_error("Invalid enum value '" + s + "'.");
}
void XformDescriptor::reset(XformType t) {
  *this = XformDescriptor();
  if (t == XformType::Spatial) { type = XformType::Spatial; depthType = DepthXformType::None; spatialType = SpatialXformType::Identity; }
}
std::string XformDescriptor::str() const {
  std::string res; char b[160];
  if (type == XformType::Depth) {
    res = std::string(kDepthStr[int(depthType)]) + "(";
    switch (depthType) {
      case DepthXformType::Identity: break;
      case DepthXformType::Global: res += kValueStr[int(valueXform)]; break;
      case DepthXformType::Grid:
        if (gridSize[2] > 1) snprintf(b, sizeof(b), "%s, %s, %d, %d, %d, %f, %f", kValueStr[int(valueXform)], cubicInterpolation ? "Cubic" : "Linear", gridSize[0], gridSize[1], gridSize[2], depthMinMax[0], depthMinMax[1]);
        else snprintf(b, sizeof(b), "%s, %s, %d, %d, %d", kValueStr[int(valueXform)], cubicInterpolation ? "Cubic" : "Linear", gridSize[0], gridSize[1], gridSize[2]);
        res += b; break;
      default: throw std::runtime_error("Invalid depth transform type.");
    }
    res += ")";
  } else {
    res = kSpatialStr[int(spatialType)];
    if (spatialType == SpatialXformType::BilinearGrid || spatialType == SpatialXformType::BicubicGrid) { snprintf(b, sizeof(b), "(%d, %d)", gridSize[0], gridSize[1]); res += b; }
  }
  return res;
}
void XformDescriptor::parse(const std::string& s) {
  depthType = DepthXformType::None; spatialType = SpatialXformType::None;
  const size_t pos = s.find('(');
  const std::string typeStr = s.substr(0, pos);
  std::vector<std::string> args;
  auto getArgs = [&]() {
    if (pos == std::string::npos || s.empty() || s.back() != ')') throw std::runtime_error("Malformed descriptor string.");
    args = explode(s.substr(pos + 1, s.size() - 1 - (pos + 1)), ',');
    for (auto& a : args) trim(a);
  };
  auto checkNum = [&](size_t n) { if (args.size() != n) throw std::runtime_error("Incorrect number of parameters."); };
  if (type == XformType::Depth) {
    getArgs();
    if (typeStr == "BicubicGrid" || typeStr == "BilinearGrid") {   // backwards-compatibility form (:198-206)
      if (args.size() < 3) throw std::runtime_error("Incorrect number of parameters.");
      args = {args[0], typeStr == "BicubicGrid" ? "Cubic" : "Linear", args[1], args[2], "1"};
      depthType = DepthXformType::Grid;
    } else parseEnum(depthType, typeStr, kDepthStr);
    switch (depthType) {
      case DepthXformType::Identity: checkNum(0); break;
      case DepthXformType::Global: checkNum(1); parseEnum(valueXform, args[0], kValueStr); break;
      case DepthXformType::Grid:
        if (args.size() < 5) throw std::runtime_error("Incorrect number of parameters.");
        parseEnum(valueXform, args[0], kValueStr);
        if (args[1] == "Cubic") cubicInterpolation = true; else if (args[1] == "Linear") cubicInterpolation = false; else throw std::runtime_error("Invalid interpolation mode.");
        gridSize[0] = std::stoi(args[2]); gridSize[1] = std::stoi(args[3]); gridSize[2] = std::stoi(args[4]);
        if (gridSize[2] <= 1) checkNum(5); else { checkNum(7); depthMinMax[0] = std::stof(args[5]); depthMinMax[1] = std::stof(args[6]); }
        break;
      default: throw std::runtime_error("Invalid depth transform type.");
    }
  } else {
    parseEnum(spatialType, typeStr, kSpatialStr);
    if (spatialType == SpatialXformType::BilinearGrid || spatialType == SpatialXformType::BicubicGrid) { getArgs(); checkNum(2); gridSize[0] = std::stoi(args[0]); gridSize[1] = std::stoi(args[1]); }
  }
}

// --- Xform ---
void fillDepthConfig(const XformDescriptor& d, rcvd_config& cfg) {
  cfg.depth_type = int(d.depthType); cfg.value_xform = int(d.valueXform); cfg.depth_cubic = d.cubicInterpolation ? 1 : 0;
  cfg.depth_grid_x = d.gridSize[0]; cfg.depth_grid_y = d.gridSize[1];
}
void fillSpatialConfig(const XformDescriptor& d, rcvd_config& cfg) {
  cfg.spatial_type = int(d.spatialType); cfg.spatial_grid_x = d.gridSize[0]; cfg.spatial_grid_y = d.gridSize[1];
}
Xform::Xform(const XformDescriptor& desc) : desc_(desc) {
  if (desc.type == XformType::Depth) {
    const int k = valueParams();
    switch (desc.depthType) {
      case DepthXformType::Identity: break;
      case DepthXformType::Global: params_.assign(k, 1.0); break;   // lib/DepthMapTransform.cpp:531
      case DepthXformType::Grid: {
        const auto& g = desc.gridSize;
        if ((g[0] > 1 || g[1] > 1) && (g[0] < 2 || g[1] < 2)) throw std::runtime_error("Spatial grid transforms must have at least two rows and columns, respectively.");
        const int n = k * g[0] * g[1] * g[2];
        if (n <= 1) throw std::runtime_error("Grid transform cannot have an empty grid.");
        if (g[2] > 1) throw std::runtime_error("Bilateral (depth-wise) grids are not supported in this build.");
        params_.assign(n, 1.0); break; }   // :707
      default: throw std::runtime_error("Invalid depth transform type.");
    }
  } else {
    switch (desc.spatialType) {
      case SpatialXformType::Identity: break;
      case SpatialXformType::VerticalLinear: params_.assign(4, 0.0); break;
      case SpatialXformType::CornersBilinear: params_.assign(8, 0.0); break;
      case SpatialXformType::BilinearGrid: case SpatialXformType::BicubicGrid:
        if (desc.gridSize[0] < 2 || desc.gridSize[1] < 2) throw std::logic_error("Need at least two rows and columns in depth transform grid.");
        params_.assign(size_t(desc.gridSize[0]) * desc.gridSize[1] * 2, 0.0); break;
      default: throw std::runtime_error("Invalid spatial transform type.");
    }
  }
}
std::unique_ptr<Xform> Xform::clone() const { auto r = std::make_unique<Xform>(desc_); r->params_ = params_; return r; }
void Xform::copyFrom(const Xform& o) { if (o.desc_ != desc_) throw std::runtime_error("Can only copy parameters from same type of transform."); params_ = o.params_; }
std::string Xform::str() const {
  std::string res = desc_.str() + " ["; char b[64];
  for (size_t i = 0; i < params_.size(); ++i) { snprintf(b, sizeof(b), "%s%.2f", i ? ", " : "", params_[i]); res += b; }
  return res + "]";
}
void denseConfig(const XformDescriptor& d, rcvd_config& cfg) {
  memset(&cfg, 0, sizeof(cfg)); cfg.num_frames = 1; cfg.depth_type = RCVD_DEPTH_IDENTITY; cfg.value_xform = RCVD_VALUE_SCALE; cfg.spatial_type = RCVD_SPATIAL_IDENTITY;
  if (d.type == XformType::Depth) fillDepthConfig(d, cfg); else fillSpatialConfig(d, cfg);
  if (cfg.value_xform == RCVD_VALUE_NONE) cfg.value_xform = RCVD_VALUE_SCALE;
}
Image Xform::paramMap(const DepthFrame& df) const {
  if (desc_.type != XformType::Depth || desc_.depthType != DepthXformType::Grid) throw std::runtime_error("Parameter map not implemented for this transform type.");
  rcvd_config cfg; denseConfig(desc_, cfg);
  const int w = df.width(), h = df.height();
  Image out; out.create(h, w, cvMakeType(CV_64F, valueParams()));
  if (rcvd_depth_param_map(&cfg, currentDevice(), params_.data(), out.ptr<double>(), h, w) != RCVD_OK) throw std::runtime_error(rcvd_last_error());
  return out;
}
Image Xform::warp(int h, int w) const {
  if (desc_.type != XformType::Spatial) throw std::runtime_error("Transform has the wrong type.");
  rcvd_config cfg; denseConfig(desc_, cfg);
  Image out; out.create(h, w, cvMakeType(CV_32F, 2));
  if (rcvd_spatial_warp(&cfg, currentDevice(), params_.data(), out.ptr<float>(), h, w) != RCVD_OK) throw std::runtime_error(rcvd_last_error());
  return out;
}
Image Xform::apply(const Image& src) const {
  rcvd_config cfg; denseConfig(desc_, cfg);
  Image out; out.create(src.rows, src.cols, cvMakeType(CV_32F, 1));
  if (rcvd_depth_apply(&cfg, currentDevice(), params_.data(), src.ptr<float>(), out.ptr<float>(), src.rows, src.cols) != RCVD_OK) throw std::runtime_error(rcvd_last_error());
  return out;
}

// The reference starts the maximum at numeric_limits<float>::min(), the smallest positive normal float, so a range without a valid
// depth is (FLT_MAX, FLT_MIN) and a maximum below FLT_MIN (a subnormal depth) reads as FLT_MIN; both kept.
std::pair<float, float> computeDepthRange(const float* depth, size_t count) {
  float lo = std::numeric_limits<float>::max(), hi = std::numeric_limits<float>::min();
  for (size_t i = 0; i < count; ++i) {
    const float d = depth[i];
    if (std::isfinite(d) && d > 0) { lo = std::min(d, lo); hi = std::max(d, hi); }
  }
  return {lo, hi};
}

// --- Intrinsics::resolveMissingFov (lib/DepthPhoto.cpp:114-158) ---
void Intrinsics::resolveMissingFov(float aspect) {
  bool vSet = vFov > 0, hSet = hFov > 0;
  if (vSet && hSet) return;
  if (aspect == 0) throw std::runtime_error("Aspect ratio must be non-zero.");
  const float kDefaultHFov = 0.508015513f, kDefaultVFov = 0.666488587f;
  const float defaultAspect = tanf(kDefaultHFov / 2.f) / tanf(kDefaultVFov / 2.f);
  if (!vSet && !hSet) { if (aspect > defaultAspect) { vFov = kDefaultVFov; vSet = true; } else { hFov = kDefaultHFov; hSet = true; } }
  if (vSet) { const float hh = std::tan(vFov / 2.0f); hFov = std::atan(hh * aspect) * 2.0f; }
  else if (hSet) { const float hw = std::tan(hFov / 2.0f); vFov = std::atan(hw / aspect) * 2.0f; }
}

// --- Extrinsics::worldToCamera / fromWorldToCamera (lib/DepthPhoto.cpp:63-99), row-major 4x4 ---
// rotate * translate: the rows of rotate are the camera's right, up and backward vectors (orientation times the unit axes), and
// translate moves the position to the origin, so the last column is rotate times -position.
std::array<float, 16> Extrinsics::worldToCamera() const {
  const Vec3f rows[3] = {right(), up(), backward()};
  std::array<float, 16> M{};
  for (int i = 0; i < 3; ++i) {
    const Vec3f& r = rows[i];
    M[4 * i] = r.x; M[4 * i + 1] = r.y; M[4 * i + 2] = r.z;
    M[4 * i + 3] = r.x * -position.x + r.y * -position.y + r.z * -position.z;
  }
  M[15] = 1.f;
  return M;
}
// The upper 3x3 block R is taken as the rotation; the position is -(Rᵀ t) for the last column t, the orientation Quaternionf(Rᵀ).
Extrinsics Extrinsics::fromWorldToCamera(const std::array<float, 16>& W) {
  float Rt[3][3], q[4];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rt[i][j] = W[4 * j + i];
  Extrinsics e;
  e.position = {-(Rt[0][0] * W[3] + Rt[0][1] * W[7] + Rt[0][2] * W[11]), -(Rt[1][0] * W[3] + Rt[1][1] * W[7] + Rt[1][2] * W[11]),
                -(Rt[2][0] * W[3] + Rt[2][1] * W[7] + Rt[2][2] * W[11])};
  matrixToQuat(Rt, q);
  e.orientation.x = q[0]; e.orientation.y = q[1]; e.orientation.z = q[2]; e.orientation.w = q[3];
  return e;
}

// --- streams / frames ---
const Image* ColorFrame::image() {
  if (!loaded_) {
    loaded_ = true;
    const std::string fn = stream_.path() + "/frame_" + fmtInt6(index_) + stream_.extension();
    if (fileExists(fn)) {
      img_ = std::make_unique<Image>();
      if (stream_.extension() == ".raw") freadim(fn, *img_);
      else {
        Image u8 = imreadPng(fn, cvChannels(stream_.type()) == 1);
        if (u8.empty()) throw std::runtime_error("Could not read image '" + fn + "'.");
        if (cvDepth(stream_.type()) == CV_32F) {   // byte -> float: convertTo(.., 1/256) (lib/ColorStream.cpp:121-129)
          img_->create(u8.rows, u8.cols, stream_.type());
          float* d = img_->ptr<float>(); for (size_t i = 0; i < u8.data.size(); ++i) d[i] = u8.data[i] * (1.f / 256.f);
        } else *img_ = std::move(u8);
      }
      if (img_->type != stream_.type()) throw std::runtime_error("Image has incorrect type.");
      if (stream_.width_ < 0) { stream_.width_ = img_->cols; stream_.height_ = img_->rows; }
    }
  }
  return img_.get();
}
ColorFrame& ColorStream::frame(int i) { if (i < 0 || i >= int(frames_.size())) throw std::runtime_error("Frame index out of range."); return *frames_[i]; }
void ColorStream::setDir(const std::string& dir) { dir_ = dir; path_ = video_.path() + "/" + dir_; }
int ColorStream::width() { if (width_ < 0) { for (auto& f : frames_) if (f->image()) break; if (width_ < 0) width_ = height_ = 0; } return width_; }
int ColorStream::height() { width(); return height_; }

DepthFrame::DepthFrame(DepthVideo& v, DepthStream& s, int index) : video_(v), stream_(s), index_(index) { resetDepthXform(); resetSpatialXform(); }
void DepthFrame::resetDepthXform() { depthXform_ = std::make_unique<Xform>(stream_.depthXformDesc()); xformed_.reset(); }
void DepthFrame::resetSpatialXform() { spatialXform_ = std::make_unique<Xform>(stream_.spatialXformDesc()); }
int DepthFrame::width() const { return stream_.width(); }
int DepthFrame::height() const { return stream_.height(); }
float DepthFrame::invAspect() const { return video_.invAspect(); }
const Image* DepthFrame::sourceDepth() {
  if (!sourceLoaded_) {
    sourceLoaded_ = true;
    const std::string fn = stream_.path() + "/depth/frame_" + fmtInt6(index_) + ".raw";
    if (fileExists(fn)) {
      source_ = std::make_unique<Image>();
      freadim(fn, *source_);
      if (source_->type != cvMakeType(CV_32F, 1)) throw std::runtime_error("Depth image has incorrect type.");
      float* d = source_->ptr<float>();
      for (size_t i = 0; i < size_t(source_->rows) * source_->cols; ++i) d[i] = (std::isfinite(d[i]) && d[i] > 0.f) ? 1.f / d[i] : 0.f;   // lib/DepthStream.cpp:200-211
      if (stream_.width_ < 0) { stream_.width_ = source_->cols; stream_.height_ = source_->rows; }
      else if (stream_.width_ != source_->cols || stream_.height_ != source_->rows) throw std::runtime_error("Depth frame has inconsistent dimensions.");
    }
  }
  return (source_ && !source_->empty()) ? source_.get() : nullptr;
}
const Image* DepthFrame::depth() {
  // lib/DepthStream.cpp:275-291: the transformed depth is re-applied whenever the transform's descriptor or parameters differ from the
  // ones it was computed with (Python mutates transforms in place, e.g. depthXform().copyFrom(...), after depth() has been called)
  const Image* s = sourceDepth();
  if (!s) return nullptr;
  if (!xformed_ || depthXform_->desc() != appliedDesc_ || depthXform_->params() != appliedParams_) {
    appliedDesc_ = depthXform_->desc(); appliedParams_ = depthXform_->params();
    xformed_ = std::make_unique<Image>(depthXform_->apply(*s));
  }
  return xformed_.get();
}
void DepthFrame::setDepth(const Image& depth) {
  if (depth.type != cvMakeType(CV_32F, 1)) throw std::runtime_error("Depth image has incorrect type.");
  if (stream_.width_ < 0) { stream_.width_ = depth.cols; stream_.height_ = depth.rows; }
  else if (stream_.width_ != depth.cols || stream_.height_ != depth.rows) throw std::runtime_error("Depth frame has inconsistent dimensions.");
  source_ = std::make_unique<Image>(depth); sourceLoaded_ = true; clearXformedCache(); medianValid_ = false;
}
const Image* DepthFrame::warp() {
  if (!warp_ || spatialXform_->desc() != warpDesc_ || spatialXform_->params() != warpParams_) {
    const int h = stream_.height(), w = stream_.width();
    if (h <= 0 || w <= 0) throw std::runtime_error("Depth stream '" + stream_.name() + "' has no known size: it has neither depth files nor a size given at creation.");
    warp_ = std::make_unique<Image>(spatialXform_->warp(h, w));
    warpDesc_ = spatialXform_->desc(); warpParams_ = spatialXform_->params();
  }
  return warp_.get();
}
float DepthFrame::sourceDepthMedian() {
  if (!medianValid_) {
    const Image* d = sourceDepth();
    if (!d) throw std::runtime_error("Missing depth image.");
    std::vector<float> s(d->ptr<float>(), d->ptr<float>() + size_t(d->rows) * d->cols);
    std::nth_element(s.begin(), s.begin() + s.size() / 2, s.end());
    median_ = s[s.size() / 2]; medianValid_ = true;
  }
  return median_;
}
void DepthFrame::clear() { clearCache(); intrinsics = Intrinsics(); extrinsics = Extrinsics(); }
DepthFrame& DepthStream::frame(int i) { if (i < 0 || i >= int(frames_.size())) throw std::runtime_error("Frame index out of range."); return *frames_[i]; }
void DepthStream::setDir(const std::string& dir) { dir_ = dir; path_ = video_.path() + "/" + dir_; }
int DepthStream::width() { if (width_ < 0) { for (auto& f : frames_) if (f->sourceDepth()) break; if (width_ < 0) width_ = height_ = 0; } return width_; }
int DepthStream::height() { width(); return height_; }
void DepthStream::preloadSourceDepth(const std::vector<int>& frames, bool medians) {
  if (frames.empty()) return;
  auto one = [&](size_t i) { DepthFrame& f = frame(frames[i]); if (f.sourceDepth() && medians) f.sourceDepthMedian(); };
  one(0);
  parallelFor(frames.size() - 1, [&](size_t i) { one(i + 1); });
}
void DepthStream::resetDepthXforms(const XformDescriptor& desc) { depthXformDesc_ = desc; for (auto& f : frames_) f->resetDepthXform(); }
void DepthStream::resetSpatialXforms(const XformDescriptor& desc) { spatialXformDesc_ = desc; for (auto& f : frames_) f->resetSpatialXform(); }

// --- DepthVideo ---
void DepthVideo::init(const std::string& path, int width, int height, const std::vector<float>& pts) {
  colorStreams_.clear(); depthStreams_.clear();
  path_ = path; pts_ = pts; width_ = width; height_ = height;
  aspect_ = width / float(height); invAspect_ = 1.f / aspect_;
  duration_ = pts_.empty() ? 0.f : pts_.back() * pts_.size() / float(pts_.size() - 1);
}
void DepthVideo::reset() {   // the width and height stay, as in the reference
  path_.clear(); pts_.clear(); colorStreams_.clear(); depthStreams_.clear();
  duration_ = 0.f; aspect_ = 0.f; invAspect_ = 0.f;
}
int DepthVideo::timeToFrame(float time) const {
  if (pts_.empty()) throw std::runtime_error("Video has no frames.");
  if (time < pts_[0]) throw std::runtime_error("Query time before first frame's time.");
  if (time > duration_) throw std::runtime_error("Query time after video duration.");
  for (size_t i = 0; i + 1 < pts_.size(); ++i) if (time >= pts_[i] && time < pts_[i + 1]) return int(i);
  return numFrames() - 1;
}
bool DepthVideo::hasColorStream(const std::string& n) const { for (auto& s : colorStreams_) if (s->name_ == n) return true; return false; }
int DepthVideo::colorStreamIndex(const std::string& n) const { for (size_t i = 0; i < colorStreams_.size(); ++i) if (colorStreams_[i]->name_ == n) return int(i); throw std::runtime_error("Color stream '" + n + "' not found."); }
ColorStream& DepthVideo::colorStream(int i) { if (i < 0 || i >= numColorStreams()) throw std::runtime_error("Color stream index out of range."); return *colorStreams_[i]; }
void DepthVideo::createColorStream(const std::string& name, const std::string& dir, const std::string& ext, int type, std::pair<int, int> size) {
  if (type != cvMakeType(CV_8U, 1) && type != cvMakeType(CV_8U, 3) && type != cvMakeType(CV_32F, 1) && type != cvMakeType(CV_32F, 3))
    throw std::runtime_error("Color streams only support 1 or 3 channels and byte or float depth.");
  colorStreams_.push_back(std::make_unique<ColorStream>(*this));
  ColorStream& cs = *colorStreams_.back();
  cs.name_ = name; cs.setDir(dir); cs.extension_ = ext; cs.type_ = type; cs.width_ = size.first; cs.height_ = size.second;
  for (int f = 0; f < numFrames(); ++f) cs.frames_.push_back(std::make_unique<ColorFrame>(cs, f));
}
bool DepthVideo::hasDepthStream(const std::string& n) const { for (auto& s : depthStreams_) if (s->name_ == n) return true; return false; }
int DepthVideo::depthStreamIndex(const std::string& n) const { for (size_t i = 0; i < depthStreams_.size(); ++i) if (depthStreams_[i]->name_ == n) return int(i); throw std::runtime_error("Depth stream '" + n + "' not found."); }
DepthStream& DepthVideo::depthStream(int i) { if (i < 0 || i >= numDepthStreams()) throw std::runtime_error("Depth stream index out of range."); return *depthStreams_[i]; }
void DepthVideo::createDepthStream(const std::string& name, const std::string& dir, std::pair<int, int> size) {
  depthStreams_.push_back(std::make_unique<DepthStream>(*this));
  DepthStream& ds = *depthStreams_.back();
  ds.name_ = name; ds.setDir(dir); ds.depthXformDesc_.reset(); ds.spatialXformDesc_.reset(XformType::Spatial); ds.width_ = size.first; ds.height_ = size.second;
  for (int f = 0; f < numFrames(); ++f) { ds.frames_.push_back(std::make_unique<DepthFrame>(*this, ds, f)); ds.frames_.back()->intrinsics.resolveMissingFov(aspect_); }
}
void DepthVideo::printInfo() const {
  logInfo("Path: " + path_);
  char b[256]; snprintf(b, sizeof(b), "Dimensions: %d x %d (%f aspect ratio)", width_, height_, aspect_); logInfo(b);
  snprintf(b, sizeof(b), "Frame count: %d (%.2fs duration)", numFrames(), duration_); logInfo(b);
  logInfo("Color streams: " + std::to_string(numColorStreams()));
  for (auto& s : colorStreams_) logInfo("  '" + s->name_ + "' (dir '" + s->dir_ + "', extension '" + s->extension_ + "')");
  logInfo("Depth streams: " + std::to_string(numDepthStreams()));
  for (auto& s : depthStreams_) logInfo("  '" + s->name_ + "' (dir '" + s->dir_ + "', depth xform " + s->depthXformDesc_.str() + ", spatial xform " + s->spatialXformDesc_.str() + ")");
}
// video.dat, byte-compatible with the reference writer (lib/DepthVideo.cpp:300-385).
template <class T> static void wr(std::ostream& os, const T& v) { os.write(reinterpret_cast<const char*>(&v), sizeof(T)); }
static void wrstr(std::ostream& os, const std::string& s) { wr<uint64_t>(os, s.size()); os.write(s.data(), s.size()); }
static void wrXformDesc(std::ostream& os, const XformDescriptor& d) { wr<int32_t>(os, int32_t(d.type)); wrstr(os, d.str()); }
void DepthVideo::save() {
  std::ofstream os(path_ + "/video.dat", std::ios::binary);
  if (!os) throw std::runtime_error("Could not write video.dat.");
  wr<uint32_t>(os, 0xDEADBEEF); wr<uint32_t>(os, 13); wr<uint32_t>(os, 3);
  wr<int32_t>(os, numFrames()); for (float p : pts_) wr<float>(os, p);
  wr<int32_t>(os, numColorStreams());
  for (auto& cs : colorStreams_) { wrstr(os, cs->name_); wrstr(os, cs->dir_); wrstr(os, cs->extension_); wr<int32_t>(os, cs->type_); wr<int32_t>(os, cs->width_); wr<int32_t>(os, cs->height_); wr<bool>(os, false); }
  wr<int32_t>(os, numDepthStreams());
  for (auto& ds : depthStreams_) {
    wrstr(os, ds->name_); wrstr(os, ds->dir_); wrXformDesc(os, ds->depthXformDesc_); wrXformDesc(os, ds->spatialXformDesc_);
    wr<int32_t>(os, ds->width_); wr<int32_t>(os, ds->height_); wr<bool>(os, false);
    for (auto& f : ds->frames_) {
      wr<int32_t>(os, 0 /* Projection::Perspective */); wr<float>(os, f->intrinsics.vFov); wr<float>(os, f->intrinsics.hFov); wr<float>(os, f->intrinsics.centerLat); wr<float>(os, f->intrinsics.centerLon);
      wr<float>(os, f->extrinsics.position.x); wr<float>(os, f->extrinsics.position.y); wr<float>(os, f->extrinsics.position.z);
      wr<float>(os, f->extrinsics.orientation.x); wr<float>(os, f->extrinsics.orientation.y); wr<float>(os, f->extrinsics.orientation.z); wr<float>(os, f->extrinsics.orientation.w);
      wr<bool>(os, f->enabled);
      for (const Xform* x : {&f->depthXform(), &f->spatialXform()}) { wrXformDesc(os, x->desc()); os.write(reinterpret_cast<const char*>(x->params().data()), sizeof(double) * x->params().size()); }
    }
  }
  wr<float>(os, duration_); wr<int32_t>(os, width_); wr<int32_t>(os, height_); wr<float>(os, aspect_); wr<float>(os, invAspect_);
  wr<uint32_t>(os, 0xDEADBEEF);
}
// Reader for the file save() writes.  Note: the reference's own load() (lib/DepthVideo.cpp:120-298) does not consume the
// per-stream "has GOP table" byte that its save() emits (:329-332, :355-359 vs the commented-out reads at :191-197, :236-245),
// so it cannot re-read format-13 files; this reader follows the WRITER's layout.
template <class T> static T rd(std::istream& is) { T v{}; is.read(reinterpret_cast<char*>(&v), sizeof(T)); if (!is) throw std::runtime_error("Unexpected end of 'video.dat'."); return v; }
static std::string rdstr(std::istream& is) { const uint64_t n = rd<uint64_t>(is); if (n > (1u << 20)) throw std::runtime_error("Corrupt string in 'video.dat'."); std::string s(n, '\0'); is.read(s.data(), n); if (!is) throw std::runtime_error("Unexpected end of 'video.dat'."); return s; }
static XformDescriptor rdXformDesc(std::istream& is) { XformDescriptor d; d.type = XformType(rd<int32_t>(is)); const std::string str = rdstr(is); const XformType t = d.type; d.parse(str); d.type = t; return d; }
void DepthVideo::load(const std::string& path) {
  std::ifstream is(path + "/video.dat", std::ios::binary);
  if (!is) throw std::runtime_error("Could not find 'video.dat'.");
  if (rd<uint32_t>(is) != 0xDEADBEEF) throw std::runtime_error("Did not see magic marker at beginning of file.");
  const uint32_t fileFormat = rd<uint32_t>(is), dpFormat = rd<uint32_t>(is);
  if (fileFormat > 13) throw std::runtime_error("File format too new.");
  if (fileFormat < 13 || dpFormat != 3) throw std::runtime_error("File format too old.");   // only the current writer's format is supported here
  colorStreams_.clear(); depthStreams_.clear(); path_ = path;
  const int n = rd<int32_t>(is); if (n < 0 || n > (1 << 24)) throw std::runtime_error("Corrupt frame count in 'video.dat'.");
  pts_.resize(n); for (float& p : pts_) p = rd<float>(is);
  const int ncs = rd<int32_t>(is);
  for (int i = 0; i < ncs; ++i) {
    colorStreams_.push_back(std::make_unique<ColorStream>(*this));
    ColorStream& cs = *colorStreams_.back();
    cs.name_ = rdstr(is); cs.setDir(rdstr(is)); cs.extension_ = rdstr(is); cs.type_ = rd<int32_t>(is); cs.width_ = rd<int32_t>(is); cs.height_ = rd<int32_t>(is);
    if (rd<bool>(is)) throw std::runtime_error("GOP tables are not supported.");
    for (int f = 0; f < n; ++f) cs.frames_.push_back(std::make_unique<ColorFrame>(cs, f));
  }
  const int nds = rd<int32_t>(is);
  for (int i = 0; i < nds; ++i) {
    depthStreams_.push_back(std::make_unique<DepthStream>(*this));
    DepthStream& ds = *depthStreams_.back();
    ds.name_ = rdstr(is); ds.setDir(rdstr(is)); ds.depthXformDesc_ = rdXformDesc(is); ds.spatialXformDesc_ = rdXformDesc(is);
    ds.width_ = rd<int32_t>(is); ds.height_ = rd<int32_t>(is);
    if (rd<bool>(is)) throw std::runtime_error("GOP tables are not supported.");
    for (int f = 0; f < n; ++f) {
      ds.frames_.push_back(std::make_unique<DepthFrame>(*this, ds, f));
      DepthFrame& df = *ds.frames_.back();
      if (rd<int32_t>(is) != 0) throw std::runtime_error("Only perspective intrinsics are supported.");
      df.intrinsics.vFov = rd<float>(is); df.intrinsics.hFov = rd<float>(is); df.intrinsics.centerLat = rd<float>(is); df.intrinsics.centerLon = rd<float>(is);
      df.extrinsics.position.x = rd<float>(is); df.extrinsics.position.y = rd<float>(is); df.extrinsics.position.z = rd<float>(is);
      df.extrinsics.orientation.x = rd<float>(is); df.extrinsics.orientation.y = rd<float>(is); df.extrinsics.orientation.z = rd<float>(is); df.extrinsics.orientation.w = rd<float>(is);
      df.enabled = rd<bool>(is);
      for (int k = 0; k < 2; ++k) {
        const XformDescriptor d = rdXformDesc(is);
        if (k == 0 && d != ds.depthXformDesc_) throw std::runtime_error("Inconsistent depth transform.");
        Xform& x = k == 0 ? df.depthXform() : df.spatialXform();
        if (d != x.desc()) throw std::runtime_error("Inconsistent spatial transform.");
        is.read(reinterpret_cast<char*>(x.params().data()), sizeof(double) * x.params().size());
        if (!is) throw std::runtime_error("Unexpected end of 'video.dat'.");
      }
    }
  }
  duration_ = rd<float>(is); width_ = rd<int32_t>(is); height_ = rd<int32_t>(is); aspect_ = rd<float>(is); invAspect_ = rd<float>(is);
  if (rd<uint32_t>(is) != 0xDEADBEEF) throw std::runtime_error("Did not see magic marker at end of file.");
}
void DepthVideo::saveDepth(int stream) {
  DepthStream& ds = depthStream(stream);
  for (int f = 0; f < numFrames(); ++f) {
    const std::string fn = ds.path() + "/depth/frame_" + fmtInt6(f) + ".raw";
    const Image* d = ds.frame(f).depth();
    if (d) {
      Image disp; disp.create(d->rows, d->cols, cvMakeType(CV_32F, 1));
      const float* s = d->ptr<float>(); float* o = disp.ptr<float>();
      for (size_t i = 0; i < size_t(d->rows) * d->cols; ++i) o[i] = (std::isfinite(s[i]) && s[i] > 0.f) ? 1.f / s[i] : 0.f;   // invalid depth -> 0 (:611-618)
      makeDirs(ds.path() + "/depth");
      fwriteim(fn, disp);
    } else if (fileExists(fn)) {
      std::remove(fn.c_str());
    }
  }
}
// Entries of a directory sorted by name: std::filesystem (like boost::filesystem in the reference) iterates in no specified order.
static std::vector<fs::directory_entry> sortedEntries(const std::string& dir) {
  std::vector<fs::directory_entry> v{fs::directory_iterator(dir), fs::directory_iterator()};
  std::sort(v.begin(), v.end(), [](const fs::directory_entry& a, const fs::directory_entry& b) { return a.path().filename() < b.path().filename(); });
  return v;
}

void importVideo(DepthVideo& video, const std::string& path, bool discoverStreams) {
  logInfo("Importing 3D video '" + path + "'...");
  std::ifstream is(path + "/frames.txt", std::ios::binary);
  if (is.fail()) throw std::runtime_error("Could not open frame file.");
  int n = -1, w = -1, h = -1; is >> n >> w >> h;
  if (n <= 0) throw std::runtime_error("Invalid frame file.");
  std::vector<float> pts(n); float minPts = 0.f;
  for (int i = 0; i < n; ++i) {
    float p; is >> p; if (i == 0) minPts = p; p -= minPts;
    if (i > 0 && p <= pts[i - 1]) throw std::runtime_error("Non-monotonic PTS detected.");
    pts[i] = p;
  }
  video.init(path, w, h, pts);
  if (!discoverStreams) return;

  // Stream discovery (:39-195), in the reference's order.  Fixed colour streams first: directory, stream name, extension, type.
  logInfo("  Discovering color streams...");
  struct FixedStream { const char *dir, *name, *ext; int type; };
  static const FixedStream kFixed[] = {{"color_full", "full", ".png", cvMakeType(CV_32F, 3)}, {"color_down", "down", ".raw", cvMakeType(CV_32F, 3)},
                                       {"color_down_png", "down_png", ".png", cvMakeType(CV_32F, 3)}, {"dynamic_mask", "dynamic_mask", ".png", cvMakeType(CV_8U, 1)}};
  for (const FixedStream& c : kFixed)
    if (fs::is_directory(path + "/" + c.dir)) { logInfo(std::string("    Found color stream '") + c.dir + "'."); video.createColorStream(c.name, c.dir, c.ext, c.type, {-1, -1}); }
  // Then every other subdirectory with a stream_info.txt of type "color".  Like the reference, a directory is skipped when its name
  // equals a fixed stream's name (not its directory).  Sorted by name, which is the reference's full-path order.
  for (const fs::directory_entry& e : sortedEntries(path)) {
    if (!e.is_directory()) continue;
    const std::string rel = fs::relative(e.path(), path).string();
    if (std::any_of(std::begin(kFixed), std::end(kFixed), [&](const FixedStream& c) { return rel == c.name; })) continue;
    const std::string infoFile = e.path().string() + "/stream_info.txt";
    if (!fs::exists(infoFile)) continue;
    std::ifstream info(infoFile, std::ios::binary);
    if (info.fail()) throw std::runtime_error("Could not open frame file.");   // the reference's message
    std::string type, ext, format; info >> type;
    if (type != "color") continue;
    info >> ext >> format;
    int cvType;
    if (format == "32FC3") cvType = cvMakeType(CV_32F, 3);
    else if (format == "8UC1") cvType = cvMakeType(CV_8U, 1);
    else throw std::runtime_error("Invalid format string.");
    logInfo("    Found color stream '" + rel + "' (" + ext + ", " + format + ").");
    video.createColorStream(rel, rel, ext, cvType, {-1, -1});
  }
  // Depth streams: every directory below the video with a depth/ subdirectory (not descended into), in sorted relative-path order.
  logInfo("  Discovering depth streams...");
  std::vector<std::string> depthStreams;
  std::function<void(const std::string&)> visit = [&](const std::string& dir) {
    for (const fs::directory_entry& e : sortedEntries(dir)) {
      if (!e.is_directory()) continue;
      if (fs::is_directory(e.path() / "depth")) depthStreams.push_back(fs::relative(e.path(), path).string());
      else visit(e.path().string());
    }
  };
  visit(path);
  std::sort(depthStreams.begin(), depthStreams.end());
  for (const std::string& s : depthStreams) {
    logInfo("    Found depth stream '" + s + "'.");
    if (s == "depth_colmap_dense") {   // COLMAP's depth is scaled into depth_colmap_dense_imported, which the stream then reads
      importColmapDepth(video);
      video.createDepthStream(s, "depth_colmap_dense_imported", {-1, -1});
    } else if (s != "depth_colmap_dense_imported") {
      video.createDepthStream(s, s, {-1, -1});
      const std::string posesFile = path + "/" + s + "/poses.txt";
      if (fs::exists(posesFile)) importPoses(video, posesFile, video.numDepthStreams() - 1);
    }
  }
  // The first COLMAP reconstruction found sets the cameras of every depth stream.
  for (const std::string& npz : {path + "/metadata.npz", path + "/colmap_dense/metadata.npz"}) {
    if (!fs::is_regular_file(npz)) continue;
    logInfo("  Importing COLMAP reconstruction from '" + npz + "'...");
    for (int s = 0; s < video.numDepthStreams(); ++s) importColmapRecon(video, npz, s, false);
    break;
  }
  const std::string trackFile = path + "/track2d.csv";
  if (fs::is_regular_file(trackFile)) {
    logInfo("  Importing tracks from '" + trackFile + "'...");
    importTracks(video, trackFile);
  }
}

void importPoses(DepthVideo& video, const std::string& posesFile, int stream) {
  logInfo("Importing poses from '" + posesFile + "' to stream " + std::to_string(stream) + ".");
  DepthStream& ds = video.depthStream(stream);
  std::ifstream is(posesFile, std::ios::binary);
  if (is.fail()) throw std::runtime_error("Could not open poses file.");
  int n = -1; is >> n;
  if (n > video.numFrames()) throw std::runtime_error("Poses file has more frames than the video.");
  for (int i = 0; i < n; ++i) {   // position x y z, quaternion x y z w, hFov, vFov
    float v[9] = {};
    for (float& x : v) is >> x;
    DepthFrame& f = ds.frame(i);
    f.enabled = true;
    f.extrinsics.position = {v[0], v[1], v[2]};
    f.extrinsics.orientation.x = v[3]; f.extrinsics.orientation.y = v[4]; f.extrinsics.orientation.z = v[5]; f.extrinsics.orientation.w = v[6];
    f.intrinsics.hFov = v[7]; f.intrinsics.vFov = v[8];
  }
  for (int i = std::max(n, 0); i < video.numFrames(); ++i) ds.frame(i).enabled = false;
}

float loadScale(const std::string& path) {
  logInfo("Searching 'scales.csv'...");
  // When several scales.csv exist below path, the last one visited wins, as in the reference; entries are visited in sorted name order
  // so that which one that is does not depend on the file system.
  std::string csv;
  std::function<void(const std::string&)> visit = [&](const std::string& dir) {
    for (const fs::directory_entry& e : sortedEntries(dir)) {
      if (e.path().filename() == "scales.csv") csv = e.path().string();
      else if (e.is_directory()) visit(e.path().string());
    }
  };
  visit(path);
  // The reference starts the sum at 1, so the scale is (1 + sum) / count rather than the mean of the listed scales; kept as it is.
  float scale = 1.f;
  if (csv.empty()) { logInfo("Could not find 'scales.csv'. Using default scale."); return scale; }
  std::ifstream f(csv);
  if (f.fail()) throw std::runtime_error("Could not open 'scales.csv'.");
  int count = 0;
  for (std::string line; std::getline(f, line);) {
    const std::vector<std::string> parts = explode(line, ',');
    if (parts.size() != 2) { logInfo("ERROR: invalid line '" + line + "'."); continue; }
    scale += float(std::atof(parts[1].c_str()));
    ++count;
  }
  if (count > 0) scale /= count;
  logInfo("  Scale = " + std::to_string(scale) + ".");
  return scale;
}

void importColmapDepth(DepthVideo& video) {
  logInfo("Importing COLMAP depth maps...");
  const std::string src = video.path() + "/depth_colmap_dense/depth", dst = video.path() + "/depth_colmap_dense_imported/depth";
  if (fileExists(dst)) { logInfo("  Destination directory already exists, skipping."); return; }
  if (!fs::is_directory(src)) throw std::runtime_error("COLMAP depth directory '" + src + "' does not exist.");
  makeDirs(dst);
  const float scale = loadScale(video.path());
  for (const fs::directory_entry& e : sortedEntries(src)) {
    const std::string name = e.path().stem().string();   // the reference reads <stem>.raw whatever the entry's extension
    Image depth; freadim(src + "/" + name + ".raw", depth);
    if (depth.type != cvMakeType(CV_32F, 1)) throw std::runtime_error("COLMAP depth image '" + name + ".raw' is not single-channel float.");
    float* d = depth.ptr<float>();
    for (size_t i = 0; i < size_t(depth.rows) * depth.cols; ++i) d[i] = (!std::isfinite(d[i]) || d[i] < 0.f) ? 0.f : d[i] * scale;
    fwriteim(dst + "/" + name + ".raw", depth);
  }
  logInfo("  Done.");
}

void importColmapRecon(DepthVideo& video, const std::string& npzFile, int stream, bool silent) {
  DepthStream& ds = video.depthStream(stream);
  const float scale = loadScale(video.path());
  // The reconstructed frames are the ones with a depth file.  Everything is checked before the stream is changed.
  std::vector<int> frames;
  for (const fs::directory_entry& e : sortedEntries(ds.path() + "/depth")) {
    const std::string name = e.path().stem().string();
    if (name.size() != 12 || name.compare(0, 6, "frame_") != 0 || name.find_first_not_of("0123456789", 6) != std::string::npos)
      throw std::runtime_error("Depth file name '" + e.path().filename().string() + "' does not have the expected format 'frame_NNNNNN.*'.");
    const int index = std::stoi(name.substr(6));
    if (index >= video.numFrames()) throw std::runtime_error("Depth file '" + e.path().filename().string() + "' is past the last frame of the video.");
    frames.push_back(index);
  }
  std::sort(frames.begin(), frames.end());
  const NpyF64 extr = npzLoadF64(npzFile, "extrinsics"), intr = npzLoadF64(npzFile, "intrinsics");
  auto shapeStr = [](const NpyF64& a) { std::string s = "("; for (size_t i = 0; i < a.shape.size(); ++i) s += (i ? ", " : "") + std::to_string(a.shape[i]); return s + ")"; };
  if (extr.shape.size() != 3 || extr.shape[1] != 3 || extr.shape[2] != 4) throw std::runtime_error("'extrinsics' in '" + npzFile + "' has shape " + shapeStr(extr) + "; expected (N, 3, 4).");
  if (intr.shape.size() != 2 || intr.shape[1] != 4) throw std::runtime_error("'intrinsics' in '" + npzFile + "' has shape " + shapeStr(intr) + "; expected (N, 4).");
  if (extr.shape[0] != intr.shape[0]) throw std::runtime_error("'" + npzFile + "' has " + std::to_string(extr.shape[0]) + " extrinsics but " + std::to_string(intr.shape[0]) + " intrinsics.");
  if (extr.shape[0] != frames.size())
    throw std::runtime_error("'" + npzFile + "' has " + std::to_string(extr.shape[0]) + " cameras but '" + ds.path() + "/depth' has " + std::to_string(frames.size()) + " depth files.");
  if (extr.fortranOrder || intr.fortranOrder) throw std::runtime_error("'" + npzFile + "' holds Fortran-order arrays; only C order is supported.");
  for (int i = 0; i < video.numFrames(); ++i) ds.frame(i).enabled = false;
  // Both the metadata and the extrinsics have +x pointing right and +y up, and the camera faces -z: the rotation's columns are the camera's
  // right, up and backward vectors in world space, the fourth column its position.
  if (!silent) logInfo("Loading Extrinsics...");
  for (size_t i = 0; i < frames.size(); ++i) {
    const double* P = &extr.data[12 * i];
    float R[3][3], q[4];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) R[r][c] = float(P[4 * r + c]);
    matrixToQuat(R, q);
    DepthFrame& df = ds.frame(frames[i]);
    df.enabled = true;
    df.extrinsics.position = {float(P[3]) / scale, float(P[7]) / scale, float(P[11]) / scale};
    df.extrinsics.orientation.x = q[0]; df.extrinsics.orientation.y = q[1]; df.extrinsics.orientation.z = q[2]; df.extrinsics.orientation.w = q[3];
    if (!silent) {
      char b[200]; const Extrinsics& x = df.extrinsics;
      snprintf(b, sizeof(b), "  Frame %d: position %g %g %g, orientation %g %g %g %g", frames[i], x.position.x, x.position.y, x.position.z, x.orientation.x, x.orientation.y, x.orientation.z, x.orientation.w);
      logInfo(b);
    }
  }
  if (!silent) logInfo("Loading Intrinsics...");
  const int w = ds.width(), h = ds.height();
  for (size_t i = 0; i < frames.size(); ++i) {
    const double fx = intr.data[4 * i], fy = intr.data[4 * i + 1];
    Intrinsics in;
    in.hFov = float(2 * std::atan2(w / 2.0, fx));
    in.vFov = float(2 * std::atan2(h / 2.0, fy));
    ds.frame(frames[i]).intrinsics = in;
    if (!silent) { char b[160]; snprintf(b, sizeof(b), "  Frame %d: fx %g fy %g -> hFov %g vFov %g", frames[i], fx, fy, in.hFov, in.vFov); logInfo(b); }
  }
}

// track2d.csv: one "frame, track, x, y" line per observation in pixels of the "full" stream, frames in non-decreasing order.  Both
// coordinates are divided by the image width.  A line without four fields is reported and skipped; any other line parses with atoi /
// atof as in the reference, so a header line is an observation of track 0 at frame 0 at (0, 0).  (The reference trims each field
// first; atoi and atof skip leading white space and stop at trailing white space, so that changes nothing.)  Where the reference
// asserts or indexes before its first frame -- an observation that is not on the frame after its track's last one, a negative frame --
// a RuntimeError is raised and no file is written.
void importTracks(DepthVideo& video, const std::string& trackFile) {
  std::ifstream f(trackFile);
  if (f.fail()) throw std::runtime_error("Cannot open track file.");
  const Image* img = video.colorStream("full").frame(0).image();
  if (!img) throw std::runtime_error("Color stream 'full' has no image for frame 0, whose width the track coordinates are divided by.");
  const float w = float(img->cols);
  DepthVideoTrackTable tt;
  std::map<int, int> tableId;   // track id in the file -> id in the table
  int lastFrame = -1;
  for (std::string line; std::getline(f, line);) {
    const std::vector<std::string> parts = explode(line, ',');
    if (parts.size() != 4) { logInfo("ERROR: invalid line '" + line + "'."); continue; }
    const int frame = std::atoi(parts[0].c_str()), track = std::atoi(parts[1].c_str());
    const float x = float(std::atof(parts[2].c_str())), y = float(std::atof(parts[3].c_str()));
    if (frame < lastFrame) throw std::runtime_error("ERROR: Frames not in consecutive order.");
    if (frame < 0) throw std::runtime_error("Track file '" + trackFile + "' has an observation at frame " + std::to_string(frame) + ".");
    for (; lastFrame < frame; ++lastFrame) tt.frames.emplace_back();
    const std::array<float, 2> obs{{x / w, y / w}};
    const auto it = tableId.find(track);
    int id;
    if (it == tableId.end()) {
      id = tableId[track] = int(tt.tracks.size());
      tt.tracks.emplace_back();
      tt.tracks.back().valid = true; tt.tracks.back().firstFrame = frame;
    } else {
      id = it->second;
      const DepthVideoTrack& t = tt.tracks[id];
      const int next = t.firstFrame + int(t.obs.size());
      if (frame != next)
        throw std::runtime_error("Track " + std::to_string(track) + " in '" + trackFile + "' has an observation at frame " + std::to_string(frame) +
                                 " after its last one at frame " + std::to_string(next - 1) + "; each must follow on the next frame.");
    }
    tt.tracks[id].obs.push_back(obs);
    tt.frames[frame].insert(id);
  }
  tt.save(video.path() + "/long_tracks.tracktable");
}

// --- .npz archives: a zip file (PKWARE APPNOTE) of .npy members, stored (np.savez) or deflated (np.savez_compressed).  numpy writes
// every member with zip64 extra fields; the central directory gives each member's sizes and local header offset. ---
static uint16_t le16(const uint8_t* p) { return uint16_t(p[0] | (p[1] << 8)); }
static uint32_t le32(const uint8_t* p) { return uint32_t(le16(p)) | (uint32_t(le16(p + 2)) << 16); }
static uint64_t le64(const uint8_t* p) { return uint64_t(le32(p)) | (uint64_t(le32(p + 4)) << 32); }

// .npy: magic, version, header length, then a Python dict literal {'descr': '<f8', 'fortran_order': False, 'shape': (3, 4), } and the data
static NpyF64 parseNpy(const std::vector<uint8_t>& b, const std::string& what) {
  auto bad = [&](const std::string& why) { return std::runtime_error(what + " is not a readable .npy array: " + why + "."); };
  if (b.size() < 10 || memcmp(b.data(), "\x93NUMPY", 6) != 0) throw bad("no .npy magic");
  size_t hoff = 10, hlen = le16(&b[8]);
  if (b[6] == 2 || b[6] == 3) { if (b.size() < 12) throw bad("truncated header"); hoff = 12; hlen = le32(&b[8]); }
  else if (b[6] != 1) throw bad("unknown format version " + std::to_string(b[6]));
  if (hlen > b.size() - hoff) throw bad("truncated header");
  const std::string h(b.begin() + hoff, b.begin() + hoff + hlen);
  auto value = [&](const char* key) {
    size_t p = h.find(std::string("'") + key + "'");
    if (p != std::string::npos) p = h.find(':', p);
    if (p != std::string::npos) p = h.find_first_not_of(' ', p + 1);
    if (p == std::string::npos) throw bad(std::string("no '") + key + "' in the header");
    return p;
  };
  NpyF64 a;
  size_t p = value("descr"), q = h.find('\'', p + 1);
  if (h[p] != '\'' || q == std::string::npos) throw bad("malformed 'descr'");
  const std::string descr = h.substr(p + 1, q - p - 1);
  p = value("fortran_order");
  if (h.compare(p, 4, "True") == 0) a.fortranOrder = true;
  else if (h.compare(p, 5, "False") != 0) throw bad("malformed 'fortran_order'");
  p = value("shape"); q = h.find(')', p);
  if (h[p] != '(' || q == std::string::npos) throw bad("malformed 'shape'");
  size_t count = 1;
  for (std::string d : explode(h.substr(p + 1, q - p - 1), ',')) {
    trim(d);
    if (d.empty()) continue;
    if (d.find_first_not_of("0123456789") != std::string::npos) throw bad("malformed 'shape'");
    a.shape.push_back(std::stoull(d));
    if (__builtin_mul_overflow(count, a.shape.back(), &count)) throw bad("the shape is too large");
  }
  if (descr != "<f8") throw std::runtime_error(what + " has dtype '" + descr + "'; only little-endian float64 ('<f8') is supported.");
  if (b.size() - hoff - hlen != count * sizeof(double)) throw bad("the data size does not match the shape");
  a.data.resize(count);
  if (count) memcpy(a.data.data(), &b[hoff + hlen], count * sizeof(double));   // the host is little-endian (x86-64, aarch64)
  return a;
}

NpyF64 npzLoadF64(const std::string& fileName, const std::string& key) {
  std::ifstream is(fileName, std::ios::binary);
  if (!is) throw std::runtime_error("Could not open '" + fileName + "'.");
  const std::vector<uint8_t> buf((std::istreambuf_iterator<char>(is)), std::istreambuf_iterator<char>());
  auto bad = [&](const std::string& why) { return std::runtime_error("'" + fileName + "' is not a readable .npz archive: " + why + "."); };
  auto at = [&](uint64_t off, uint64_t len) { if (off > buf.size() || len > buf.size() - off) throw bad("truncated"); return buf.data() + off; };
  // end-of-central-directory record: the last one in the final 22 + 65535 (longest comment) bytes
  if (buf.size() < 22) throw bad("too short");
  size_t eocd = buf.size() - 22;
  while (le32(&buf[eocd]) != 0x06054b50) { if (eocd == 0 || buf.size() - eocd >= 22 + 65535) throw bad("no end-of-central-directory record"); --eocd; }
  uint64_t entries = le16(&buf[eocd + 10]), off = le32(&buf[eocd + 16]);
  if (entries == 0xFFFF || off == 0xFFFFFFFF) {   // zip64: the locator just before the record points to the zip64 record
    if (eocd < 20 || le32(&buf[eocd - 20]) != 0x07064b50) throw bad("no zip64 end-of-central-directory locator");
    const uint8_t* z = at(le64(&buf[eocd - 12]), 56);
    if (le32(z) != 0x06064b50) throw bad("bad zip64 end-of-central-directory record");
    entries = le64(z + 32); off = le64(z + 48);
  }
  const std::string member = key + ".npy";
  for (uint64_t e = 0; e < entries; ++e) {
    const uint8_t* c = at(off, 46);
    if (le32(c) != 0x02014b50) throw bad("bad central directory entry");
    const uint16_t method = le16(c + 10), nameLen = le16(c + 28), extraLen = le16(c + 30), commentLen = le16(c + 32);
    const uint32_t crc = le32(c + 16);
    uint64_t csize = le32(c + 20), usize = le32(c + 24), local = le32(c + 42);
    const uint8_t* name = at(off + 46, uint64_t(nameLen) + extraLen + commentLen);
    off += 46 + uint64_t(nameLen) + extraLen + commentLen;
    if (std::string(reinterpret_cast<const char*>(name), nameLen) != member) continue;
    // zip64 extended information (id 1): the 64-bit values of the saturated fields, in this order
    for (const uint8_t *x = name + nameLen, *end = x + extraLen; x + 4 <= end;) {
      const uint8_t *v = x + 4, *ve = v + le16(x + 2);
      if (ve > end) throw bad("malformed extra field");
      if (le16(x) == 1) {
        auto take = [&](uint64_t& f) { if (f != 0xFFFFFFFF) return; if (v + 8 > ve) throw bad("short zip64 field"); f = le64(v); v += 8; };
        take(usize); take(csize); take(local);
      }
      x = ve;
    }
    const uint8_t* lh = at(local, 30);
    if (le32(lh) != 0x04034b50) throw bad("bad local header");
    const uint8_t* data = at(local + 30 + le16(lh + 26) + le16(lh + 28), csize);
    if (usize > UINT_MAX || csize > UINT_MAX) throw bad("member '" + member + "' is larger than 4 GiB");
    std::vector<uint8_t> raw(usize);
    if (method == 0) {
      if (csize != usize) throw bad("stored member '" + member + "' has inconsistent sizes");
      if (usize) memcpy(raw.data(), data, usize);
    } else if (method == 8) {
      z_stream zs{}; int rc = inflateInit2(&zs, -MAX_WBITS);   // raw deflate, no zlib header
      if (rc == Z_OK) {
        zs.next_in = const_cast<Bytef*>(data); zs.avail_in = uInt(csize); zs.next_out = raw.data(); zs.avail_out = uInt(usize);
        rc = inflate(&zs, Z_FINISH);
        inflateEnd(&zs);
      }
      if (rc != Z_STREAM_END || zs.total_out != usize) throw bad("member '" + member + "' does not inflate");
    } else {
      throw bad("member '" + member + "' uses compression method " + std::to_string(method) + "; only stored and deflated members are supported");
    }
    if (crc32(0L, raw.data(), uInt(usize)) != crc) throw bad("member '" + member + "' fails its CRC check");
    return parseNpy(raw, "'" + key + "' in '" + fileName + "'");
  }
  throw std::runtime_error("'" + fileName + "' has no array '" + key + "'.");
}

// --- pose conversions (lib/PoseOptimizer.cpp:769-781, :968-974) ---
void quatToAngleAxis(const Quatf& qf, double aa[3]) {
  const double qx = qf.x, qy = qf.y, qz = qf.z, qw = qf.w;
  auto rot = [&](double vx, double vy, double vz, double o[3]) {   // Eigen quaternion * vector in double
    double ux = qy * vz - qz * vy, uy = qz * vx - qx * vz, uz = qx * vy - qy * vx; ux += ux; uy += uy; uz += uz;
    o[0] = vx + qw * ux + (qy * uz - qz * uy); o[1] = vy + qw * uy + (qz * ux - qx * uz); o[2] = vz + qw * uz + (qx * uy - qy * ux);
  };
  double right[3], up[3], front[3]; rot(1, 0, 0, right); rot(0, 1, 0, up); rot(-0.0, -0.0, -1, front);
  // rotation.col(0) = right, col(1) = up, col(2) = -front ; R(i,j) = col j, row i
  double R[3][3]; for (int i = 0; i < 3; ++i) { R[i][0] = right[i]; R[i][1] = up[i]; R[i][2] = -front[i]; }
  // ceres::RotationMatrixToQuaternion
  double q[4]; const double trace = R[0][0] + R[1][1] + R[2][2];
  if (trace >= 0.0) { double t = std::sqrt(trace + 1.0); q[0] = 0.5 * t; t = 0.5 / t; q[1] = (R[2][1] - R[1][2]) * t; q[2] = (R[0][2] - R[2][0]) * t; q[3] = (R[1][0] - R[0][1]) * t; }
  else {
    int i = 0; if (R[1][1] > R[0][0]) i = 1; if (R[2][2] > R[i][i]) i = 2; const int j = (i + 1) % 3, k = (j + 1) % 3;
    double t = std::sqrt(R[i][i] - R[j][j] - R[k][k] + 1.0); q[i + 1] = 0.5 * t; t = 0.5 / t;
    q[0] = (R[k][j] - R[j][k]) * t; q[j + 1] = (R[j][i] + R[i][j]) * t; q[k + 1] = (R[k][i] + R[i][k]) * t;
  }
  // ceres::QuaternionToAngleAxis
  const double s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (s2 > 0.0) {
    const double s = std::sqrt(s2), c = q[0];
    const double two_theta = 2.0 * ((c < 0.0) ? std::atan2(-s, -c) : std::atan2(s, c));
    const double k = two_theta / s; aa[0] = q[1] * k; aa[1] = q[2] * k; aa[2] = q[3] * k;
  } else { aa[0] = q[1] * 2.0; aa[1] = q[2] * 2.0; aa[2] = q[3] * 2.0; }
}
Quatf angleAxisToQuat(const double aa[3]) {
  double R[3][3];   // R[i][j]: row i, column j  (ceres::AngleAxisToRotationMatrix, column-major adapter)
  const double th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (th2 > std::numeric_limits<double>::epsilon()) {
    const double th = std::sqrt(th2), wx = aa[0] / th, wy = aa[1] / th, wz = aa[2] / th, c = std::cos(th), s = std::sin(th);
    R[0][0] = c + wx * wx * (1.0 - c); R[1][0] = wz * s + wx * wy * (1.0 - c); R[2][0] = -wy * s + wx * wz * (1.0 - c);
    R[0][1] = wx * wy * (1.0 - c) - wz * s; R[1][1] = c + wy * wy * (1.0 - c); R[2][1] = wx * s + wy * wz * (1.0 - c);
    R[0][2] = wy * s + wx * wz * (1.0 - c); R[1][2] = -wx * s + wy * wz * (1.0 - c); R[2][2] = c + wz * wz * (1.0 - c);
  } else {
    R[0][0] = 1; R[1][0] = aa[2]; R[2][0] = -aa[1]; R[0][1] = -aa[2]; R[1][1] = 1; R[2][1] = aa[0]; R[0][2] = aa[1]; R[1][2] = -aa[0]; R[2][2] = 1;
  }
  double q[4]; matrixToQuat(R, q);   // Eigen::Quaterniond(Matrix3d)
  Quatf o; o.x = float(q[0]); o.y = float(q[1]); o.z = float(q[2]); o.w = float(q[3]); return o;
}

}  // namespace rcvdh
