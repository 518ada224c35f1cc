// constraints.cpp -- FlowConstraintsCollection (reference lib/FlowConstraints.cpp) and the OpenCV
// image operators it relies on, restated (cvtColor BGR2GRAY, cornerMinEigenVal(blockSize 3),
// distanceTransform(DIST_L2, 5)).  Two builders produce identical lists: the GPU builder (default; rcvd_build_constraints,
// csrc/rcvd_builder.cuh, SURVEY.md section 8f-2) and the sequential host builder below, which is the reference's own CPU
// stage restated and is selected explicitly with RCVD_CONSTRAINT_BUILDER=host (no automatic fallback: without a CUDA
// device the default builder fails).
#include "model.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <fstream>
#include <sstream>
#include <stdexcept>
#include <sys/stat.h>

namespace rcvdh {

static bool fileExists(const std::string& f) { struct stat st; return stat(f.c_str(), &st) == 0; }
static std::string pairName(const char* fmt, const std::string& path, int a, int b) { char buf[512]; snprintf(buf, sizeof(buf), fmt, path.c_str(), a, b); return buf; }

// cv::cvtColor(COLOR_BGR2GRAY) for CV_32FC3 in the operation order of OpenCV 4.13's vector body (RGB2Gray<float>, found by search
// against cv2, tests/test_host.py): fma(r, 0.299f, fma(b, 0.114f, g * 0.587f)).  Built with -ffp-contract=off: every fusion is explicit.
Image bgr2gray32f(const Image& bgr) {
  if (bgr.type != cvMakeType(CV_32F, 3)) throw std::runtime_error("bgr2gray32f expects CV_32FC3.");
  Image g; g.create(bgr.rows, bgr.cols, cvMakeType(CV_32F, 1));
  const float* s = bgr.ptr<float>(); float* d = g.ptr<float>();
  const float cb = 0.114f, cg = 0.587f, cr = 0.299f;
  for (size_t i = 0; i < size_t(bgr.rows) * bgr.cols; ++i) d[i] = std::fmaf(s[3 * i + 2], cr, std::fmaf(s[3 * i], cb, s[3 * i + 1] * cg));
  return g;
}
static inline int reflect101(int p, int n) { if (n == 1) return 0; while (p < 0 || p >= n) { if (p < 0) p = -p; else p = 2 * n - 2 - p; } return p; }
// cv::cornerMinEigenVal(src, dst, blockSize = 3, ksize = 3, BORDER_DEFAULT) for CV_32FC1, bit-exact with cv2 4.13 (AVX2 paths):
// Sobel with the scale 1/(2^(ksize-1) * blockSize) = 1/12 folded into the smoothing kernel (cv::Sobel), fused where OpenCV's
// universal intrinsics fuse; covariance products; 3x3 box sum accumulated in double (cv::boxFilter, CV_64F sum type, normalize =
// false) and rounded once; then (a + c) - sqrt((a - c)^2 + b^2) with a = dxx/2, b = dxy, c = dyy/2, unfused.
Image cornerMinEigenVal3(const Image& src) {
  const int h = src.rows, w = src.cols;
  const float scale = 1.f / 12.f, scale2 = 2.f * scale;
  std::vector<float> dx(size_t(w) * h), dy(size_t(w) * h);
  const float* S = src.ptr<float>();
  auto at = [&](int y, int x) { return S[size_t(reflect101(y, h)) * w + reflect101(x, w)]; };
  std::vector<float> rd(size_t(w) * h), rs(size_t(w) * h);   // row derivative [-1 0 1] (unscaled), row smoothing [s 2s s]
  const int wvec = w & ~3;                                    // SymmRowSmallVec_32f body; the scalar tail fuses the other way round
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    const float a = at(y, x - 1), b = at(y, x), c = at(y, x + 1);
    rd[size_t(y) * w + x] = c - a;
    const float lr = a + c;
    rs[size_t(y) * w + x] = x < wvec ? std::fmaf(b, scale2, lr * scale) : std::fmaf(lr, scale, b * scale2);
  }
  auto rdAt = [&](int y, int x) { return rd[size_t(reflect101(y, h)) * w + x]; };
  auto rsAt = [&](int y, int x) { return rs[size_t(reflect101(y, h)) * w + x]; };
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    dx[size_t(y) * w + x] = std::fmaf(rdAt(y - 1, x) + rdAt(y + 1, x), scale, rdAt(y, x) * scale2);   // column [s 2s s] (SymmColumnSmallVec_32f)
    dy[size_t(y) * w + x] = rsAt(y + 1, x) - rsAt(y - 1, x);                                          // column [-1 0 1]
  }
  std::vector<float> cxx(size_t(w) * h), cxy(size_t(w) * h), cyy(size_t(w) * h);
  for (size_t i = 0; i < size_t(w) * h; ++i) { cxx[i] = dx[i] * dx[i]; cxy[i] = dx[i] * dy[i]; cyy[i] = dy[i] * dy[i]; }
  auto box = [&](const std::vector<float>& in, std::vector<float>& out) {
    std::vector<double> tmp(size_t(w) * h);
    for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) tmp[size_t(y) * w + x] = (double(in[size_t(y) * w + reflect101(x - 1, w)]) + double(in[size_t(y) * w + x])) + double(in[size_t(y) * w + reflect101(x + 1, w)]);
    // ColumnSum<double, float>: the running sum slides down the column (its last bit decides exact float ties, so the recurrence is kept)
    for (int x = 0; x < w; ++x) {
      double sum = tmp[size_t(reflect101(-1, h)) * w + x] + tmp[x];
      for (int y = 0; y < h; ++y) {
        const double s0 = sum + tmp[size_t(reflect101(y + 1, h)) * w + x];
        out[size_t(y) * w + x] = float(s0);
        sum = s0 - tmp[size_t(reflect101(y - 1, h)) * w + x];
      }
    }
  };
  std::vector<float> bxx(size_t(w) * h), bxy(size_t(w) * h), byy(size_t(w) * h);
  box(cxx, bxx); box(cxy, bxy); box(cyy, byy);
  Image out; out.create(h, w, cvMakeType(CV_32F, 1));
  float* D = out.ptr<float>();
  for (size_t i = 0; i < size_t(w) * h; ++i) {
    const float a = bxx[i] * 0.5f, b = bxy[i], c = byy[i] * 0.5f;
    D[i] = (a + c) - std::sqrt((a - c) * (a - c) + b * b);
  }
  return out;
}
// cv::distanceTransform(src, dst, DIST_L2, DIST_MASK_5): two-pass 5x5 chamfer with fixed-point weights
// (1, 1.4, 2.1969) << 16.
Image distanceTransformL2_5(const Image& bin) {
  const int h = bin.rows, w = bin.cols, B = 2, step = w + 2 * B;
  const unsigned HV = 65536u, DIAG = unsigned(1.4f * 65536.f + 0.5f), LONG = unsigned(2.1969f * 65536.f + 0.5f);
  const unsigned INIT = unsigned(INT_MAX) >> 2, DMAX = unsigned(INT_MAX - (1 << 16)) ;
  std::vector<unsigned> tmp(size_t(step) * (h + 2 * B), INIT);
  auto T = [&](int y, int x) -> unsigned& { return tmp[size_t(y + B) * step + x + B]; };
  for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) {
    if (!bin.data[size_t(y) * w + x]) { T(y, x) = 0; continue; }
    unsigned t0 = T(y - 2, x - 1) + LONG, t;
    t = T(y - 2, x + 1) + LONG; if (t0 > t) t0 = t;
    t = T(y - 1, x - 2) + LONG; if (t0 > t) t0 = t;
    t = T(y - 1, x - 1) + DIAG; if (t0 > t) t0 = t;
    t = T(y - 1, x) + HV; if (t0 > t) t0 = t;
    t = T(y - 1, x + 1) + DIAG; if (t0 > t) t0 = t;
    t = T(y - 1, x + 2) + LONG; if (t0 > t) t0 = t;
    t = T(y, x - 1) + HV; if (t0 > t) t0 = t;
    T(y, x) = t0;
  }
  Image out; out.create(h, w, cvMakeType(CV_32F, 1));
  const float scale = 1.f / 65536.f;
  for (int y = h - 1; y >= 0; --y) for (int x = w - 1; x >= 0; --x) {
    unsigned t0 = T(y, x), t;
    if (t0 > HV) {
      t = T(y + 2, x + 1) + LONG; if (t0 > t) t0 = t;
      t = T(y + 2, x - 1) + LONG; if (t0 > t) t0 = t;
      t = T(y + 1, x + 2) + LONG; if (t0 > t) t0 = t;
      t = T(y + 1, x + 1) + DIAG; if (t0 > t) t0 = t;
      t = T(y + 1, x) + HV; if (t0 > t) t0 = t;
      t = T(y + 1, x - 1) + DIAG; if (t0 > t) t0 = t;
      t = T(y + 1, x - 2) + LONG; if (t0 > t) t0 = t;
      t = T(y, x + 1) + HV; if (t0 > t) t0 = t;
      T(y, x) = t0;
    }
    t0 = t0 > DMAX ? DMAX : t0;
    out.ptr<float>()[size_t(y) * w + x] = float(t0 * scale);
  }
  return out;
}

// ---------------------------------------------------------------------------
FlowConstraintsCollection::FlowConstraintsCollection(DepthVideo& video, const FlowConstraintsParams& params)
    : video_(&video), path_(video.path()), params_(params) {
  logInfo("Setting up flow constraints...");
  const std::string listFile = path_ + "/flow_list.json";
  if (!fileExists(listFile)) throw std::runtime_error("Flow list file does not exist.");
  // flow_list.json (flow.py:53-74): [[header...], [a, b, ratio], ...]; only the two leading ints of rows >= 1 matter (:59-72)
  std::ifstream is(listFile); std::stringstream ss; ss << is.rdbuf(); const std::string txt = ss.str();
  int depth = 0, row = -1; size_t i = 0;
  while (i < txt.size()) {
    const char ch = txt[i];
    if (ch == '[') { ++depth; if (depth == 2) { ++row; if (row >= 1) {
          int vals[2] = {0, 0}; int nv = 0; size_t j = i + 1;
          while (j < txt.size() && txt[j] != ']' && nv < 2) {
            while (j < txt.size() && (txt[j] == ' ' || txt[j] == ',' || txt[j] == '\n' || txt[j] == '\t')) ++j;
            size_t k = j; while (k < txt.size() && txt[k] != ',' && txt[k] != ']') ++k;
            vals[nv++] = int(std::stod(txt.substr(j, k - j))); j = k;
          }
          if (nv == 2 && params.frameRange.inRange(vals[0]) && params.frameRange.inRange(vals[1])) pairs_.emplace(PairKey(vals[0], vals[1]), std::vector<PairConstraint>());
        } } }
    else if (ch == ']') --depth;
    ++i;
  }
  for (int t = params.frameRange.firstFrame() + 1; t <= params.frameRange.lastFrame() - 1; ++t)
    if (params.frameRange.inRange(t - 1) && params.frameRange.inRange(t) && params.frameRange.inRange(t + 1)) triplets_.emplace(t, std::vector<TripletConstraint>());
  if (params.doNotUseCache) compute();
  else if (!load()) { compute(); save(); }
}

// flow_constraints.dat (lib/FlowConstraints.cpp:116-224)
template <class T> static T rd(std::istream& is) { T v; is.read(reinterpret_cast<char*>(&v), sizeof(T)); return v; }
template <class T> static void wr(std::ostream& os, const T& v) { os.write(reinterpret_cast<const char*>(&v), sizeof(T)); }
bool FlowConstraintsCollection::load() {
  const std::string fn = path_ + "/flow_constraints.dat";
  if (!fileExists(fn)) { logInfo("Constraints cache file '" + fn + "' does not exist."); return false; }
  logInfo("Loading cached constraints from '" + fn + "'...");
  std::ifstream is(fn, std::ios::binary);
  if (rd<uint32_t>(is) != 0xDEADBEEF) throw std::runtime_error("Did not see magic marker at beginning of file.");
  const uint32_t fmt = rd<uint32_t>(is);
  if (fmt > 3) throw std::runtime_error("File format too new.");
  if (fmt < 3) throw std::runtime_error("File format too old.");
  if (rd<int32_t>(is) != params_.matchSeparation) { logInfo("Cache file has the wrong parameters... Not loading."); return false; }
  for (auto& kv : pairs_) {
    const int a = rd<int32_t>(is), b = rd<int32_t>(is);
    if (a != kv.first.first || b != kv.first.second) throw std::runtime_error("Read incorrect pair from file.");
    const uint64_t n = rd<uint64_t>(is); kv.second.resize(n);
    for (auto& c : kv.second) { is.read(reinterpret_cast<char*>(c.loc), sizeof(float) * 4); c.isStatic = true; }
  }
  for (auto& kv : triplets_) {
    if (rd<int32_t>(is) != kv.first) throw std::runtime_error("Read incorrect triplet from file.");
    const uint64_t n = rd<uint64_t>(is); kv.second.resize(n);
    for (auto& c : kv.second) { is.read(reinterpret_cast<char*>(c.loc), sizeof(float) * 6); c.isStatic = true; }
  }
  if (rd<uint32_t>(is) != 0xDEADBEEF) throw std::runtime_error("Did not see magic marker at end of file.");
  return true;
}
void FlowConstraintsCollection::save() {
  const std::string fn = path_ + "/flow_constraints.dat";
  logInfo("Writing constraints to '" + fn + "'...");
  std::ofstream os(fn, std::ios::binary);
  wr<uint32_t>(os, 0xDEADBEEF); wr<uint32_t>(os, 3); wr<int32_t>(os, params_.matchSeparation);
  for (auto& kv : pairs_) { wr<int32_t>(os, kv.first.first); wr<int32_t>(os, kv.first.second); wr<uint64_t>(os, kv.second.size()); for (auto& c : kv.second) os.write(reinterpret_cast<const char*>(c.loc), sizeof(float) * 4); }
  for (auto& kv : triplets_) { wr<int32_t>(os, kv.first); wr<uint64_t>(os, kv.second.size()); for (auto& c : kv.second) os.write(reinterpret_cast<const char*>(c.loc), sizeof(float) * 6); }
  wr<uint32_t>(os, 0xDEADBEEF);
}

Image FlowConstraintsCollection::dynamicDistance(int frame) {   // :257-286
  if (video_->hasColorStream("dynamic_mask")) {
    const Image* m = video_->colorStream("dynamic_mask").frame(frame).image();
    if (!m) throw std::runtime_error("Dynamic mask stream is missing a frame.");
    Image bin; bin.create(m->rows, m->cols, cvMakeType(CV_8U, 1));
    for (size_t i = 0; i < bin.data.size(); ++i) bin.data[i] = m->data[i] < 127 ? 0 : 255;
    return distanceTransformL2_5(bin);
  }
  ColorStream& cs = video_->colorStream("down");
  Image d; d.create(cs.height(), cs.width(), cvMakeType(CV_32F, 1));
  std::fill(d.ptr<float>(), d.ptr<float>() + size_t(d.rows) * d.cols, 3.402823466e+38f);
  return d;
}
// RCVD_CONSTRAINT_BUILDER: unset, empty or "gpu" selects the device path of the constraint operations, "host" the sequential
// restatement; anything else is an error.  There is no automatic fallback.
static bool hostConstraintPath() {
  const char* sel = std::getenv("RCVD_CONSTRAINT_BUILDER");
  if (sel && !(std::string(sel) == "host" || std::string(sel) == "gpu" || std::string(sel).empty())) throw std::runtime_error("RCVD_CONSTRAINT_BUILDER must be 'gpu' or 'host'.");
  return sel && std::string(sel) == "host";
}
void FlowConstraintsCollection::compute() {
  logInfo("Computing constraints...");
  if (hostConstraintPath()) {
    for (auto& kv : pairs_) compute(kv.first);
    for (auto& kv : triplets_) computeTriplet(kv.first);
  } else {
    computeOnDevice();
  }
}

namespace {
template <class C> struct Pixel { float cornerStrength; C data; bool operator<(const Pixel& o) const { return cornerStrength > o.cornerStrength; } };
struct FlowMask { Image flow, mask; };
FlowMask loadFlowAndMask(DepthVideo& video, const std::string& path, int a, int b) {   // :226-255
  ColorStream& cs = video.colorStream("down");
  const int w = cs.width(), h = cs.height();
  const std::string ff = pairName("%s/flow/flow_%06d_%06d.raw", path, a, b);
  if (!fileExists(ff)) throw std::runtime_error("Flow file does not exist.");
  FlowMask r; freadim(ff, r.flow);
  if (r.flow.cols != w || r.flow.rows != h || r.flow.type != cvMakeType(CV_32F, 2)) throw std::runtime_error("Flow has the wrong size.");
  const std::string mf = pairName("%s/flow_mask/mask_%06d_%06d.png", path, a, b);
  if (!fileExists(mf)) throw std::runtime_error("Mask file does not exist.");
  r.mask = imreadPng(mf, true);
  if (r.mask.cols != w || r.mask.rows != h) throw std::runtime_error("Mask has the wrong size.");
  return r;
}
// sampleConstraints (:352-397): sort by corner strength (std::sort, not stable), greedy disc stamping.
template <class C, int REF> void sampleConstraints(DepthVideo& video, int sep, std::vector<Pixel<C>>& pixels, std::vector<C>& output, int nobs) {
  ColorStream& cs = video.colorStream("down");
  const int w = cs.width(), h = cs.height();
  std::stable_sort(pixels.begin(), pixels.end());   // the reference's std::sort leaves equal scores unordered; scan order breaks ties here and on the GPU
  std::vector<uint8_t> invalid(size_t(w) * h, 0);
  const int size = 2 * sep + 1;
  std::vector<uint8_t> disk(size_t(size) * size);
  for (int y = 0; y < size; ++y) for (int x = 0; x < size; ++x) { const int rx = x - sep, ry = y - sep; disk[size_t(y) * size + x] = (rx * rx + ry * ry <= sep * sep) ? 255 : 0; }
  const float sx = 1.f / w, sy = video.invAspect() / h;
  for (const auto& p : pixels) {
    const int rxp = int(p.data.loc[REF][0]), ryp = int(p.data.loc[REF][1]);
    if (invalid[size_t(ryp) * w + rxp]) continue;
    C c = p.data;
    for (int o = 0; o < nobs; ++o) { c.loc[o][0] = p.data.loc[o][0] * sx; c.loc[o][1] = p.data.loc[o][1] * sy; }
    output.push_back(c);
    const int mx0 = std::max(0, rxp - sep), mx1 = std::min(w - 1, rxp + sep), my0 = std::max(0, ryp - sep), my1 = std::min(h - 1, ryp + sep);
    for (int my = my0; my <= my1; ++my) { const int dy = my - (ryp - sep);
      for (int mx = mx0; mx <= mx1; ++mx) { const int dx = mx - (rxp - sep); if (disk[size_t(dy) * size + dx]) invalid[size_t(my) * w + mx] = 255; } }
  }
}
}  // namespace

void FlowConstraintsCollection::compute(const PairKey& pair) {   // :401-465
  ColorStream& cs = video_->colorStream("down");
  const Image* color = cs.frame(pair.first).image();
  if (!color) throw std::runtime_error("Missing color frame.");
  const int w = color->cols, h = color->rows;
  FlowMask fm = loadFlowAndMask(*video_, path_, pair.first, pair.second);
  Image dd0 = dynamicDistance(pair.first), dd1 = dynamicDistance(pair.second);
  const float dsx = dd0.cols / float(cs.width()), dsy = dd0.rows / float(cs.height());
  Image corner = cornerMinEigenVal3(bgr2gray32f(*color));
  std::vector<Pixel<PairConstraint>> pixels; pixels.reserve(size_t(w) * h);
  for (int iy0 = 0; iy0 < h; ++iy0) {
    const float* cornerPtr = corner.ptr<float>(iy0); const float* flowPtr = fm.flow.ptr<float>(iy0); const uint8_t* maskPtr = fm.mask.ptr<uint8_t>(iy0);
    const int iy0s = int(iy0 * dsy + 0.5f);
    const float* dd0Ptr = dd0.ptr<float>(iy0s);
    for (int ix0 = 0; ix0 < w; ++ix0) {
      const int ix0s = int(ix0 * dsx + 0.5f);
      if (maskPtr[ix0] && dd0Ptr[ix0s] > params_.minDynamicDistance) {
        const float fx1 = ix0 + flowPtr[2 * ix0], fy1 = iy0 + flowPtr[2 * ix0 + 1];
        const int ix1 = int(fx1 + 0.5f), iy1 = int(fy1 + 0.5f);
        if (ix1 >= 0 && ix1 < w && iy1 >= 0 && iy1 < h) {
          const int ix1s = int(fx1 * dsx + 0.5f), iy1s = int(fy1 * dsy + 0.5f);
          if (dd1.ptr<float>(iy1s)[ix1s] > params_.minDynamicDistance) {
            Pixel<PairConstraint> p; p.cornerStrength = cornerPtr[ix0];
            p.data.loc[0][0] = float(ix0); p.data.loc[0][1] = float(iy0); p.data.loc[1][0] = fx1; p.data.loc[1][1] = fy1; p.data.isStatic = true;
            pixels.push_back(p);
          }
        }
      }
    }
  }
  sampleConstraints<PairConstraint, 0>(*video_, params_.matchSeparation, pixels, pairs_.at(pair), 2);
}
void FlowConstraintsCollection::computeTriplet(int triplet) {   // :467-550 (quirks kept: score read at ix0, third test on dynamicDistance1)
  ColorStream& cs = video_->colorStream("down");
  const Image* color = cs.frame(triplet).image();
  if (!color) throw std::runtime_error("Missing color frame.");
  const int w = color->cols, h = color->rows;
  const std::string f10 = pairName("%s/flow/flow_%06d_%06d.raw", path_, triplet, triplet - 1), f12 = pairName("%s/flow/flow_%06d_%06d.raw", path_, triplet, triplet + 1);
  if (!fileExists(f10) || !fileExists(f12)) { return; }   // triplets are only used by the (default-off) smoothness loss
  FlowMask a = loadFlowAndMask(*video_, path_, triplet, triplet - 1), b = loadFlowAndMask(*video_, path_, triplet, triplet + 1);
  Image dd0 = dynamicDistance(triplet - 1), dd1 = dynamicDistance(triplet);
  const float dsx = dd0.cols / float(cs.width()), dsy = dd0.rows / float(cs.height());
  Image corner = cornerMinEigenVal3(bgr2gray32f(*color));
  std::vector<Pixel<TripletConstraint>> pixels;
  for (int iy1 = 0; iy1 < h; ++iy1) {
    const float* cornerPtr = corner.ptr<float>(iy1);
    const int iy1s = int(iy1 * dsy + 0.5f);
    for (int ix1 = 0; ix1 < w; ++ix1) {
      const int ix1s = int(ix1 * dsx + 0.5f);
      if (a.mask.ptr<uint8_t>(iy1)[ix1] && b.mask.ptr<uint8_t>(iy1)[ix1] && dd1.ptr<float>(iy1s)[ix1s] > params_.minDynamicDistance) {
        const float fx0 = ix1 + a.flow.ptr<float>(iy1)[2 * ix1], fy0 = iy1 + a.flow.ptr<float>(iy1)[2 * ix1 + 1];
        const int ix0 = int(fx0 + 0.5f), iy0 = int(fy0 + 0.5f);
        const float fx2 = ix1 + b.flow.ptr<float>(iy1)[2 * ix1], fy2 = iy1 + b.flow.ptr<float>(iy1)[2 * ix1 + 1];
        const int ix2 = int(fx2 + 0.5f), iy2 = int(fy2 + 0.5f);
        if (ix0 >= 0 && ix0 < w && iy0 >= 0 && iy0 < h && ix2 >= 0 && ix2 < w && iy2 >= 0 && iy2 < h) {
          const int ix0s = int(fx0 * dsx + 0.5f), iy0s = int(fy0 * dsy + 0.5f), ix2s = int(fx2 * dsx + 0.5f), iy2s = int(fy2 * dsy + 0.5f);
          if (dd0.ptr<float>(iy0s)[ix0s] > params_.minDynamicDistance && dd1.ptr<float>(iy2s)[ix2s] > params_.minDynamicDistance) {
            Pixel<TripletConstraint> p; p.cornerStrength = cornerPtr[ix0];
            p.data.loc[0][0] = fx0; p.data.loc[0][1] = fy0; p.data.loc[1][0] = float(ix1); p.data.loc[1][1] = float(iy1); p.data.loc[2][0] = fx2; p.data.loc[2][1] = fy2; p.data.isStatic = true;
            pixels.push_back(p);
          }
        }
      }
    }
  }
  sampleConstraints<TripletConstraint, 1>(*video_, params_.matchSeparation, pixels, triplets_.at(triplet), 3);
}

// All pairs and triplets through rcvd_build_constraints, in batches that bound the host staging memory.
namespace { template <class T> struct RawBuf {   // uninitialised array (new T[n] default-initialises trivial types: no fill)
  explicit RawBuf(size_t n) : p(n ? new T[n] : nullptr) {}
  T* data() { return p.get(); }
  std::unique_ptr<T[]> p;
}; }
void FlowConstraintsCollection::computeOnDevice() {
  ColorStream& cs = video_->colorStream("down");
  const int w = cs.width(), h = cs.height();
  if (w <= 0 || h <= 0) throw std::runtime_error("Missing color frame.");
  const size_t plane = size_t(w) * h;
  // frames referenced by any item -> local indices
  std::map<int, int> local;
  for (auto& kv : pairs_) { local[kv.first.first] = 0; local[kv.first.second] = 0; }
  std::vector<int> trips;
  for (auto& kv : triplets_) {
    const int t = kv.first;
    if (!fileExists(pairName("%s/flow/flow_%06d_%06d.raw", path_, t, t - 1)) || !fileExists(pairName("%s/flow/flow_%06d_%06d.raw", path_, t, t + 1))) continue;
    trips.push_back(t); local[t - 1] = 0; local[t] = 0; local[t + 1] = 0;
  }
  if (local.empty()) return;
  int F = 0; for (auto& kv : local) kv.second = F++;
  std::vector<float> color(size_t(F) * plane * 3), dyn;
  const bool hasDyn = video_->hasColorStream("dynamic_mask");
  int dw = 0, dh = 0;
  // colour frames (+ distance transforms of the dynamic masks) into the staging arrays: files, PNG decoding and the chamfer pass are
  // independent per frame -> host threads; the first frame goes alone because it fixes the streams' dimensions
  std::vector<int> fr; fr.reserve(local.size()); for (auto& kv : local) fr.push_back(kv.first);   // local index = position
  auto stageFrame = [&](size_t i) {
    const Image* img = cs.frame(fr[i]).image();
    if (!img) throw std::runtime_error("Missing color frame.");
    if (img->cols != w || img->rows != h || img->type != cvMakeType(CV_32F, 3)) throw std::runtime_error("Color frame has the wrong size or type.");
    std::memcpy(color.data() + i * plane * 3, img->ptr<float>(), plane * 3 * sizeof(float));
    if (hasDyn) {
      Image dd = dynamicDistance(fr[i]);
      if (i == 0) { dw = dd.cols; dh = dd.rows; dyn.resize(size_t(F) * dw * dh); }
      if (dd.cols != dw || dd.rows != dh) throw std::runtime_error("Dynamic masks have inconsistent dimensions.");
      std::memcpy(dyn.data() + i * size_t(dw) * dh, dd.ptr<float>(), size_t(dw) * dh * sizeof(float));
    }
  };
  stageFrame(0);
  parallelFor(fr.size() - 1, [&](size_t i) { stageFrame(i + 1); });
  rcvd_builder_params prm{};
  prm.num_frames = F; prm.width = w; prm.height = h; prm.dyn_width = dw; prm.dyn_height = dh; prm.match_separation = params_.matchSeparation;
  prm.min_dynamic_distance = params_.minDynamicDistance; prm.inv_aspect = video_->invAspect();
  const size_t kBatchBytes = size_t(768) << 20;   // staging budget per call
  const size_t perPair = plane * 9, perTrip = plane * 18;
  std::vector<PairKey> keys; for (auto& kv : pairs_) keys.push_back(kv.first);
  size_t pi = 0, ti = 0;
  while (pi < keys.size() || ti < trips.size()) {
    const size_t np = std::min(keys.size() - pi, std::max<size_t>(1, kBatchBytes / perPair));
    const size_t budgetLeft = kBatchBytes > np * perPair ? kBatchBytes - np * perPair : 0;
    const size_t nt = pi + np >= keys.size() ? std::min(trips.size() - ti, std::max<size_t>(np == 0 ? 1 : 0, budgetLeft / perTrip)) : 0;
    std::vector<int32_t> pf(np * 2), tf(nt);
    // staging arrays are written slot by slot below: no zero fill (std::vector's value-initialisation of ~0.7 GB per batch cost more
    // wall-clock than reading and decoding the files)
    RawBuf<float> pflow(np * plane * 2), tflow(nt * 2 * plane * 2);
    RawBuf<uint8_t> pmask(np * plane), tmask(nt * 2 * plane);
    // flow + mask files of the batch (file reads and PNG inflation dominate the builder's wall-clock): one slot per item, host threads
    parallelFor(np, [&](size_t k) {
      const PairKey& key = keys[pi + k];
      FlowMask fm = loadFlowAndMask(*video_, path_, key.first, key.second);
      pf[2 * k] = local.at(key.first); pf[2 * k + 1] = local.at(key.second);
      std::memcpy(pflow.data() + k * plane * 2, fm.flow.ptr<float>(), plane * 2 * sizeof(float)); std::memcpy(pmask.data() + k * plane, fm.mask.ptr<uint8_t>(), plane);
    });
    for (size_t k = 0; k < nt; ++k) {
      const int t = trips[ti + k]; tf[k] = local.at(t);
      if (local.at(t - 1) != local.at(t) - 1) throw std::runtime_error("Triplet frames must be consecutive in the constraint frame range.");
    }
    parallelFor(nt * 2, [&](size_t q) {
      const size_t k = q / 2; const int s2 = int(q % 2); const int t = trips[ti + k];
      FlowMask fm = loadFlowAndMask(*video_, path_, t, s2 == 0 ? t - 1 : t + 1);
      std::memcpy(tflow.data() + (k * 2 + s2) * plane * 2, fm.flow.ptr<float>(), plane * 2 * sizeof(float)); std::memcpy(tmask.data() + (k * 2 + s2) * plane, fm.mask.ptr<uint8_t>(), plane);
    });
#ifdef RCVD_STAGE_SELFCHECK   // development check of the threaded staging against a sequential reload (make CXXFLAGS+=-DRCVD_STAGE_SELFCHECK)
    {
      for (size_t k = 0; k < np; ++k) {
        const PairKey& key = keys[pi + k];
        FlowMask fm = loadFlowAndMask(*video_, path_, key.first, key.second);
        if (pf[2 * k] != local.at(key.first) || pf[2 * k + 1] != local.at(key.second) || std::memcmp(pflow.data() + k * plane * 2, fm.flow.ptr<float>(), plane * 2 * sizeof(float)) ||
            std::memcmp(pmask.data() + k * plane, fm.mask.ptr<uint8_t>(), plane)) throw std::logic_error("stage selfcheck: pair staging differs");
      }
      for (size_t k = 0; k < nt; ++k) for (int s2 = 0; s2 < 2; ++s2) {
        const int t = trips[ti + k];
        FlowMask fm = loadFlowAndMask(*video_, path_, t, s2 == 0 ? t - 1 : t + 1);
        if (std::memcmp(tflow.data() + (k * 2 + s2) * plane * 2, fm.flow.ptr<float>(), plane * 2 * sizeof(float)) || std::memcmp(tmask.data() + (k * 2 + s2) * plane, fm.mask.ptr<uint8_t>(), plane))
          throw std::logic_error("stage selfcheck: triplet staging differs");
      }
      for (size_t i = 0; i < fr.size(); ++i) {
        const Image* img = cs.frame(fr[i]).image();
        if (std::memcmp(color.data() + i * plane * 3, img->ptr<float>(), plane * 3 * sizeof(float))) throw std::logic_error("stage selfcheck: colour staging differs");
        if (hasDyn) { Image dd = dynamicDistance(fr[i]); if (std::memcmp(dyn.data() + i * size_t(dw) * dh, dd.ptr<float>(), size_t(dw) * dh * sizeof(float))) throw std::logic_error("stage selfcheck: distance staging differs"); }
      }
      fprintf(stderr, "stage selfcheck ok: %zu pairs, %zu triplets, %zu frames\n", np, nt, fr.size());
    }
#endif
    prm.num_pairs = int(np); prm.num_triplets = int(nt);
    std::vector<int64_t> poff(np + 1, 0), toff(nt + 1, 0);
    const int sep = std::max(1, params_.matchSeparation);
    int64_t pcap = int64_t(np) * int64_t(std::min<size_t>(plane, 4 * plane / (size_t(sep) * sep) + 64)), tcap = int64_t(nt) * int64_t(std::min<size_t>(plane, 4 * plane / (size_t(sep) * sep) + 64));
    std::vector<float> pout, tout;
    for (int attempt = 0; attempt < 2; ++attempt) {
      pout.resize(size_t(pcap) * 4); tout.resize(size_t(tcap) * 6);
      const int rc = rcvd_build_constraints(&prm, currentDevice(), color.data(), hasDyn ? dyn.data() : nullptr, pf.data(), pflow.data(), pmask.data(), tf.data(), tflow.data(), tmask.data(),
                                            poff.data(), pout.data(), pcap, toff.data(), tout.data(), tcap);
      if (rc == RCVD_OK) break;
      if (attempt == 0 && (poff[np] > pcap || toff[nt] > tcap)) { pcap = poff[np]; tcap = toff[nt]; continue; }   // sizes are known now
      throw std::runtime_error(std::string("GPU constraint builder failed: ") + rcvd_last_error());
    }
    for (size_t k = 0; k < np; ++k) {
      std::vector<PairConstraint>& out = pairs_.at(keys[pi + k]); out.clear(); out.resize(size_t(poff[k + 1] - poff[k]));
      for (size_t c = 0; c < out.size(); ++c) { std::memcpy(out[c].loc, pout.data() + (size_t(poff[k]) + c) * 4, 16); out[c].isStatic = true; }
    }
    for (size_t k = 0; k < nt; ++k) {
      std::vector<TripletConstraint>& out = triplets_.at(trips[ti + k]); out.clear(); out.resize(size_t(toff[k + 1] - toff[k]));
      for (size_t c = 0; c < out.size(); ++c) { std::memcpy(out[c].loc, tout.data() + (size_t(toff[k]) + c) * 6, 24); out[c].isStatic = true; }
    }
    pi += np; ti += nt;
  }
  rcvd_trim_device_memory(currentDevice());
}

// The pair and triplet lists as rcvd_static_flags and rcvd_prune_static_flags take them, in map order: pair frames / triplet centres,
// offsets, locations and one flag byte per constraint (the current flag with `withFlags`, else 0 for the call to overwrite).
struct FlagLists { std::vector<int32_t> pf, tc; std::vector<int64_t> po{0}, to{0}; std::vector<float> pl, tl; std::vector<uint8_t> ps, ts; };
template <class Pairs, class Trips> static FlagLists packFlagLists(const Pairs& pairs, const Trips& trips, bool withFlags) {
  FlagLists l;
  for (auto& kv : pairs) {
    l.pf.push_back(kv.first.first); l.pf.push_back(kv.first.second); l.po.push_back(l.po.back() + int64_t(kv.second.size()));
    for (auto& c : kv.second) { l.pl.insert(l.pl.end(), &c.loc[0][0], &c.loc[0][0] + 4); l.ps.push_back(withFlags && c.isStatic); }
  }
  for (auto& kv : trips) {
    l.tc.push_back(kv.first); l.to.push_back(l.to.back() + int64_t(kv.second.size()));
    for (auto& c : kv.second) { l.tl.insert(l.tl.end(), &c.loc[0][0], &c.loc[0][0] + 6); l.ts.push_back(withFlags && c.isStatic); }
  }
  return l;
}
template <class Pairs, class Trips> static void unpackFlags(const FlagLists& l, Pairs& pairs, Trips& trips) {
  size_t i = 0; for (auto& kv : pairs) for (auto& c : kv.second) c.isStatic = l.ps[i++] != 0;
  i = 0; for (auto& kv : trips) for (auto& c : kv.second) c.isStatic = l.ts[i++] != 0;
}

void FlowConstraintsCollection::resetStaticFlag() {
  for (auto& kv : pairs_) for (auto& c : kv.second) c.isStatic = true;
  for (auto& kv : triplets_) for (auto& c : kv.second) c.isStatic = true;
}
void FlowConstraintsCollection::setStaticFlagFromDynamicMask(int distance) {   // :573-660 (y is scaled by the mask WIDTH, :618-621)
  if (!video_->hasColorStream("dynamic_mask")) { resetStaticFlag(); return; }
  logInfo("Setting static flag from dynamic masks...");
  ColorStream& ms = video_->colorStream("dynamic_mask");
  const int w = ms.width(), h = ms.height();
  {
    // default: distance transforms + per-constraint lookups on the device (rcvd_static_flags); RCVD_CONSTRAINT_BUILDER=host
    // selects the sequential restatement below (no automatic fallback)
    if (!hostConstraintPath()) {
      const int F = video_->numFrames(); const size_t plane = size_t(w) * h;
      std::vector<uint8_t> masks(size_t(F) * plane, 255);
      std::vector<uint8_t> used(F, 0);
      for (auto& kv : pairs_) { used[kv.first.first] = 1; used[kv.first.second] = 1; }
      for (auto& kv : triplets_) { used[kv.first - 1] = 1; used[kv.first] = 1; used[kv.first + 1] = 1; }
      for (int f = 0; f < F; ++f) {
        if (!used[f]) continue;
        const Image* m = ms.frame(f).image();
        if (!m) throw std::runtime_error("Dynamic mask stream is missing a frame.");
        if (m->cols != w || m->rows != h) throw std::runtime_error("Dynamic masks have inconsistent dimensions.");
        std::memcpy(masks.data() + size_t(f) * plane, m->data.data(), plane);
      }
      FlagLists l = packFlagLists(pairs_, triplets_, false);
      const int rc = rcvd_static_flags(currentDevice(), masks.data(), F, h, w, float(distance), int(l.pf.size() / 2), l.pf.data(), l.po.data(), l.pl.data(),
                                       l.ps.data(), int(l.tc.size()), l.tc.data(), l.to.data(), l.tl.data(), l.ts.data(), nullptr);
      if (rc != RCVD_OK) throw std::runtime_error(std::string("rcvd_static_flags failed: ") + rcvd_last_error());
      unpackFlags(l, pairs_, triplets_);
      return;
    }
  }
  std::vector<Image> masks(video_->numFrames());
  auto getMask = [&](int f) -> const Image& {
    if (masks[f].empty()) { Image dd = dynamicDistance(f); masks[f].create(dd.rows, dd.cols, cvMakeType(CV_8U, 1));
      for (int y = 0; y < h; ++y) for (int x = 0; x < w; ++x) masks[f].data[size_t(y) * dd.cols + x] = dd.ptr<float>(y)[x] > distance ? 255 : 0; }
    return masks[f];
  };
  for (auto& kv : pairs_) {
    const Image& m0 = getMask(kv.first.first); const Image& m1 = getMask(kv.first.second);
    for (auto& c : kv.second) {
      const int ix0 = int(c.loc[0][0] * w), iy0 = int(c.loc[0][1] * w), ix1 = int(c.loc[1][0] * w), iy1 = int(c.loc[1][1] * w);
      c.isStatic = m0.data[size_t(iy0) * m0.cols + ix0] && m1.data[size_t(iy1) * m1.cols + ix1];
    }
  }
  for (auto& kv : triplets_) {
    const Image& m0 = getMask(kv.first - 1); const Image& m1 = getMask(kv.first); const Image& m2 = getMask(kv.first + 1);
    for (auto& c : kv.second) {
      const int x0 = int(c.loc[0][0] * w), y0 = int(c.loc[0][1] * w), x1 = int(c.loc[1][0] * w), y1 = int(c.loc[1][1] * w), x2 = int(c.loc[2][0] * w), y2 = int(c.loc[2][1] * w);
      c.isStatic = m0.data[size_t(y0) * m0.cols + x0] && m1.data[size_t(y1) * m1.cols + x1] && m2.data[size_t(y2) * m2.cols + x2];
    }
  }
}
void FlowConstraintsCollection::pruneStaticFlag(int distance) {   // :662-748
  ColorStream& ds = video_->colorStream("down");
  const int w = ds.width(), h = ds.height();
  const bool host = hostConstraintPath();
  // the stamps come from non-static pair constraints only: without one (or with a negative radius, where the reference fails in
  // OpenCV's Mat allocation) no flag can change
  bool anyDynamic = false;
  for (auto& kv : pairs_) for (auto& c : kv.second) anyDynamic = anyDynamic || !c.isStatic;
  if (!anyDynamic || distance < 0) return;
  if (!host) {
    // default: disc stamps into per-frame bit planes + per-constraint lookups on the device (rcvd_prune_static_flags)
    const int F = video_->numFrames();
    FlagLists l = packFlagLists(pairs_, triplets_, true);
    const int rc = rcvd_prune_static_flags(currentDevice(), F, h, w, distance, int(l.pf.size() / 2), l.pf.data(), l.po.data(), l.pl.data(), l.ps.data(),
                                           int(l.tc.size()), l.tc.data(), l.to.data(), l.tl.data(), l.ts.data());
    if (rc != RCVD_OK) throw std::runtime_error(std::string("rcvd_prune_static_flags failed: ") + rcvd_last_error());
    unpackFlags(l, pairs_, triplets_);
    return;
  }
  const int size = 2 * distance + 1;
  std::vector<uint8_t> disk(size_t(size) * size);
  for (int y = 0; y < size; ++y) for (int x = 0; x < size; ++x) { const int rx = x - distance, ry = y - distance; disk[size_t(y) * size + x] = (rx * rx + ry * ry <= distance * distance) ? 255 : 0; }
  std::vector<std::vector<uint8_t>> masks(video_->numFrames(), std::vector<uint8_t>(size_t(w) * h, 0));
  for (int frame = 0; frame < video_->numFrames(); ++frame)
    for (auto& kv : pairs_) {
      if (kv.first.first != frame && kv.first.second != frame) continue;
      for (auto& c : kv.second) {
        if (c.isStatic) continue;
        const float* loc = (kv.first.first == frame) ? c.loc[0] : c.loc[1];
        const int x = int(loc[0] * w), y = int(loc[1] * w);
        const int mx0 = std::max(0, x - distance), mx1 = std::min(w - 1, x + distance), my0 = std::max(0, y - distance), my1 = std::min(h - 1, y + distance);
        for (int my = my0; my <= my1; ++my) for (int mx = mx0; mx <= mx1; ++mx) if (disk[size_t(my - (y - distance)) * size + (mx - (x - distance))]) masks[frame][size_t(my) * w + mx] = 255;
      }
    }
  // lookups clamped to the image like the device's (k_prune_lookup): with a "down" aspect other than the video's, int(loc.y * w)
  // can reach h, where the reference reads past the frame
  auto at = [&](int frame, const float* loc) {
    const int x = std::min(std::max(int(loc[0] * w), 0), w - 1), y = std::min(std::max(int(loc[1] * w), 0), h - 1);
    return masks[frame][size_t(y) * w + x] != 0;
  };
  for (auto& kv : pairs_) for (auto& c : kv.second)
    if (at(kv.first.first, c.loc[0]) || at(kv.first.second, c.loc[1])) c.isStatic = false;
  for (auto& kv : triplets_) for (auto& c : kv.second)
    if (at(kv.first - 1, c.loc[0]) || at(kv.first, c.loc[1]) || at(kv.first + 1, c.loc[2])) c.isStatic = false;
}

}  // namespace rcvdh
