// export_text.hpp -- the text the reference's export commands write, without the library or any third-party dependency:
//   ostreamFloat        a float put on a std::ostream with its default format (PCD VIEWPOINT, the pose .txt of
//                       saveIndividualCloudsToFile, graph_mgr_io.cpp:414-418)
//   YamlFileStorage     the subset of cv::FileStorage's YAML writer (OpenCV 4.13, persistence_yml.cpp) that
//                       saveAllFeaturesToFile (graph_mgr_io.cpp:445-497) uses: a block sequence of flow maps of doubles, and
//                       a CV_8U matrix
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace rgbdslam_b200 {

// std::ostream << float with the stream's defaults: the float widened to double, printed as "%g" (precision 6)
inline std::string ostreamFloat(float v) {
  char buf[32];
  std::snprintf(buf, sizeof(buf), "%g", (double)v);
  return buf;
}

// cv::FileStorage (YAML, WRITE) as far as these calls go; text() is the file after release().  Writing a float forwards a
// double, as cv::write(FileStorage&, const String&, float) does.
class YamlFileStorage {
 public:
  YamlFileStorage() : text_("%YAML:1.0\n---\n") { stack_.push_back(Struct{0, kMap | kEmpty}); }

  // fs << key << "[" ... fs << "]": a block sequence
  void startSeq(const char* key) { startStruct(key, kSeq, nullptr); }
  // fs << "{:" ... fs << "}": a flow map, an element of the current sequence
  void startFlowMap() { startStruct(nullptr, kMap | kFlow, nullptr); }
  void endStruct() {
    if (stack_.size() < 2) throw std::logic_error("YamlFileStorage: no open structure");
    const Struct& cur = stack_.back();
    if (cur.flags & kFlow) {
      if (line_.size() > (size_t)cur.indent && !(cur.flags & kEmpty)) line_ += ' ';
      line_ += (cur.flags & kMap) ? '}' : ']';
    } else if (cur.flags & kEmpty) {
      flush();
      line_ += (cur.flags & kMap) ? "{}" : "[]";
    }
    stack_.pop_back();
    stack_.back().flags &= ~kEmpty;
  }
  void writeReal(const char* key, double v) { writeScalar(key, doubleToString(v).c_str()); }
  void writeInt(const char* key, int v) { writeScalar(key, std::to_string(v).c_str()); }
  // fs << key << m for a rows x cols CV_8U matrix (row-major bytes)
  void writeMatU8(const char* key, const uint8_t* data, int rows, int cols) {
    startStruct(key, kMap, "opencv-matrix");
    writeInt("rows", rows);
    writeInt("cols", cols);
    writeScalar("dt", "u");
    startStruct("data", kSeq | kFlow, nullptr);
    for (size_t i = 0; i < (size_t)rows * cols; i++) writeScalar(nullptr, std::to_string((int)data[i]).c_str());
    endStruct();
    endStruct();
  }
  // FileStorage::release: closes what is open and returns the file's text
  const std::string& release() {
    while (stack_.size() > 1) endStruct();
    flush();
    return text_;
  }

  // cv::FileStorage's doubleToString: an integer value that fits an int as "%d.", NaN as ".Nan", +-inf as ".Inf" / "-.Inf",
  // every other value as "%.17g"
  static std::string doubleToString(double v) {
    if (std::isnan(v)) return ".Nan";
    if (std::isinf(v)) return v < 0 ? "-.Inf" : ".Inf";
    char buf[40];
    if (v >= -2147483648.0 && v <= 2147483647.0 && std::nearbyint(v) == v) std::snprintf(buf, sizeof(buf), "%d.", (int)v);
    else std::snprintf(buf, sizeof(buf), "%.17g", v);
    return buf;
  }

 private:
  enum { kSeq = 1, kMap = 2, kFlow = 4, kEmpty = 8 };
  static constexpr int kIndent = 3;        // CV_YML_INDENT
  static constexpr int kWrapMargin = 71;   // FileStorage's wrap_margin
  struct Struct {
    int indent, flags;
  };
  std::string text_, line_;  // the written text and the line being built (its first `space_` bytes are the indent)
  int space_ = 0;
  std::vector<Struct> stack_;

  // FileStorage::Impl::flush: ends the current line if it holds more than its indent, and starts one at the current indent
  void flush() {
    if (line_.size() > (size_t)space_) text_ += line_ + "\n";
    space_ = stack_.back().indent;
    line_.assign(space_, ' ');
  }
  void startStruct(const char* key, int flags, const char* type_name) {
    std::string data;
    if (flags & kFlow) data = std::string(type_name ? std::string("!!") + type_name + " " : "") + ((flags & kMap) ? '{' : '[');
    else if (type_name) data = std::string("!!") + type_name;
    writeScalar(key, data.empty() ? nullptr : data.c_str());
    const Struct& parent = stack_.back();
    Struct s{parent.indent, flags | kEmpty};
    if (!(parent.flags & kFlow)) s.indent += kIndent + ((flags & kFlow) ? 1 : 0);
    stack_.back().flags &= ~kEmpty;
    stack_.push_back(s);
    if (!(flags & kFlow)) flush();
  }
  // YAMLEmitter::writeScalar
  void writeScalar(const char* key, const char* data) {
    Struct& cur = stack_.back();
    const size_t keylen = key ? std::strlen(key) : 0, datalen = data ? std::strlen(data) : 0;
    if (cur.flags & kFlow) {
      if (!(cur.flags & kEmpty)) line_ += ',';
      const size_t new_offset = line_.size() + keylen + datalen;
      if (new_offset > (size_t)kWrapMargin && new_offset - cur.indent > 10) flush();
      else line_ += ' ';
    } else {
      flush();
      if (!(cur.flags & kMap)) {
        line_ += '-';
        if (data) line_ += ' ';
      }
    }
    if (key) {
      line_ += key;
      line_ += ':';
      if (!(cur.flags & kFlow) && data) line_ += ' ';
    }
    if (data) line_ += data;
    cur.flags &= ~kEmpty;
  }
};

}  // namespace rgbdslam_b200
