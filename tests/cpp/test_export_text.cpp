// The text writers of include/rgbdslam_b200/export_text.hpp, without the library.
//   test_export_text yaml spec.bin out.yml: spec.bin is int32 n, n x 3 float32 locations, int32 rows, rows x 32 bytes; writes
//     what saveAllFeaturesToFile's calls make of them (Feature_Locations, then Feature_Descriptors).
//   test_export_text g spec.bin: spec.bin is int32 n, n float32; prints ostreamFloat of each, one per line.
#include <cstdio>
#include <vector>

#include "rgbdslam_b200/export_text.hpp"

using namespace rgbdslam_b200;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = std::fopen(argv[2], "rb");
  int32_t n = 0;
  if (!f || std::fread(&n, 4, 1, f) != 1) return 2;
  const bool yaml = std::string(argv[1]) == "yaml";
  std::vector<float> v((size_t)n * (yaml ? 3 : 1));
  if (std::fread(v.data(), 4, v.size(), f) != v.size()) return 2;
  if (!yaml) {
    for (float x : v) std::printf("%s\n", ostreamFloat(x).c_str());
    return 0;
  }
  int32_t rows = 0;
  if (std::fread(&rows, 4, 1, f) != 1) return 2;
  std::vector<uint8_t> desc((size_t)rows * 32);
  if (std::fread(desc.data(), 1, desc.size(), f) != desc.size()) return 2;
  std::fclose(f);
  YamlFileStorage fs;
  fs.startSeq("Feature_Locations");
  for (int32_t i = 0; i < n; i++) {
    fs.startFlowMap();
    fs.writeReal("x", v[3 * i]);
    fs.writeReal("y", v[3 * i + 1]);
    fs.writeReal("z", v[3 * i + 2]);
    fs.endStruct();
  }
  fs.endStruct();
  fs.writeMatU8("Feature_Descriptors", desc.data(), rows, 32);
  const std::string& text = fs.release();
  FILE* o = argc > 3 ? std::fopen(argv[3], "wb") : nullptr;
  if (!o || std::fwrite(text.data(), 1, text.size(), o) != text.size()) return 2;
  std::fclose(o);
  return 0;
}
