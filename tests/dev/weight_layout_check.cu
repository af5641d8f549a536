// weight_layout_check.cu -- runs csrc/weight_arena.cuh's host layout step for tests/test_weight_layouts.py (no GPU needed).
//   weight_layout_check layout d0 d1 d2 p ld n half dtype dtype16 scale dst_bytes src.bin out.bin
//     src.bin: the n source elements; out.bin: a dst_bytes destination that starts as 0xa5 bytes after weight_layout's
//     bytes were placed where weight_upload says bind copies them.
//   weight_layout_check seed <seed> <name>   prints init_random's seed for the tensor `name`
#include <stdio.h>
#include <stdlib.h>

#include "../../speech_to_speech_b200/csrc/weight_arena.cuh"

int main(int argc, char** argv) {
  if (argc == 4 && strcmp(argv[1], "seed") == 0) {
    printf("%llu\n", (unsigned long long)weight_seed(strtoull(argv[2], nullptr, 10), argv[3]));
    return 0;
  }
  if (argc != 15) { fprintf(stderr, "usage: see the header of weight_layout_check.cu\n"); return 2; }
  WeightSlot s;
  s.as(atoi(argv[1]), atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]));
  s.n = atoll(argv[7]);
  s.half = atoi(argv[8]) != 0;
  const int dtype = atoi(argv[9]), dtype16 = atoi(argv[10]);
  s.scale = strtof(argv[11], nullptr);
  std::vector<uint8_t> src((size_t)s.n * (dtype == S2S_F32 ? 4 : 2)), dst((size_t)atoll(argv[12]), 0xa5), bytes;
  FILE* f = fopen(argv[13], "rb");
  if (!f || fread(src.data(), 1, src.size(), f) != src.size()) { fprintf(stderr, "cannot read %s\n", argv[13]); return 2; }
  fclose(f);
  weight_layout(s, src.data(), dtype, dtype16, bytes);
  const WeightUpload u = weight_upload(s);
  if (u.width * u.height != bytes.size() || u.offset + (u.height - 1) * u.pitch + u.width > dst.size()) {
    fprintf(stderr, "upload of %zu x %zu bytes does not fit\n", u.height, u.width);
    return 1;
  }
  for (size_t r = 0; r < u.height; ++r) memcpy(dst.data() + u.offset + r * u.pitch, bytes.data() + r * u.width, u.width);
  f = fopen(argv[14], "wb");
  if (!f || fwrite(dst.data(), 1, dst.size(), f) != dst.size()) { fprintf(stderr, "cannot write %s\n", argv[14]); return 2; }
  fclose(f);
  return 0;
}
