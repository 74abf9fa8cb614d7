// TEST INFRASTRUCTURE.  Exposes the number conversion of the device text parser (gpu-pruner_b200/csrc/gpr_text.cuh,
// compiled as plain C++) on stdin/stdout so that tests/test_text_numbers.py can compare it with Python's correctly
// rounded float():
//   E <mantissa> <exp10>   ->  "<ok> <hex bits of the binary64>"      eisel_lemire
//   V <decimal text>       ->  "<consumed> <hex bits of the f32> <tiny>"   parse_value (0 consumed = declined)
//   T <timestamp text>     ->  "<offset of ','> <seconds>"            parse_timestamp on "[<text>,"
//   S <threshold> <text>   ->  "<consumed> <hex f32> <hex up> <hex down>"   parse_value into a power plane (power_snap)
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../gpu-pruner_b200/csrc/gpr_text.cuh"

namespace tx = gpr::text;
struct Buf {
  const uint8_t* p;
  uint32_t operator[](uint32_t i) const { return p[i]; }
};

int main() {
  char line[512];
  while (fgets(line, sizeof line, stdin)) {
    const size_t n = strcspn(line, "\r\n");
    line[n] = 0;
    if (line[0] == 'E') {
      unsigned long long man;
      int e10;
      if (sscanf(line + 2, "%llu %d", &man, &e10) != 2) return 2;
      double d = 0;
      const bool ok = tx::eisel_lemire(man, e10, &d);
      uint64_t bits;
      memcpy(&bits, &d, 8);
      printf("%d %016" PRIx64 "\n", ok ? 1 : 0, ok ? bits : 0);
    } else if (line[0] == 'V') {
      uint8_t buf[256] = {0};
      const size_t len = strlen(line + 2);
      memcpy(buf, line + 2, len);
      buf[len] = '"';
      float f = 0;
      uint32_t tiny = 0;
      const uint32_t q = tx::parse_value(Buf{buf}, 0, tx::kMaxSample - 2, &f, &tiny);
      uint32_t bits;
      memcpy(&bits, &f, 4);
      printf("%u %08x %u\n", q == len ? q : 0u, q == len ? bits : 0u, tiny);
    } else if (line[0] == 'S') {
      // S <threshold> <decimal text>  ->  "<consumed> <hex bits of the stored power sample> <hex up> <hex down>"
      char* rest = nullptr;
      const double thr = strtod(line + 2, &rest);
      while (*rest == ' ') ++rest;
      uint8_t buf[256] = {0};
      const size_t len = strlen(rest);
      memcpy(buf, rest, len);
      buf[len] = '"';
      float f = 0;
      uint32_t tiny = 0;
      const tx::PowerSnap snap = tx::power_snap(thr);
      const uint32_t q = tx::parse_value(Buf{buf}, 0, tx::kMaxSample - 2, &f, &tiny, snap);
      uint32_t bits, up, down;
      memcpy(&bits, &f, 4), memcpy(&up, &snap.up, 4), memcpy(&down, &snap.down, 4);
      printf("%u %08x %08x %08x\n", q == len ? q : 0u, q == len ? bits : 0u, up, down);
    } else if (line[0] == 'T') {
      uint8_t buf[256] = {0};
      const size_t len = strlen(line + 2);
      buf[0] = '[';
      memcpy(buf + 1, line + 2, len);
      buf[len + 1] = ',';
      int64_t ts = 0;
      const uint32_t q = tx::parse_timestamp(Buf{buf}, 0, &ts);
      printf("%u %" PRId64 "\n", q, q ? ts : 0);
    }
  }
  return 0;
}
