// TEST AND MEASUREMENT INFRASTRUCTURE.  Prometheus' XOR appender (tsdb/chunkenc/xor.go) in C++, for batches too large
// for the Python encoder of tests/chunks_ref.py, which it mirrors line for line (tests/test_chunks_encode.py holds the
// two equal byte for byte).
//     chunks_encode DIR PER_CHUNK
// DIR/offsets.u64 (n_series + 1), ts.i64 and bits.u64 (the samples, series after series, values as float64 bits) ->
// DIR/series_chunks.u64, chunk_bytes.u64, data.u8: each series cut into chunks of at most PER_CHUNK samples.
#include <stdint.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>
#include <vector>

template <class T>
static std::vector<T> read_all(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) {
    fprintf(stderr, "cannot read %s\n", path.c_str());
    exit(2);
  }
  f.seekg(0, std::ios::end);
  std::vector<T> v((size_t)f.tellg() / sizeof(T));
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(v.size() * sizeof(T)));
  return v;
}

template <class T>
static void write_all(const std::string& path, const std::vector<T>& v) {
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), (std::streamsize)(v.size() * sizeof(T)));
}

struct Writer {
  std::vector<uint8_t>& out;
  uint32_t free_bits = 0;   // unused low bits of the last byte
  void put(uint64_t v, int n) {
    for (int k = n - 1; k >= 0; --k) {
      if (free_bits == 0) out.push_back(0), free_bits = 8;
      --free_bits;
      out.back() |= (uint8_t)(((v >> k) & 1u) << free_bits);
    }
  }
  void uvarint(uint64_t x) {
    while (x >= 0x80) put((x & 0x7f) | 0x80, 8), x >>= 7;
    put(x, 8);
  }
};

static bool bit_range(int64_t x, int n) { return -((1ll << (n - 1)) - 1) <= x && x <= (1ll << (n - 1)); }

static void encode(const int64_t* ts, const uint64_t* bits, size_t n, std::vector<uint8_t>& out) {
  out.push_back((uint8_t)(n >> 8)), out.push_back((uint8_t)n);
  Writer w{out};
  uint64_t t_prev = 0, delta_prev = 0, v_prev = 0;
  int lead = 0xff, trail = 0;
  for (size_t i = 0; i < n; ++i) {
    const uint64_t t = (uint64_t)ts[i], v = bits[i];
    if (i == 0) {
      w.uvarint((t << 1) ^ (uint64_t)((int64_t)t >> 63));
      w.put(v, 64);
    } else {
      const uint64_t delta = t - t_prev;
      if (i == 1) {
        w.uvarint(delta);
      } else {
        const int64_t dod = (int64_t)(delta - delta_prev);
        if (dod == 0) w.put(0, 1);
        else if (bit_range(dod, 14)) w.put(0b10, 2), w.put((uint64_t)dod & 0x3fff, 14);
        else if (bit_range(dod, 17)) w.put(0b110, 3), w.put((uint64_t)dod & 0x1ffff, 17);
        else if (bit_range(dod, 20)) w.put(0b1110, 4), w.put((uint64_t)dod & 0xfffff, 20);
        else w.put(0b1111, 4), w.put((uint64_t)dod, 64);
      }
      delta_prev = delta;
      const uint64_t x = v ^ v_prev;
      if (x == 0) {
        w.put(0, 1);
      } else {
        w.put(1, 1);
        int new_lead = __builtin_clzll(x), new_trail = __builtin_ctzll(x);
        if (new_lead > 31) new_lead = 31;
        if (lead != 0xff && new_lead >= lead && new_trail >= trail) {
          w.put(0, 1), w.put(x >> trail, 64 - lead - trail);
        } else {
          lead = new_lead, trail = new_trail;
          const int sig = 64 - lead - trail;
          w.put(1, 1), w.put((uint64_t)lead, 5), w.put((uint64_t)sig & 63u, 6), w.put(x >> trail, sig);
        }
      }
    }
    t_prev = t, v_prev = v;
  }
}

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: chunks_encode DIR PER_CHUNK\n");
    return 2;
  }
  const std::string dir = argv[1];
  const size_t per = (size_t)atol(argv[2]);
  if (per == 0 || per > 65535) return 2;
  const std::vector<uint64_t> offsets = read_all<uint64_t>(dir + "/offsets.u64");
  const std::vector<int64_t> ts = read_all<int64_t>(dir + "/ts.i64");
  const std::vector<uint64_t> bits = read_all<uint64_t>(dir + "/bits.u64");
  if (offsets.empty() || offsets.back() != ts.size() || ts.size() != bits.size()) return 2;
  std::vector<uint64_t> series_chunks{0}, chunk_bytes{0};
  std::vector<uint8_t> data;
  data.reserve(ts.size() * 3);
  for (size_t s = 0; s + 1 < offsets.size(); ++s) {
    for (uint64_t i = offsets[s]; i < offsets[s + 1]; i += per) {
      const size_t n = (size_t)std::min<uint64_t>(per, offsets[s + 1] - i);
      encode(ts.data() + i, bits.data() + i, n, data);
      chunk_bytes.push_back(data.size());
    }
    series_chunks.push_back(chunk_bytes.size() - 1);
  }
  write_all(dir + "/series_chunks.u64", series_chunks);
  write_all(dir + "/chunk_bytes.u64", chunk_bytes);
  write_all(dir + "/data.u8", data);
  return 0;
}
