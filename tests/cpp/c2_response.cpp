// The synthetic DCGM universe of DESIGN.md §7 as a Prometheus range-query response (TEST INFRASTRUCTURE).
//
//   c2_response OUT PLANE SEED P G T_TOTAL T0 C_LO C_HI
//
// writes the compact matrix JSON of plane PLANE (0 = DCGM_FI_DEV_GPU_UTIL, 1 = DCGM_FI_DEV_POWER_USAGE) of the
// universe P pods x G GPUs x T_TOTAL columns, columns C_LO <= c < C_HI, column c at unix time T0 + c (1 s step).
// Every cell is the oracle's own (gpo_synth_cell, oracle/gpr_oracle.c); a NaN cell (scrape gap, the gappy class'
// missing prefix) is an absent sample, and a series without a sample in the range is absent, as Prometheus
// answers.  Labels follow gph_synth_response (gpu-pruner_b200/host/capi.cpp).
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

extern "C" float gpo_synth_cell(uint64_t seed, int plane, uint64_t series, uint32_t t, uint32_t n_samples);

int main(int argc, char** argv) {
  if (argc != 10) {
    fprintf(stderr, "usage: c2_response OUT PLANE SEED P G T_TOTAL T0 C_LO C_HI\n");
    return 2;
  }
  const int plane = atoi(argv[2]);
  const uint64_t seed = strtoull(argv[3], nullptr, 0);
  const unsigned P = (unsigned)atoi(argv[4]), G = (unsigned)atoi(argv[5]), T = (unsigned)atoi(argv[6]);
  const long long t0 = atoll(argv[7]);
  const unsigned c_lo = (unsigned)atoi(argv[8]), c_hi = (unsigned)atoi(argv[9]);
  FILE* f = fopen(argv[1], "wb");
  if (!f || c_lo > c_hi || c_hi > T) return 1;
  const char* metric = plane == 0 ? "DCGM_FI_DEV_GPU_UTIL" : "DCGM_FI_DEV_POWER_USAGE";
  fputs("{\"status\":\"success\",\"data\":{\"resultType\":\"matrix\",\"result\":[", f);
  std::string values;
  char tmp[64];
  bool first = true;
  for (unsigned pod = 0; pod < P; ++pod)
    for (unsigned g = 0; g < G; ++g) {
      values.clear();
      const uint64_t s = (uint64_t)pod * G + g;
      for (unsigned c = c_lo; c < c_hi; ++c) {
        const float v = gpo_synth_cell(seed, plane, s, c, T);
        if (std::isnan(v)) continue;
        snprintf(tmp, sizeof tmp, "%s[%lld,\"%d\"]", values.empty() ? "" : ",", t0 + (long long)c, (int)v);
        values += tmp;
      }
      if (values.empty()) continue;
      fprintf(f,
              "%s{\"metric\":{\"__name__\":\"%s\",\"Hostname\":\"node-%u\",\"UUID\":\"GPU-%u-%u\",\"device\":\"nvidia%u\","
              "\"exported_container\":\"main\",\"exported_namespace\":\"ns-%u\",\"exported_pod\":\"pod-%u\",\"gpu\":\"%u\","
              "\"instance\":\"10.0.0.1:9400\",\"job\":\"dcgm\",\"modelName\":\"NVIDIA B200\"},\"values\":[%s]}",
              first ? "" : ",", metric, pod % 512, pod, g, g, pod % 64, pod, g, values.c_str());
      first = false;
    }
  fputs("]}}", f);
  return fclose(f) == 0 ? 0 : 1;
}
