// Test-only: matchLongestPrefix read at chosen endpoints (eppscore_prefix_match) under the sequential execution policy of
// index_emu.cpp.  It walks each request's blocks with the shared lookup and membership code of csrc/prefix_table.cuh
// (table_find, slot_holds), the code prefix_match_kernel runs per lane, so tests/test_prefix_match_cpu.py checks that code
// against the oracle's matchLongestPrefix on the CPU.  The emu_* entry points of index_emu.cpp build the index.
#include "index_emu.cpp"

extern "C" {
// out[r*k + j]: the blocks of request r before its first miss whose set holds endpoints[r*k + j]; 0 outside [0, limit)
void match_emu(void* h, int R, int k, int limit, const uint64_t* hashes, const uint16_t* nh, int stride, const int32_t* endpoints,
               uint16_t* out) {
  Emu* e = static_cast<Emu*>(h);
  for (int r = 0; r < R; r++) {
    uint16_t* o = out + (size_t)r * k;
    const int32_t* eps = endpoints + (size_t)r * k;
    for (int j = 0; j < k; j++) o[j] = 0;
    for (int b = 0; b < nh[r]; b++) {
      uint32_t raw = 0;
      TSlot* s = table_find(e->x, &e->tv, hashes[(size_t)r * stride + b], &raw);
      if (!s) break;
      for (int j = 0; j < k; j++) {
        const uint32_t p = (uint32_t)eps[j];
        if (p < (uint32_t)limit && slot_holds(e->x, &e->tv, s, raw, p)) o[j]++;
      }
    }
  }
}
}
