// toon_emu.cpp — the token-parallel TOON kernel body (csrc/json_tp.h) on the CPU warp emulator (tests/hostsim/warp_emu.cpp), with
// the device's two passes: the first pass, and for a unit it hands over as a mixed list-item array (FB_MIXED_ITEM) the resolving pass
// toon_tp_kernel runs behind it.  Built by tools/toon_emu.py; development and test aid, not part of libcfgpu.so.
#include <string.h>

#include <vector>

#include "../mcp_context_forge_b200/csrc/json_tp.h"
#include "../tests/hostsim/warp_emu.h"

// resolve_mixed: run the pass with that setting.  Returns the TS_* status (7 = handed over; *reason = FB_*), *collectives = the warp
// collectives the run took, or < 0 when a status was not warp-uniform.
extern "C" int toon_emu_unit(const uint8_t* text, uint32_t n, uint8_t* out, uint32_t out_cap, uint32_t* out_len, int report_errors, int order,
                             int resolve_mixed, uint32_t* reason, unsigned long long* collectives) {
  // the kernel reads whole 1 KiB steps on a 16-byte grid: the padding of the device buffers; `order` bits 4.. shift the alignment
  std::vector<uint8_t> buf(64 + n + 2048, 0xFF);
  uint8_t* base = buf.data() + 32;
  base += (16 - ((uintptr_t)base & 15u)) & 15u;
  uint8_t* s = base + (((uint32_t)order >> 4) & 15u);
  memcpy(s, text, n);
  std::vector<cftp::GTok> toks(n / 2 + 64);
  std::vector<cftp::Shared> sh(1);
  std::vector<uint8_t> stage_buf(cftp::STAGE + 64);
  uint8_t* stage = stage_buf.data() + ((16 - ((uintptr_t)stage_buf.data() & 15u)) & 15u);
  int status[32];
  uint32_t olen[32];
  wemu::run_warp([&](uint32_t lane) {
    uint32_t ol = 0;
    status[lane] = cftp::toon_unit(s, n, toks.data(), (uint32_t)toks.size(), out, out_cap, &ol, sh[0], stage, report_errors != 0, resolve_mixed != 0);
    olen[lane] = ol;
  }, order & 1);
  for (int i = 1; i < 32; ++i) if (status[i] != status[0] || olen[i] != olen[0]) return -100 - i;
  *out_len = olen[0];
  *reason = (uint32_t)status[0] >> 8;
  *collectives = wemu::collectives();
  return status[0] & 0xFF;
}
