// toon_emu.cpp — the token-parallel TOON kernel body (csrc/json_tp.h) on the CPU warp emulator (tests/hostsim/warp_emu.cpp).
// Built by tools/toon_emu.py; development and test aid, not part of libcfgpu.so.
#include <string.h>

#include <vector>

#include "../mcp_context_forge_b200/csrc/json_tp.h"
#include "../tests/hostsim/warp_emu.h"

// mode 0: the first attempt alone (toon_unit without its retry, as toon_tp_kernel runs it under CF_TOON_NO_HANDOVER)
// mode 1: tokenize, then analyze in resolve mode and emit: the separate resolving pass the kernel used to run over the units the first
//         attempt handed over as mixed list-item arrays (the reference the in-place retry is compared with)
// mode 2: toon_unit with its in-place retry, as toon_tp_kernel runs it
// Returns the TS_* status (7 = handed over; *reason = FB_*), *collectives = the warp collectives the run took, or < 0 when a status
// was not warp-uniform.
extern "C" int toon_emu_unit(const uint8_t* text, uint32_t n, uint8_t* out, uint32_t out_cap, uint32_t* out_len, int report_errors, int order,
                             int mode, uint32_t* reason, unsigned long long* collectives) {
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
  const uint32_t cap = (uint32_t)toks.size();
  int status[32];
  uint32_t olen[32];
  wemu::run_warp([&](uint32_t lane) {
    uint32_t ol = 0;
    if (mode == 1) {
      uint32_t ntok = 0;
      status[lane] = cftp::tokenize(s, n, toks.data(), cap, sh[0], stage, &ntok);
      if (!status[lane]) {
        tpw::sync();
        status[lane] = cftp::toon_tokens<true>(s, toks.data(), ntok, cap, out, out_cap, &ol, sh[0], stage, report_errors != 0);
      }
    } else {
      status[lane] = cftp::toon_unit(s, n, toks.data(), cap, out, out_cap, &ol, sh[0], stage, report_errors != 0, mode == 2);
    }
    olen[lane] = ol;
  }, order & 1);
  for (int i = 1; i < 32; ++i) if (status[i] != status[0] || olen[i] != olen[0]) return -100 - i;
  *out_len = olen[0];
  *reason = (uint32_t)status[0] >> 8;
  *collectives = wemu::collectives();
  return status[0] & 0xFF;
}
