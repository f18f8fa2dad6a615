// Error reporting + device queries shared by every translation unit of libdvd_b200.so.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>

namespace dvd {

static thread_local char g_err[512] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("DVD_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

int num_sms() {
  static int cached[16] = {0};     // per device
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return 148;
  if (cached[dev] > 0) return cached[dev];
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) {
    cached[dev] = n;
    return n;
  }
  return 132;  // H100 SXM
}

}  // namespace dvd

extern "C" const char* dvd_last_error(void) { return dvd::g_err; }
extern "C" int dvd_version(void) { return 103; }
/* sizes of the structs that cross the C ABI by pointer (which: 0 dvd_loss_cfg, 1 dvd_mlp_cfg, 2 dvd_conv_desc, 3 dvd_pack_item,
 * 4 dvd_vis_panel, 5 dvd_vis_map): a binding in another language checks its own layout against these */
extern "C" long dvd_struct_size(int which) {
  switch (which) {
    case 0: return (long)sizeof(dvd_loss_cfg);
    case 1: return (long)sizeof(dvd_mlp_cfg);
    case 2: return (long)sizeof(dvd_conv_desc);
    case 3: return (long)sizeof(dvd_pack_item);
    case 4: return (long)sizeof(dvd_vis_panel);
    case 5: return (long)sizeof(dvd_vis_map);
    default: return -1;
  }
}
