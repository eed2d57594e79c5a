// nvrtc_compile.h — NVRTC front door (sm_90a cubins) and the source hash used as cache key.
#pragma once
#include <cstdint>
#include <string>

namespace hnb_rt {

uint64_t fnv1a64(const std::string& s);

// Compile `source` for sm_90a. On success `cubin` holds the device binary and `log` the (possibly
// empty) compiler log; on failure `log` holds the error text.
// `fast_math`: FMA contraction + approximate division / square root (HNB_EFFECT_FAST_MATH); default is strict IEEE.
bool nvrtc_compile_sm90a(const std::string& source, const std::string& name, std::string& cubin, std::string& log, bool fast_math = false);

}  // namespace hnb_rt
