// nvrtc_compile.cpp — run-time compilation of generated effect kernels for sm_90a.
// ≙ the naga WGSL->SPIR-V step behind wgpu's create_shader_module in the reference; the result is a
// cubin (not PTX) so no driver JIT is involved at load time.
#include "nvrtc_compile.h"

#include <nvrtc.h>

#include <vector>

namespace hnb_rt {

uint64_t fnv1a64(const std::string& s) {
    uint64_t h = 0xcbf29ce484222325ull;
    for (unsigned char c : s) {
        h ^= c;
        h *= 0x100000001b3ull;
    }
    return h;
}

bool nvrtc_compile_sm90a(const std::string& source, const std::string& name, std::string& cubin, std::string& log, bool fast_math) {
    nvrtcProgram prog = nullptr;
    nvrtcResult r = nvrtcCreateProgram(&prog, source.c_str(), name.c_str(), 0, nullptr, nullptr);
    if (r != NVRTC_SUCCESS) {
        log = std::string("nvrtcCreateProgram: ") + nvrtcGetErrorString(r);
        return false;
    }
    // -fmad=false: no FMA contraction, so add/mul sequences are bit-exact with the CPU oracle
    // (SURVEY.md §7 "fp parity"). No fast-math: IEEE division and square root.
    // HNB_EFFECT_FAST_MATH: contraction and approximate div/sqrt, but NOT --use_fast_math (its sin/cos/exp
    // intrinsics have absolute, not relative, error bounds and would break the 1e-5 relative tolerance).
    std::vector<const char*> opts = {"-arch=sm_90a", "-std=c++17", "-lineinfo", "-default-device", "-diag-suppress=550", "-diag-suppress=177",
                                     "--ptxas-options=-v"};
    if (fast_math) {
        opts.push_back("-fmad=true");
        opts.push_back("-prec-div=false");
        opts.push_back("-prec-sqrt=false");
    } else {
        opts.push_back("-fmad=false");
    }
    r = nvrtcCompileProgram(prog, (int)opts.size(), opts.data());
    size_t log_size = 0;
    nvrtcGetProgramLogSize(prog, &log_size);
    if (log_size > 1) {
        std::vector<char> buf(log_size + 1, 0);
        nvrtcGetProgramLog(prog, buf.data());
        log.assign(buf.data());
    }
    if (r != NVRTC_SUCCESS) {
        log = std::string("nvrtcCompileProgram: ") + nvrtcGetErrorString(r) + "\n" + log;
        nvrtcDestroyProgram(&prog);
        return false;
    }
    size_t sz = 0;
    r = nvrtcGetCUBINSize(prog, &sz);
    if (r != NVRTC_SUCCESS || sz == 0) {
        log = std::string("nvrtcGetCUBINSize: ") + nvrtcGetErrorString(r);
        nvrtcDestroyProgram(&prog);
        return false;
    }
    cubin.resize(sz);
    r = nvrtcGetCUBIN(prog, &cubin[0]);
    nvrtcDestroyProgram(&prog);
    if (r != NVRTC_SUCCESS) {
        log = std::string("nvrtcGetCUBIN: ") + nvrtcGetErrorString(r);
        return false;
    }
    return true;
}

}  // namespace hnb_rt
