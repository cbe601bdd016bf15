// NVRTC + cubin cache (rbd_jit.cpp) for a complete source text that some part of the library generated itself (rbd_deriv_jit.cpp).
#pragma once
#include <string>
#include <vector>

namespace rbd {

// Compiles `src` for sm_90a, or fetches the cubin from the cache directory (key = hash of the text, file <hash>_<tag>.cubin).
// fmad = false compiles with --fmad=false.  Returns false with `err` set when NVRTC is unavailable or compilation fails.
bool jit_compile_text(const std::string& tag, const std::string& src, bool fmad, std::vector<char>& cubin, bool compile_if_missing,
                      bool* from_cache, std::string& err);

}  // namespace rbd
