#pragma once
#include <string>
#include <vector>
#include <cstdint>
#include <unistd.h>

namespace mb2 {

struct JitModule {
    std::vector<char> cubin;
    // nodeKernels[i] is the mangled name of a mwGPU::nodeKern<NodeT>
    // instantiation, nodeMetas[i] the matching mwGPU::nodeMeta<NodeT> global.
    std::vector<std::string> nodeKernels;
    std::vector<std::string> nodeMetas;
    std::string cachePath;
    bool fromCache = false;
};

std::string moduleDir();

// fast_math: FMA contraction on; use_cache: look the cubin up in and store it to cache_dir
bool jitCompile(const std::vector<std::string> &sources,
                const std::vector<std::string> &user_flags,
                int opt_mode, bool fast_math, bool use_cache, const std::string &cache_dir,
                JitModule *out, std::string *err);

}
