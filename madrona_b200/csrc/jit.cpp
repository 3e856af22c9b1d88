// jit.cpp -- compile the simulator's own sources for sm_90a with NVRTC.
//
// Same contract as the reference's MWCudaExecutor constructor
// (src/mw/cuda_exec.cpp:643-1032 compileCode, :1327-1526 buildKernels): the
// caller passes CompileConfig::userSources / userCompileFlags and the engine
// compiles them as *device* code ("-default-device": unannotated functions are
// __device__, exactly as in the reference build, src/mw/CMakeLists.txt:38-47)
// against the device-side Madrona headers.  Differences by design:
//   * all user sources form ONE translation unit (unity build) -> one cubin,
//     no nvJitLink step, whole-program optimisation;
//   * no megakernel is generated: every ParallelForNode instantiation is its
//     own __global__ (mwGPU::nodeKern<NodeT>); they are discovered from the
//     cubin's ELF symbol table rather than by grepping PTX text;
//   * IEEE mode (--fmad=false, precise div/sqrt) so float results match the
//     CPU oracle built with -ffp-contract=off; MADRONA_B200_FAST_MATH=1 opts
//     into contraction.
#include "jit.hpp"

#include <nvrtc.h>
#include <dlfcn.h>
#include <sys/stat.h>
#include <dirent.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <algorithm>

namespace mb2 {

static std::string g_module_dir;

std::string moduleDir()
{
    if (!g_module_dir.empty()) return g_module_dir;
    Dl_info info;
    if (dladdr((void *)&moduleDir, &info) && info.dli_fname) {
        std::string p(info.dli_fname);
        size_t slash = p.rfind('/');
        g_module_dir = slash == std::string::npos ? "." : p.substr(0, slash);
    } else {
        g_module_dir = ".";
    }
    return g_module_dir;
}

static bool readFile(const std::string &path, std::string *out)
{
    std::ifstream f(path, std::ios::binary);
    if (!f) return false;
    std::stringstream ss;
    ss << f.rdbuf();
    *out = ss.str();
    return true;
}

static uint64_t fnv1a(uint64_t h, const void *data, size_t n)
{
    const unsigned char *p = (const unsigned char *)data;
    for (size_t i = 0; i < n; i++) {
        h ^= p[i];
        h *= 0x100000001b3ull;
    }
    return h;
}

static uint64_t hashString(uint64_t h, const std::string &s)
{
    h = fnv1a(h, s.data(), s.size());
    unsigned char sep = 0xff;
    return fnv1a(h, &sep, 1);
}

static void hashDir(uint64_t *h, const std::string &dir)
{
    std::vector<std::string> names;
    if (DIR *d = opendir(dir.c_str())) {
        while (dirent *e = readdir(d)) {
            if (e->d_name[0] == '.') continue;
            names.push_back(e->d_name);
        }
        closedir(d);
    }
    std::sort(names.begin(), names.end());
    for (const std::string &n : names) {
        std::string p = dir + "/" + n;
        struct stat st;
        if (stat(p.c_str(), &st) != 0) continue;
        if (S_ISDIR(st.st_mode)) {
            hashDir(h, p);
        } else {
            std::string body;
            if (readFile(p, &body)) {
                *h = hashString(*h, n);
                *h = hashString(*h, body);
            }
        }
    }
}

// ---- cubin ELF symbol scan -------------------------------------------------

struct Elf64Ehdr {
    unsigned char ident[16];
    uint16_t type, machine;
    uint32_t version;
    uint64_t entry, phoff, shoff;
    uint32_t flags;
    uint16_t ehsize, phentsize, phnum, shentsize, shnum, shstrndx;
};
struct Elf64Shdr {
    uint32_t name, type;
    uint64_t flags, addr, offset, size;
    uint32_t link, info;
    uint64_t addralign, entsize;
};
struct Elf64Sym {
    uint32_t name;
    unsigned char info, other;
    uint16_t shndx;
    uint64_t value, size;
};

static const char kKernPrefix[] = "_ZN7madrona5mwGPU8nodeKernI";
static const char kMetaPrefix[] = "_ZN7madrona5mwGPU8nodeMetaI";

static bool scanCubinSymbols(const std::vector<char> &cubin,
                             std::vector<std::string> *kerns,
                             std::vector<std::string> *metas,
                             std::string *err)
{
    if (cubin.size() < sizeof(Elf64Ehdr) || memcmp(cubin.data(), "\x7f" "ELF", 4) != 0) {
        *err = "JIT output is not an ELF cubin";
        return false;
    }
    Elf64Ehdr eh;
    memcpy(&eh, cubin.data(), sizeof(eh));
    for (uint16_t i = 0; i < eh.shnum; i++) {
        Elf64Shdr sh;
        memcpy(&sh, cubin.data() + eh.shoff + (size_t)i * eh.shentsize, sizeof(sh));
        if (sh.type != 2 /* SHT_SYMTAB */) continue;
        Elf64Shdr str;
        memcpy(&str, cubin.data() + eh.shoff + (size_t)sh.link * eh.shentsize, sizeof(str));
        size_t n = sh.size / sizeof(Elf64Sym);
        for (size_t s = 0; s < n; s++) {
            Elf64Sym sym;
            memcpy(&sym, cubin.data() + sh.offset + s * sizeof(Elf64Sym), sizeof(sym));
            if (sym.name >= str.size) continue;
            const char *name = cubin.data() + str.offset + sym.name;
            int type = sym.info & 0xf;
            if (type == 2 /* FUNC */ && strncmp(name, kKernPrefix, sizeof(kKernPrefix) - 1) == 0) {
                if (std::find(kerns->begin(), kerns->end(), name) == kerns->end())
                    kerns->push_back(name);
            } else if (type == 1 /* OBJECT */ &&
                       strncmp(name, kMetaPrefix, sizeof(kMetaPrefix) - 1) == 0) {
                if (std::find(metas->begin(), metas->end(), name) == metas->end())
                    metas->push_back(name);
            }
        }
    }
    return true;
}

static bool pairKernels(JitModule *m, const std::vector<std::string> &kerns,
                        const std::vector<std::string> &metas, std::string *err)
{
    // kernel  = P_k + X + "EE" + <params>,  meta = P_m + X + "EE"
    const size_t pk = sizeof(kKernPrefix) - 1, pm = sizeof(kMetaPrefix) - 1;
    for (const std::string &k : kerns) {
        std::string found;
        for (const std::string &v : metas) {
            std::string x_ee = v.substr(pm);
            if (k.compare(pk, x_ee.size(), x_ee) == 0) {
                if (x_ee.size() > found.size()) found = v;
            }
        }
        if (found.empty()) {
            *err = "no nodeMeta symbol for kernel " + k +
                   " (is the system function declared static?)";
            return false;
        }
        m->nodeKernels.push_back(k);
        m->nodeMetas.push_back(found);
    }
    return true;
}

// ---- compile ---------------------------------------------------------------

bool jitCompile(const std::vector<std::string> &sources,
                const std::vector<std::string> &user_flags,
                int opt_mode, bool fast_math, bool use_cache, const std::string &cache_dir,
                JitModule *out, std::string *err)
{
    const std::string mod = moduleDir();
    const std::string dev_inc = mod + "/device";
    const std::string std_inc = mod + "/device/std";
    const std::string csrc_inc = mod + "/csrc";
    std::string cuda_inc = "/usr/local/cuda/include";
    if (const char *env = getenv("CUDA_HOME")) cuda_inc = std::string(env) + "/include";

    if (const char *env = getenv("MADRONA_MWGPU_FORCE_DEBUG")) {
        if (env[0] == '1') opt_mode = 2;
    }

    std::vector<std::string> opts = {
        "-arch=sm_90a",
        "-std=c++20",
        "-default-device",
        "-lineinfo",
        "-DMADRONA_GPU_MODE=1",
        "-DMADRONA_MW_MODE=1",
        "-DMADRONA_B200=1",
        "-I" + std_inc,
        "-I" + dev_inc,
        "-I" + csrc_inc,
        "-I" + cuda_inc,
        "--diag-suppress=177,550,20012,20011,3056",
    };
    if (!fast_math) {
        opts.push_back("--fmad=false");
        opts.push_back("--prec-div=true");
        opts.push_back("--prec-sqrt=true");
        opts.push_back("--ftz=false");
    } else {
        opts.push_back("--fmad=true");
    }
    if (opt_mode == 2) {
        opts.push_back("-G");
    }
    for (const std::string &f : user_flags) opts.push_back(f);

    // unity translation unit
    std::string unity =
        "#include <madrona/state.hpp>\n"
        "extern \"C\" { __constant__ mb2::EngineState *mb2_engine_state; }\n";
    for (const std::string &s : sources) unity += "#include \"" + s + "\"\n";

    // ---- cache lookup
    uint64_t h = 0xcbf29ce484222325ull;
    int nv_major = 0, nv_minor = 0;
    nvrtcVersion(&nv_major, &nv_minor);
    h = fnv1a(h, &nv_major, sizeof(nv_major));
    h = fnv1a(h, &nv_minor, sizeof(nv_minor));
    for (const std::string &o : opts) {
        // include paths are machine specific; hash their contents instead
        if (o.rfind("-I", 0) == 0) continue;
        h = hashString(h, o);
    }
    for (const std::string &s : sources) {
        std::string body;
        if (!readFile(s, &body)) {
            *err = "cannot read user source " + s;
            return false;
        }
        size_t slash = s.rfind('/');
        h = hashString(h, slash == std::string::npos ? s : s.substr(slash + 1));
        h = hashString(h, body);
        // sibling headers of the source (sim.hpp next to sim.cpp)
        if (slash != std::string::npos) hashDir(&h, s.substr(0, slash));
    }
    hashDir(&h, dev_inc);
    {
        std::string body;
        if (readFile(csrc_inc + "/mb2_state.h", &body)) h = hashString(h, body);
        if (readFile(csrc_inc + "/physics_state.h", &body)) h = hashString(h, body);
        if (readFile(csrc_inc + "/render_state.h", &body)) h = hashString(h, body);
    }
    for (const std::string &f : user_flags) {
        if (f.rfind("-I", 0) == 0) hashDir(&h, f.substr(2));
    }

    char hex[32];
    snprintf(hex, sizeof(hex), "%016llx", (unsigned long long)h);
    const std::string cache_path = cache_dir + "/" + hex + ".cubin";
    out->cachePath = cache_path;

    std::string cached;
    if (use_cache && readFile(cache_path, &cached) && !cached.empty()) {
        out->cubin.assign(cached.begin(), cached.end());
        out->fromCache = true;
    } else {
        nvrtcProgram prog;
        nvrtcResult r = nvrtcCreateProgram(&prog, unity.c_str(), "mb2_unity.cu",
                                           0, nullptr, nullptr);
        if (r != NVRTC_SUCCESS) {
            *err = std::string("nvrtcCreateProgram: ") + nvrtcGetErrorString(r);
            return false;
        }
        std::vector<const char *> copts;
        for (const std::string &o : opts) copts.push_back(o.c_str());
        r = nvrtcCompileProgram(prog, (int)copts.size(), copts.data());
        size_t log_size = 0;
        nvrtcGetProgramLogSize(prog, &log_size);
        std::string log(log_size, '\0');
        if (log_size > 1) nvrtcGetProgramLog(prog, log.data());
        if (r != NVRTC_SUCCESS) {
            *err = std::string("NVRTC compile failed: ") + nvrtcGetErrorString(r) +
                   "\n" + log;
            nvrtcDestroyProgram(&prog);
            return false;
        }
        if (getenv("MADRONA_MWGPU_VERBOSE_COMPILE") && log_size > 1) {
            fprintf(stderr, "%s\n", log.c_str());
        }
        size_t cubin_size = 0;
        r = nvrtcGetCUBINSize(prog, &cubin_size);
        if (r != NVRTC_SUCCESS || cubin_size == 0) {
            *err = "NVRTC produced no cubin";
            nvrtcDestroyProgram(&prog);
            return false;
        }
        out->cubin.resize(cubin_size);
        nvrtcGetCUBIN(prog, out->cubin.data());
        nvrtcDestroyProgram(&prog);
        out->fromCache = false;

        if (use_cache) {
            mkdir(cache_dir.c_str(), 0755);
            std::string tmp = cache_path + ".tmp" + std::to_string((long)getpid());
            std::ofstream f(tmp, std::ios::binary);
            if (f) {
                f.write(out->cubin.data(), (std::streamsize)out->cubin.size());
                f.close();
                rename(tmp.c_str(), cache_path.c_str());
            }
        }
    }

    std::vector<std::string> kerns, metas;
    if (!scanCubinSymbols(out->cubin, &kerns, &metas, err)) return false;
    return pairKernels(out, kerns, metas, err);
}

}
