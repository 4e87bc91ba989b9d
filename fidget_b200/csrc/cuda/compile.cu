// Compiled tapes (include/fidget_cuda.h, fc_tape_compile): one tape turned into straight-line sm_90a kernels for the
// three bulk evaluators, compiled at run time with NVRTC and loaded with the runtime's library API.
//
// Bit identity with the interpreters rests on three things, all kept here:
//  * NVRTC compiles the project's own dev_ops.cuh (embedded into the library at build time), so every clause runs the
//    same arithmetic the interpreters run;
//  * the NVRTC options carry build.sh's numeric flags (no FMA contraction, IEEE division and square root, denormals);
//  * each (opcode, form) maps to the dev_ops call the interpreter's handler for it makes (k_map below).
// Two things the interpreters never let the optimiser see stay hidden from it here as well: immediates are read from a
// __constant__ table of bit patterns (a literal 1.0 would let `x * 1.0` fold to `x`, which keeps a NaN payload the
// multiplication would have replaced), and every clause result passes an empty asm statement, so no later clause can
// fold against what an earlier one produced (the zero partials of gr1(), the equal bounds of iv1()).
#include <dlfcn.h>
#include <link.h>
#include <nvrtc.h>
#include <sys/stat.h>

#include <chrono>

#include "capi_internal.h"

extern const char k_dev_ops_source[];   // dev_ops.cuh as text (dev_ops_src.cc, written by build.sh)

namespace {

// ---- NVRTC, opened on first use --------------------------------------------------------------------------------------
struct Nvrtc {
    decltype(&::nvrtcVersion) version = nullptr;
    decltype(&::nvrtcCreateProgram) create = nullptr;
    decltype(&::nvrtcCompileProgram) compile = nullptr;
    decltype(&::nvrtcGetProgramLogSize) log_size = nullptr;
    decltype(&::nvrtcGetProgramLog) log = nullptr;
    decltype(&::nvrtcGetCUBINSize) cubin_size = nullptr;
    decltype(&::nvrtcGetCUBIN) cubin = nullptr;
    decltype(&::nvrtcDestroyProgram) destroy = nullptr;
    decltype(&::nvrtcGetErrorString) error = nullptr;
    uint32_t ver = 0;   // major * 1000 + minor * 10
    std::string failure;
};

bool is_dir(const std::string& p) {
    struct stat st;
    return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}

// FIDGET_B200_NVRTC (a file or the directory holding it, and then nothing else); else libnvrtc.so.12 by soname; else
// $CUDA_HOME/lib64 (default /usr/local/cuda)
const Nvrtc& nvrtc() {
    static Nvrtc n;
    static std::once_flag once;
    std::call_once(once, [] {
        std::vector<std::string> tried;
        void* h = nullptr;
        auto open = [&](const std::string& p) {
            tried.push_back(p);
            if (!h) h = dlopen(p.c_str(), RTLD_NOW | RTLD_LOCAL);
        };
        const char* env = getenv("FIDGET_B200_NVRTC");
        if (env && *env) {
            const std::string p(env);
            if (is_dir(p)) { open(p + "/libnvrtc.so.12"); open(p + "/libnvrtc.so"); }
            else open(p);
        } else {
            open("libnvrtc.so.12");
            const char* home = getenv("CUDA_HOME");
            const std::string lib = std::string(home && *home ? home : "/usr/local/cuda") + "/lib64/";
            open(lib + "libnvrtc.so.12");
            open(lib + "libnvrtc.so");
        }
        if (!h) {
            n.failure = "NVRTC could not be loaded; looked for";
            for (auto& t : tried) n.failure += " " + t;
            n.failure += env && *env ? " (FIDGET_B200_NVRTC)" : "; set FIDGET_B200_NVRTC to its path";
            return;
        }
#define FC_SYM(field, name) n.field = reinterpret_cast<decltype(n.field)>(dlsym(h, name))
        FC_SYM(version, "nvrtcVersion");
        FC_SYM(create, "nvrtcCreateProgram");
        FC_SYM(compile, "nvrtcCompileProgram");
        FC_SYM(log_size, "nvrtcGetProgramLogSize");
        FC_SYM(log, "nvrtcGetProgramLog");
        FC_SYM(cubin_size, "nvrtcGetCUBINSize");
        FC_SYM(cubin, "nvrtcGetCUBIN");
        FC_SYM(destroy, "nvrtcDestroyProgram");
        FC_SYM(error, "nvrtcGetErrorString");
#undef FC_SYM
        if (!n.version || !n.create || !n.compile || !n.log_size || !n.log || !n.cubin_size || !n.cubin || !n.destroy ||
            !n.error) {
            n.failure = "NVRTC at " + tried.back() + " lacks an entry point (cubin output needs NVRTC 11.1 or later)";
            n.version = nullptr;
            return;
        }
        int major = 0, minor = 0;
        n.version(&major, &minor);
        n.ver = uint32_t(major * 1000 + minor * 10);
        // NVRTC opens libnvrtc-builtins.so.<major>.<minor> by soname at its first compile; a copy without a runpath to
        // its own directory (the CUDA toolkit's) would not find it, so load it from beside libnvrtc first
        struct link_map* lm = nullptr;
        if (dlinfo(h, RTLD_DI_LINKMAP, &lm) == 0 && lm && lm->l_name) {
            std::string dir(lm->l_name);
            const size_t slash = dir.rfind('/');
            if (slash != std::string::npos) {
                dir.resize(slash);
                dlopen((dir + "/libnvrtc-builtins.so." + std::to_string(major) + "." + std::to_string(minor)).c_str(),
                       RTLD_NOW | RTLD_GLOBAL);
            }
        }
    });
    return n;
}

// ---- source generation ----------------------------------------------------------------------------------------------
enum Kind : int { K_FLOAT = 0, K_GRAD = 1, K_INTERVAL = 2 };
const char* const k_kernel_name[3] = {"fc_compiled_f32", "fc_compiled_grad", "fc_compiled_interval"};

const char* const k_op_name[OP_COUNT] = {
    "OP_OUTPUT", "OP_INPUT", "OP_COPY", "OP_NEG", "OP_ABS", "OP_RECIP", "OP_SQRT", "OP_SQUARE", "OP_FLOOR", "OP_CEIL",
    "OP_ROUND", "OP_NOT", "OP_RAND", "OP_SIN", "OP_COS", "OP_TAN", "OP_ASIN", "OP_ACOS", "OP_ATAN", "OP_EXP", "OP_LN",
    "OP_ADD", "OP_SUB", "OP_MUL", "OP_DIV", "OP_ATAN2", "OP_COMPARE", "OP_MIX", "OP_MOD", "OP_MIN", "OP_MAX", "OP_AND",
    "OP_OR", "OP_MEM"};

// (opcode, form) -> the dev_ops call of the interpreter behind each kind: k_float_slice (f32), k_grad_slice (grad) and
// run_interval's handlers (interval).  $a / $b are the operands (a register, or the immediate as the kind's value),
// $k the bare f32 immediate, $o the opcode.  A unary opcode's row is its F_RR form.  Rows not listed take the default
// of their class: f32_unary / f32_binary, gr_unary / gr_binary, iv_unary / iv_binary (iv_choice_op for min / max /
// and / or, which also yield the choice).
struct MapRow {
    uint32_t op, form;
    const char *f32, *grad, *itv;
};
const MapRow k_map[] = {
    {OP_ADD, F_RR, nullptr, "gr_add($a, $b)", "iv_add($a, $b)"},
    {OP_ADD, F_RI, nullptr, "gr_add($a, $b)", "iv_add($a, $b)"},
    {OP_ADD, F_IR, nullptr, "gr_add($a, $b)", "iv_add($a, $b)"},
    {OP_SUB, F_RR, nullptr, "gr_sub($a, $b)", "iv_sub($a, $b)"},
    {OP_SUB, F_RI, nullptr, "gr_sub($a, $b)", "iv_sub($a, $b)"},
    {OP_SUB, F_IR, nullptr, "gr_sub($a, $b)", "iv_sub($a, $b)"},
    {OP_MUL, F_RR, nullptr, "gr_mul($a, $b)", "iv_mul($a, $b)"},
    {OP_MUL, F_RI, nullptr, "gr_mul_f($a, $k)", "iv_mul_f($a, $k)"},
    {OP_MUL, F_IR, nullptr, "gr_mul($a, $b)", "iv_mul($a, $b)"},
    {OP_DIV, F_RR, nullptr, "gr_div($a, $b)", nullptr},
    {OP_DIV, F_RI, nullptr, "gr_div($a, $b)", nullptr},
    {OP_DIV, F_IR, nullptr, "gr_div($a, $b)", nullptr},
    {OP_NEG, F_RR, nullptr, "gr_neg($a)", "iv_neg($a)"},
    {OP_ABS, F_RR, nullptr, nullptr, "iv_abs($a)"},
    {OP_SQRT, F_RR, nullptr, nullptr, "iv_sqrt($a)"},
    {OP_SQUARE, F_RR, nullptr, "gr_mul($a, $a)", "iv_square($a)"},
};

std::string map_call(int kind, uint32_t op, uint32_t form) {
    for (const MapRow& r : k_map)
        if (r.op == op && r.form == form) {
            const char* s = kind == K_FLOAT ? r.f32 : kind == K_GRAD ? r.grad : r.itv;
            if (s) return s;
        }
    static const char* const unary[3] = {"f32_unary($o, $a)", "gr_unary($o, $a)", "iv_unary($o, $a)"};
    static const char* const binary[3] = {"f32_binary($o, $a, $b)", "gr_binary($o, $a, $b)", "iv_binary($o, $a, $b)"};
    if (kind == K_INTERVAL && op_is_choice(op)) return "iv_choice_op($o, $a, $b, c)";
    return op_is_unary(op) ? unary[kind] : binary[kind];
}

std::string subst(std::string s, const std::string& a, const std::string& b, const std::string& k, const char* o) {
    auto rep = [&](const char* key, const std::string& v) {
        for (size_t at = s.find(key); at != std::string::npos; at = s.find(key, at + v.size())) s.replace(at, 2, v);
    };
    rep("$a", a);
    rep("$b", b);
    rep("$k", k);
    rep("$o", o);
    return s;
}

// Shared by every kind: parameter structs laid out as BulkParams / TracingParams (kernels.cuh), the immediates and the
// optimisation barrier.
const char k_prelude[] = R"(#include "dev_ops.cuh"
using namespace fdev;
struct BulkParams { const uint2* tape; uint32_t n_ops, n_vars, n_outputs, n_slots; uint64_t n; const void* const* vars; void* const* outs; };
struct TracingParams { const uint2* tape; uint32_t n_ops, n_vars, n_outputs, n_choices, n_slots; uint64_t n; const float* vars; float* out; uint8_t* choices; uint8_t* simplify; };
__constant__ float fc_zero = 0.0f;
#define KF(i) __uint_as_float(fc_imm[i])
#define KG(i) make_float4(KF(i), fc_zero, fc_zero, fc_zero)   // gr1(imm), its zeros as opaque as the interpreters'
FD float opq(float v) { asm("" : "+f"(v)); return v; }
FD float2 opq(float2 v) { asm("" : "+f"(v.x), "+f"(v.y)); return v; }
FD float4 opq(float4 v) { asm("" : "+f"(v.x), "+f"(v.y), "+f"(v.z), "+f"(v.w)); return v; }
)";

constexpr uint32_t COMPILED_THREADS = 128;

void gen_kernel(int kind, const std::vector<uint2>& cl, uint32_t n_vars, uint32_t n_outputs,
                const std::vector<uint32_t>& imm_index, std::string& s) {
    static const char* const type[3] = {"float", "float4", "float2"};
    const char* T = type[kind];
    std::vector<bool> reg(256, false), in(n_vars, false), out(n_outputs, false);
    std::vector<uint32_t> mems;
    for (const uint2& c : cl) {
        const uint32_t op = (c.x & 0xff) >> 2, form = c.x & 3, o = (c.x >> 8) & 0xff, l = (c.x >> 16) & 0xff, r = c.x >> 24;
        if (op == OP_OUTPUT) { reg[l] = true; out[c.y] = true; continue; }
        if (op == OP_INPUT) in[c.y] = true;
        if (op == OP_MEM) { if (std::find(mems.begin(), mems.end(), c.y) == mems.end()) mems.push_back(c.y); }
        if (o != 0xff) reg[o] = true;
        if (l != 0xff && !(op_is_binary(op) && form == F_IR)) reg[l] = true;
        if (r != 0xff && op_is_binary(op) && form != F_RI) reg[r] = true;
    }
    char buf[160];
    s += "extern \"C\" __global__ void __launch_bounds__(" + std::to_string(COMPILED_THREADS) + ") ";
    s += k_kernel_name[kind];
    s += kind == K_INTERVAL ? "(const __grid_constant__ TracingParams p) {\n" : "(const __grid_constant__ BulkParams p) {\n";
    if (kind != K_INTERVAL) {
        for (uint32_t i = 0; i < n_vars; ++i)
            if (in[i]) { snprintf(buf, sizeof buf, "  const %s* __restrict__ in%u = (const %s*)p.vars[%u];\n", T, i, T, i); s += buf; }
        for (uint32_t o = 0; o < n_outputs; ++o)
            if (out[o]) { snprintf(buf, sizeof buf, "  %s* __restrict__ out%u = (%s*)p.outs[%u];\n", T, o, T, o); s += buf; }
    }
    s += "  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;\n"
         "  for (uint64_t idx = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < p.n; idx += stride) {\n";
    if (kind == K_INTERVAL) {
        snprintf(buf, sizeof buf, "    const float* v = p.vars + idx * %uu;\n    float* o = p.out + idx * %uu;\n", n_vars * 2,
                 n_outputs * 2);
        s += buf;
        s += "    uint8_t* ch = p.choices ? p.choices + idx * p.n_choices : nullptr;\n    bool any = false;\n";
    }
    const char* zero = kind == K_FLOAT ? "0.0f" : kind == K_GRAD ? "make_float4(0.0f, 0.0f, 0.0f, 0.0f)" : "make_float2(0.0f, 0.0f)";
    for (uint32_t k = 0; k < 256; ++k)
        if (reg[k]) { snprintf(buf, sizeof buf, "    %s r%u = %s;\n", T, k, zero); s += buf; }
    for (uint32_t m : mems) { snprintf(buf, sizeof buf, "    %s m%u = %s;\n", T, m, zero); s += buf; }
    uint32_t n_choice = 0;
    for (size_t i = 0; i < cl.size(); ++i) {
        const uint2 c = cl[i];
        const uint32_t op = (c.x & 0xff) >> 2, form = c.x & 3, o = (c.x >> 8) & 0xff, l = (c.x >> 16) & 0xff, r = c.x >> 24;
        char kf[32], imm[48];
        snprintf(kf, sizeof kf, "KF(%u)", imm_index[i]);
        if (kind == K_FLOAT) snprintf(imm, sizeof imm, "%s", kf);
        else if (kind == K_GRAD) snprintf(imm, sizeof imm, "KG(%u)", imm_index[i]);
        else snprintf(imm, sizeof imm, "iv1(%s)", kf);
        const std::string R = "r" + std::to_string(o), L = "r" + std::to_string(l), Rr = "r" + std::to_string(r);
        if (op == OP_OUTPUT) {
            if (kind == K_INTERVAL) snprintf(buf, sizeof buf, "    o[%u] = %s.x; o[%u] = %s.y;\n", 2 * c.y, L.c_str(), 2 * c.y + 1, L.c_str());
            else snprintf(buf, sizeof buf, "    out%u[idx] = %s;\n", c.y, L.c_str());
            s += buf;
        } else if (op == OP_INPUT) {
            if (kind == K_INTERVAL) snprintf(buf, sizeof buf, "    %s = iv(v[%u], v[%u]);\n", R.c_str(), 2 * c.y, 2 * c.y + 1);
            else snprintf(buf, sizeof buf, "    %s = in%u[idx];\n", R.c_str(), c.y);
            s += buf;
        } else if (op == OP_COPY) {
            s += "    " + R + " = " + (form == F_RI ? std::string(imm) : L) + ";\n";
        } else if (op == OP_MEM) {
            const std::string M = "m" + std::to_string(c.y);
            s += form == F_RI ? "    " + R + " = " + M + ";\n" : "    " + M + " = " + L + ";\n";
        } else {
            const std::string a = form == F_IR ? std::string(imm) : L, b = form == F_RI ? std::string(imm) : Rr;
            const std::string call = subst(map_call(kind, op, form), a, b, kf, k_op_name[op]);
            if (kind == K_INTERVAL && op_is_choice(op)) {
                snprintf(buf, sizeof buf, " if (ch) ch[%u] = uint8_t(c); any |= c != 3u; }\n", n_choice++);
                s += "    { uint32_t c; " + R + " = opq(" + call + ");" + buf;
            } else {
                s += "    " + R + " = opq(" + call + ");\n";
            }
        }
    }
    if (kind == K_INTERVAL) s += "    if (p.simplify) p.simplify[idx] = any ? 1 : 0;\n";
    s += "  }\n}\n";
}

// One source per kind: the prelude, the immediates of the tape (distinct bit patterns), the kernel
std::string gen_source(int kind, const std::vector<uint2>& cl, uint32_t n_vars, uint32_t n_outputs) {
    std::vector<uint32_t> bits, index(cl.size(), 0);
    for (size_t i = 0; i < cl.size(); ++i) {
        const uint32_t op = (cl[i].x & 0xff) >> 2, form = cl[i].x & 3;
        const bool has_imm = (op == OP_COPY && form == F_RI) || (op_is_binary(op) && (form == F_RI || form == F_IR));
        if (!has_imm) continue;
        auto at = std::find(bits.begin(), bits.end(), cl[i].y);
        index[i] = uint32_t(at - bits.begin());
        if (at == bits.end()) bits.push_back(cl[i].y);
    }
    std::string s = k_prelude;
    // 64 KiB of constant bank per module: larger tables go to global memory (still opaque to the optimiser)
    s += bits.size() <= 16000 ? "__constant__" : "__device__";
    s += " uint32_t fc_imm[" + std::to_string(std::max<size_t>(bits.size(), 1)) + "] = {";
    char buf[16];
    for (size_t i = 0; i < bits.size(); ++i) {
        snprintf(buf, sizeof buf, "%s%s0x%08xu", i ? "," : "", i % 8 ? " " : "\n  ", bits[i]);
        s += buf;
    }
    s += bits.empty() ? "0u};\n" : "};\n";
    gen_kernel(kind, cl, n_vars, n_outputs, index, s);
    return s;
}

// ---- cubin attributes -----------------------------------------------------------------------------------------------
// The module-wide .nv.info section lists, per kernel symbol (sh_info of the kernel's .text section), its register count
// (EIATTR_REGCOUNT, 0x2f) and its stack frame, which holds the spills (EIATTR_FRAME_SIZE, 0x11): {symbol, value}
void cubin_attrs(const std::vector<char>& cubin, const char* kernel, uint32_t& regs, uint32_t& local) {
    regs = local = 0;
    if (cubin.size() < sizeof(Elf64_Ehdr)) return;
    const auto* eh = reinterpret_cast<const Elf64_Ehdr*>(cubin.data());
    if (memcmp(eh->e_ident, ELFMAG, SELFMAG) != 0 || eh->e_ident[EI_CLASS] != ELFCLASS64) return;
    if (eh->e_shoff + size_t(eh->e_shnum) * sizeof(Elf64_Shdr) > cubin.size() || eh->e_shstrndx >= eh->e_shnum) return;
    const auto* sh = reinterpret_cast<const Elf64_Shdr*>(cubin.data() + eh->e_shoff);
    const char* names = cubin.data() + sh[eh->e_shstrndx].sh_offset;
    const std::string text = std::string(".text.") + kernel;
    int64_t sym = -1;
    const Elf64_Shdr* info = nullptr;
    for (int i = 0; i < eh->e_shnum; ++i) {
        const char* name = names + sh[i].sh_name;
        if (text == name) sym = sh[i].sh_info;
        if (!strcmp(name, ".nv.info") && sh[i].sh_offset + sh[i].sh_size <= cubin.size()) info = &sh[i];
    }
    if (sym < 0 || !info) return;
    const uint8_t* q = reinterpret_cast<const uint8_t*>(cubin.data()) + info->sh_offset;
    const uint8_t* end = q + info->sh_size;
    while (q + 4 <= end) {
        const uint8_t fmt = q[0], attr = q[1];
        uint16_t size;
        memcpy(&size, q + 2, 2);
        q += 4;
        if (fmt != 0x04) continue;   // only EIFMT_SVAL entries carry a payload after the size
        uint32_t kv[2];
        if (size == 8 && q + 8 <= end) {
            memcpy(kv, q, 8);
            if (kv[0] == sym && attr == 0x2f) regs = kv[1];
            if (kv[0] == sym && attr == 0x11) local = kv[1];
        }
        q += size;
    }
}

int32_t compile_kind(int kind, const std::vector<uint2>& cl, uint32_t n_vars, uint32_t n_outputs, std::string& src,
                     std::vector<char>& cubin, float& ms) {
    const Nvrtc& n = nvrtc();
    if (!n.version) return fail(FC_ERR_UNSUPPORTED, n.failure);
    const auto t0 = std::chrono::steady_clock::now();
    src = gen_source(kind, cl, n_vars, n_outputs);
    nvrtcProgram prog = nullptr;
    const char* hdr[1] = {k_dev_ops_source};
    const char* hdr_name[1] = {"dev_ops.cuh"};
    nvrtcResult r = n.create(&prog, src.c_str(), "fc_compiled.cu", 1, hdr, hdr_name);
    if (r != NVRTC_SUCCESS) return fail(FC_ERR_INVALID, std::string("nvrtcCreateProgram: ") + n.error(r));
    // build.sh's numeric flags: the interpreters are compiled with exactly these
    const char* opts[] = {"-arch=sm_90a", "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false"};
    r = n.compile(prog, int(sizeof opts / sizeof opts[0]), opts);
    if (r != NVRTC_SUCCESS) {
        size_t len = 0;
        n.log_size(prog, &len);
        std::string log(len, '\0');
        if (len) n.log(prog, &log[0]);
        n.destroy(&prog);
        return fail(FC_ERR_INVALID, std::string("NVRTC: ") + n.error(r) + ": " + log.c_str());
    }
    size_t size = 0;
    n.cubin_size(prog, &size);
    cubin.resize(size);
    if (size) n.cubin(prog, cubin.data());
    n.destroy(&prog);
    ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return FC_OK;
}

int32_t compile_all(const std::vector<uint2>& cl, uint32_t n_vars, uint32_t n_outputs, uint32_t kinds,
                    fc_compiled_info& info, std::vector<char> (&cubins)[3], std::string* source) {
    if (kinds == 0 || (kinds & ~(FC_COMPILE_FLOAT | FC_COMPILE_GRAD | FC_COMPILE_INTERVAL)))
        return fail(FC_ERR_INVALID, "kinds: a non-empty set of FC_COMPILE_FLOAT | FC_COMPILE_GRAD | FC_COMPILE_INTERVAL");
    info = fc_compiled_info{};
    for (int k = 0; k < 3; ++k) {
        if (!(kinds & (1u << k))) continue;
        std::string src;
        if (int32_t rc = compile_kind(k, cl, n_vars, n_outputs, src, cubins[k], info.compile_ms[k])) return rc;
        cubin_attrs(cubins[k], k_kernel_name[k], info.regs[k], info.local_bytes[k]);
        info.cubin_bytes += cubins[k].size();
        if (source) *source += src;
    }
    info.kinds = kinds;
    info.nvrtc_version = nvrtc().ver;
    return FC_OK;
}

}  // namespace

struct fc_compiled {
    fc_ctx* ctx = nullptr;
    fc_tape* tape = nullptr;
    cudaLibrary_t lib[3] = {};
    cudaKernel_t kernel[3] = {};
    unsigned grid_per_sm[3] = {};
    fc_compiled_info info{};
};

namespace {

// Grid: one point per thread in a grid-stride loop, as many blocks per SM as the kernel's registers let be resident
unsigned compiled_grid(const fc_compiled* c, int kind, uint64_t n) {
    const uint64_t blocks = (n + COMPILED_THREADS - 1) / COMPILED_THREADS;
    return unsigned(std::max<uint64_t>(1, std::min<uint64_t>(blocks, uint64_t(c->ctx->sm_count) * c->grid_per_sm[kind])));
}

int32_t launch_compiled(const fc_compiled* c, int kind, uint64_t n, void* params) {
    if (!n) return FC_OK;
    void* args[1] = {params};
    CU(cudaLaunchKernel(reinterpret_cast<const void*>(c->kernel[kind]), dim3(compiled_grid(c, kind, n)),
                        dim3(COMPILED_THREADS), args, 0, c->ctx->stream));
    return FC_OK;
}

int32_t check_kind(fc_eval* e, const fc_compiled* c, int kind) {
    if (!e || !c) return fail(FC_ERR_INVALID, "null argument");
    if (e->ctx != c->ctx) return fail(FC_ERR_INVALID, "the evaluator and the compiled tape belong to different contexts");
    if (!(c->info.kinds & (1u << kind)))
        return fail(FC_ERR_INVALID, std::string("this tape was not compiled for ") + k_kernel_name[kind]);
    return FC_OK;
}

}  // namespace

extern "C" {

int32_t fc_compile_check(const uint32_t* words, size_t n_words, uint8_t reg_count, uint32_t mem_count, uint32_t n_vars,
                         uint32_t n_outputs, uint32_t kinds, char* source, size_t cap, size_t* n_source,
                         fc_compiled_info* info) {
    if (!info) return fail(FC_ERR_INVALID, "null info");
    std::vector<uint2> cl;
    uint32_t nch = 0;
    if (int32_t rc = transcode(words, n_words, reg_count, mem_count, n_vars, n_outputs, cl, nch)) return rc;
    std::vector<char> cubins[3];
    std::string src;
    if (int32_t rc = compile_all(cl, n_vars, n_outputs, kinds, *info, cubins, &src)) return rc;
    if (n_source) *n_source = src.size();
    if (source && cap) {
        const size_t k = std::min(cap - 1, src.size());
        memcpy(source, src.data(), k);
        source[k] = '\0';
    }
    return FC_OK;
}

int32_t fc_tape_compile(fc_ctx* ctx, const fc_tape* tape, uint32_t kinds, fc_compiled** out) {
    if (!ctx || !tape || !out) return fail(FC_ERR_INVALID, "null argument");
    if (tape->ctx != ctx) return fail(FC_ERR_INVALID, "the tape belongs to another context");
    fc_compiled_info info{};
    std::vector<char> cubins[3];
    if (int32_t rc = compile_all(tape->host, tape->info.n_vars, tape->info.n_outputs, kinds, info, cubins, nullptr)) return rc;
    CU(cudaSetDevice(ctx->device));
    fc_compiled* c = new fc_compiled();
    c->ctx = ctx;
    c->info = info;
    for (int k = 0; k < 3; ++k) {
        if (!(kinds & (1u << k))) continue;
        cudaError_t e = cudaLibraryLoadData(&c->lib[k], cubins[k].data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
        if (e == cudaSuccess) e = cudaLibraryGetKernel(&c->kernel[k], c->lib[k], k_kernel_name[k]);
        if (e != cudaSuccess) {
            for (auto l : c->lib) if (l) cudaLibraryUnload(l);
            delete c;
            return fail(FC_ERR_CUDA, std::string("loading ") + k_kernel_name[k] + ": " + cudaGetErrorString(e));
        }
        // resident blocks per SM from the register file (64 K registers, allocated per warp in units of 256)
        const uint32_t per_warp = ((std::max(info.regs[k], 1u) * 32 + 255) / 256) * 256;
        c->grid_per_sm[k] = std::max(1u, std::min(16u, 65536u / (per_warp * (COMPILED_THREADS / 32))));
    }
    fc_tape_retain(const_cast<fc_tape*>(tape));
    c->tape = const_cast<fc_tape*>(tape);
    *out = c;
    return FC_OK;
}

int32_t fc_compiled_get_info(const fc_compiled* c, fc_compiled_info* info) {
    if (!c || !info) return fail(FC_ERR_INVALID, "null argument");
    *info = c->info;
    return FC_OK;
}

int32_t fc_compiled_release(fc_compiled* c) {
    if (!c) return fail(FC_ERR_INVALID, "null compiled tape");
    cudaSetDevice(c->ctx->device);
    cudaStreamSynchronize(c->ctx->stream);
    for (auto l : c->lib) if (l) cudaLibraryUnload(l);
    fc_tape_release(c->tape);
    delete c;
    return FC_OK;
}

int32_t fc_compiled_float_slice_eval(fc_eval* e, const fc_compiled* c, const float* const* vars, float* const* out,
                                     uint64_t n) {
    if (int32_t rc = check_kind(e, c, K_FLOAT)) return rc;
    return bulk_eval(e, c->tape, reinterpret_cast<const void* const*>(vars), reinterpret_cast<void* const*>(out), n, 4,
                     [&](BulkParams& p, const std::vector<const void*>&) { return launch_compiled(c, K_FLOAT, n, &p); });
}
int32_t fc_compiled_grad_slice_eval(fc_eval* e, const fc_compiled* c, const fc_grad* const* vars, fc_grad* const* out,
                                    uint64_t n) {
    if (int32_t rc = check_kind(e, c, K_GRAD)) return rc;
    return bulk_eval(e, c->tape, reinterpret_cast<const void* const*>(vars), reinterpret_cast<void* const*>(out), n, 16,
                     [&](BulkParams& p, const std::vector<const void*>&) { return launch_compiled(c, K_GRAD, n, &p); });
}
int32_t fc_compiled_interval_eval_batch(fc_eval* e, const fc_compiled* c, const float* vars, uint64_t n, float* out,
                                        uint8_t* choices, uint8_t* simplify) {
    if (int32_t rc = check_kind(e, c, K_INTERVAL)) return rc;
    return tracing_eval(e, c->tape, vars, n, out, choices, simplify, true,
                        [&](TracingParams& p) { return launch_compiled(c, K_INTERVAL, n, &p); });
}

}  // extern "C"
