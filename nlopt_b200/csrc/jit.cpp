// jit.cpp -- __device__ functors given as SOURCE (nlopt_b200_jit_*, include/nlopt_b200.h): compiled at run time with NVRTC
// for sm_90a, together with the map kernels of include/nlopt_b200_device_kernels.cuh, and registered through the
// nlopt_b200_*_device2 / *_mconstraint_device2 entry points.  A functor compiled here runs the header's own
// map_group_kernel / map_group_mkernel and this library's fold_groups_kernel / fold_groups_mkernel (device_backend.cu), launched as
// trampoline2 / mtrampoline2 launch them, so its values have the bits of the same functor compiled by nvcc.
//
// NVRTC is opened with dlopen at the first compile (the library gains no link dependency on it).  Compiled images are
// cached per process, keyed by source, functor name and options; an image is loaded with cudaLibraryLoadData, which
// does not depend on the current context, at the first launch.
#include <dlfcn.h>
#include <nvrtc.h>

#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include <cuda_runtime.h>

#include "nlopt_object.hpp"

// kJitKernelsHeader / kJitApiHeader: the text of include/nlopt_b200_device_kernels.cuh and include/nlopt_b200.h, written
// as raw string literals by build() (__graft_entry__.py), so the compiler needs no include path at run time
#include "jit_headers.inc"

#ifndef NLOPT_B200_CUDA_LIB64
#define NLOPT_B200_CUDA_LIB64 "/usr/local/cuda/lib64"      // build() passes the lib64 of the toolkit it builds with
#endif

namespace nb200 {
// device_backend.cu: the fold kernels of trampoline2 (m == 0) / mtrampoline2 on stream s
void fold_functor_sums(unsigned m, const double *partials, const nlopt_b200_shard &sh, double *vsums, cudaStream_t s);
}

namespace {

constexpr int kThreads = 256;       // nlopt_b200::detail::kThreads: the block size of the map kernels

// ---- NVRTC, opened at first use ------------------------------------------------------------------------------------
struct Nvrtc {
    decltype(&nvrtcCreateProgram) create = nullptr;
    decltype(&nvrtcDestroyProgram) destroy = nullptr;
    decltype(&nvrtcAddNameExpression) add_name = nullptr;
    decltype(&nvrtcCompileProgram) compile = nullptr;
    decltype(&nvrtcGetProgramLogSize) log_size = nullptr;
    decltype(&nvrtcGetProgramLog) log = nullptr;
    decltype(&nvrtcGetCUBINSize) cubin_size = nullptr;
    decltype(&nvrtcGetCUBIN) cubin = nullptr;
    decltype(&nvrtcGetLoweredName) lowered = nullptr;
    decltype(&nvrtcGetErrorString) error_string = nullptr;
    std::string error;          // why NVRTC could not be opened
};

const Nvrtc &nvrtc()
{
    static Nvrtc api;
    static std::once_flag once;
    std::call_once(once, [] {
        void *h = dlopen("libnvrtc.so.12", RTLD_NOW | RTLD_LOCAL);
        if (!h) h = dlopen(NLOPT_B200_CUDA_LIB64 "/libnvrtc.so.12", RTLD_NOW | RTLD_LOCAL);
        if (!h) {
            const char *e = dlerror();
            api.error = std::string("NVRTC (libnvrtc.so.12) could not be loaded, neither by soname nor from "
                                    NLOPT_B200_CUDA_LIB64 ": ") + (e ? e : "unknown error");
            return;
        }
        bool ok = true;
        auto sym = [&](auto &fn, const char *name) {
            fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
            ok = ok && fn;
        };
        sym(api.create, "nvrtcCreateProgram");
        sym(api.destroy, "nvrtcDestroyProgram");
        sym(api.add_name, "nvrtcAddNameExpression");
        sym(api.compile, "nvrtcCompileProgram");
        sym(api.log_size, "nvrtcGetProgramLogSize");
        sym(api.log, "nvrtcGetProgramLog");
        sym(api.cubin_size, "nvrtcGetCUBINSize");
        sym(api.cubin, "nvrtcGetCUBIN");
        sym(api.lowered, "nvrtcGetLoweredName");
        sym(api.error_string, "nvrtcGetErrorString");
        if (!ok) api.error = "libnvrtc.so.12 lacks an entry point this library needs";
    });
    return api;
}

// appended to the caller's source: a dummy functor of the other shape, so that both map kernels can be named for any
// functor and the one of its shape is the functor's own instantiation, and `info`, whose lowered name spells m, halo
// and sizeof(F) (read without a device)
const char kSuffix[] = R"jit(
namespace nlopt_b200 { namespace detail { namespace jit {
struct no_scalar {
    __device__ double operator()(unsigned long long, unsigned long long, long long, long long, const double *, double *) const
    { return 0.0; }
};
struct no_vector {
    static constexpr int m = 1;
    __device__ void operator()(unsigned long long, unsigned long long, long long, long long, const double *, double *, double *,
                               long long) const {}
};
template <bool B, class T, class E> struct pick { using type = T; };
template <class T, class E> struct pick<false, T, E> { using type = E; };
template <class F> using scalar_t = typename pick<m_of<F>::value == 0, F, no_scalar>::type;
template <class F> using vector_t = typename pick<m_of<F>::value != 0, F, no_vector>::type;
template <int M, int H, unsigned long long S> __global__ void info() {}
} } }
)jit";

// one compiled functor; shared by every handle created with the same source, name and options
struct Image {
    std::string error;          // empty when compiled and accepted
    std::string log;            // NVRTC's log
    std::vector<char> cubin;
    int m = 0, halo = 0;
    size_t param_bytes = 0;
    std::string kernel_name;    // lowered name of map_group_kernel<F> (m == 0) or map_group_mkernel<F>

    std::mutex load_mutex;
    bool loaded = false;
    cudaError_t load_error = cudaSuccess;
    cudaLibrary_t library = nullptr;
    cudaKernel_t kernel = nullptr;

    cudaKernel_t get_kernel()
    {
        std::lock_guard<std::mutex> g(load_mutex);
        if (!loaded) {
            loaded = true;
            load_error = cudaLibraryLoadData(&library, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
            if (load_error == cudaSuccess) load_error = cudaLibraryGetKernel(&kernel, library, kernel_name.c_str());
            if (load_error != cudaSuccess) {
                std::fprintf(stderr, "nlopt_b200: loading the compiled functor failed: %s\n", cudaGetErrorString(load_error));
                kernel = nullptr;
            }
        }
        return kernel;
    }
};

// "...infoILi4ELi0ELy24EEEvv" -> {4, 0, 24}
bool parse_info(const char *lowered, long long out[3])
{
    const char *p = std::strstr(lowered, "4infoI");
    if (!p) return false;
    p += 6;
    for (int k = 0; k < 3; ++k) {
        if (*p++ != 'L') return false;
        if (*p != 'i' && *p != 'y') return false;
        ++p;
        const bool neg = *p == 'n';
        if (neg) ++p;
        if (*p < '0' || *p > '9') return false;
        long long v = 0;
        while (*p >= '0' && *p <= '9') v = v * 10 + (*p++ - '0');
        if (*p++ != 'E') return false;
        out[k] = neg ? -v : v;
    }
    return true;
}

std::shared_ptr<Image> compile(const std::string &source, const std::string &name, const std::vector<std::string> &options)
{
    auto img = std::make_shared<Image>();
    const Nvrtc &api = nvrtc();
    if (!api.error.empty()) {
        img->error = api.error;
        return img;
    }
    const std::string full = std::string("#include \"nlopt_b200_device_kernels.cuh\"\n#line 1 \"functor.cu\"\n") + source + "\n" + kSuffix;
    const char *headers[] = {kJitKernelsHeader, kJitApiHeader};
    const char *header_names[] = {"nlopt_b200_device_kernels.cuh", "nlopt_b200.h"};
    nvrtcProgram prog = nullptr;
    nvrtcResult r = api.create(&prog, full.c_str(), "functor.cu", 2, headers, header_names);
    if (r != NVRTC_SUCCESS) {
        img->error = std::string("nvrtcCreateProgram: ") + api.error_string(r);
        return img;
    }
    const std::string info = "nlopt_b200::detail::jit::info<nlopt_b200::detail::m_of<" + name + ">::value, nlopt_b200::detail::halo_of<"
                           + name + ">::value, sizeof(" + name + ")>";
    const std::string scalar = "nlopt_b200::detail::map_group_kernel<nlopt_b200::detail::jit::scalar_t<" + name + ">>";
    const std::string vector = "nlopt_b200::detail::map_group_mkernel<nlopt_b200::detail::jit::vector_t<" + name + ">>";
    api.add_name(prog, info.c_str());
    api.add_name(prog, scalar.c_str());
    api.add_name(prog, vector.c_str());
    // the library's own contract: sm_90a and no contraction of a * b + c into an FMA
    std::vector<const char *> opts = {"-arch=sm_90a", "-std=c++17", "--fmad=false"};
    for (const std::string &o : options) opts.push_back(o.c_str());
    r = api.compile(prog, (int) opts.size(), opts.data());
    size_t log_size = 0;
    if (api.log_size(prog, &log_size) == NVRTC_SUCCESS && log_size > 1) {
        img->log.resize(log_size);
        api.log(prog, &img->log[0]);
        img->log.resize(log_size - 1);
    }
    if (r != NVRTC_SUCCESS) {
        img->error = std::string("compiling functor '") + name + "' failed (" + api.error_string(r) + "):\n" + img->log;
        api.destroy(&prog);
        return img;
    }
    const char *lowered_info = nullptr, *lowered_kernel = nullptr;
    long long v[3] = {0, 0, 0};
    if (api.lowered(prog, info.c_str(), &lowered_info) != NVRTC_SUCCESS || !parse_info(lowered_info, v)) {
        img->error = "could not read m, halo and sizeof of functor '" + name + "'";
    } else if (v[0] < 0 || v[0] > 16) {
        img->error = "functor '" + name + "' has m = " + std::to_string(v[0]) + ": a vector functor has 1 to 16 components";
    } else if (v[1] < 0 || v[1] > 1) {
        img->error = "functor '" + name + "' has halo = " + std::to_string(v[1]) + ": halo is 0 or 1 in this build";
    } else if (api.lowered(prog, (v[0] ? vector : scalar).c_str(), &lowered_kernel) != NVRTC_SUCCESS) {
        img->error = "could not name the map kernel of functor '" + name + "'";
    } else {
        img->m = (int) v[0];
        img->halo = (int) v[1];
        img->param_bytes = (size_t) v[2];
        img->kernel_name = lowered_kernel;
        size_t n = 0;
        if (api.cubin_size(prog, &n) != NVRTC_SUCCESS || n == 0) {
            img->error = "NVRTC returned no cubin for functor '" + name + "'";
        } else {
            img->cubin.resize(n);
            api.cubin(prog, img->cubin.data());
        }
    }
    api.destroy(&prog);
    return img;
}

// images of this process: the key spells source, name and options with their lengths
std::mutex g_cache_mutex;
std::map<std::string, std::shared_ptr<Image>> g_cache;

std::shared_ptr<Image> cached_compile(const std::string &source, const std::string &name, const std::vector<std::string> &options)
{
    std::string key;
    auto put = [&key](const std::string &s) { key += std::to_string(s.size()) + ':' + s; };
    put(source);
    put(name);
    for (const std::string &o : options) put(o);
    std::lock_guard<std::mutex> g(g_cache_mutex);
    auto it = g_cache.find(key);
    if (it != g_cache.end()) return it->second;
    auto img = compile(source, name, options);
    g_cache.emplace(key, img);
    return img;
}

// one registration: the image, an aligned copy of the caller's parameter bytes (the functor object, passed by value to
// the map kernel) and the host finish
struct alignas(16) Block16 { unsigned char b[16]; };
struct Record {
    std::shared_ptr<Image> img;
    std::vector<Block16> params;
    nlopt_b200_dfinish fin = nullptr;
    nlopt_b200_dmfinish mfin = nullptr;
    void *fin_data = nullptr;
};

// group sums of every JIT registration: [m][groups_local], reallocated when a larger shard comes (as partials2)
double *partials(size_t count)
{
    static double *p = nullptr;
    static size_t cap = 0;
    if (count > cap) {
        if (p) cudaFree(p);
        cap = count + 64;
        if (cudaMalloc(&p, cap * sizeof(double)) != cudaSuccess) {
            p = nullptr;
            cap = 0;
        }
    }
    return p;
}

// a failed load leaves NaN in the sums, so the run sees an invalid value rather than a stale one
void poison(double *vsums, size_t count, cudaStream_t s)
{
    cudaMemsetAsync(vsums, 0xff, count * sizeof(double), s);
}

// nlopt_b200_dfunc2 of a scalar functor: trampoline2's launches
void jit_trampoline2(const nlopt_b200_shard *sh, const double *x_dev, double *grad_dev, double *vsums_dev, void *data, void *stream)
{
    const Record *r = static_cast<const Record *>(data);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (sh->groups_local == 0) return;
    cudaKernel_t k = r->img->get_kernel();
    double *part = partials(sh->groups_local);
    if (!k || !part) return poison(vsums_dev + sh->vshard0, sh->local_vshards, s);
    nlopt_b200_shard shard = *sh;
    void *args[] = {const_cast<Block16 *>(r->params.data()), &shard, &x_dev, &grad_dev, &part};
    cudaLaunchKernel(reinterpret_cast<const void *>(k), dim3(sh->groups_local), dim3(kThreads), args, 0, s);
    nb200::fold_functor_sums(0, part, *sh, vsums_dev, s);
}

// nlopt_b200_dmfunc2 of a vector functor: mtrampoline2's launches
void jit_mtrampoline2(unsigned m, const nlopt_b200_shard *sh, const double *x_dev, double *grad_dev, unsigned long long grad_ld,
                      double *vsums_dev, void *data, void *stream)
{
    const Record *r = static_cast<const Record *>(data);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (sh->groups_local == 0) return;
    cudaKernel_t k = r->img->get_kernel();
    double *part = partials((size_t) m * sh->groups_local);
    if (!k || !part) {
        for (unsigned i = 0; i < m; ++i) poison(vsums_dev + 8 * i + sh->vshard0, sh->local_vshards, s);
        return;
    }
    nlopt_b200_shard shard = *sh;
    long long ld = (long long) grad_ld;
    void *args[] = {const_cast<Block16 *>(r->params.data()), &shard, &x_dev, &grad_dev, &ld, &part};
    cudaLaunchKernel(reinterpret_cast<const void *>(k), dim3(sh->groups_local), dim3(kThreads), args, 0, s);
    nb200::fold_functor_sums(m, part, *sh, vsums_dev, s);
}

double jit_finish2(double total, void *data)
{
    const Record *r = static_cast<const Record *>(data);
    return r->fin ? r->fin(total, r->fin_data) : total;
}

void jit_mfinish2(unsigned m, const double *totals, double *result, void *data)
{
    const Record *r = static_cast<const Record *>(data);
    if (r->mfin) r->mfin(m, totals, result, r->fin_data);
    else std::memcpy(result, totals, (size_t) m * sizeof(double));
}

void set_err(nlopt_opt opt, const std::string &msg)
{
    if (!opt) return;
    opt->errmsg = msg;
    opt->has_errmsg = true;
}

}  // namespace

struct nlopt_b200_jit_s {
    std::shared_ptr<Image> img;
    std::vector<std::unique_ptr<Record>> records;       // every registration made with this handle
};

namespace {

// the checks every registration makes before it reaches the _device2 entry point; returns the new record or nullptr
Record *prepare(nlopt_opt opt, nlopt_b200_jit h, const void *params, size_t param_bytes, bool vector, unsigned ntol,
                const double *tol, nlopt_result *ret)
{
    *ret = NLOPT_INVALID_ARGS;
    if (!opt) return nullptr;
    if (!h || !h->img) {
        set_err(opt, "NULL functor handle");
        return nullptr;
    }
    const Image &img = *h->img;
    if (!img.error.empty()) {
        set_err(opt, "the functor did not compile: " + img.error);
        return nullptr;
    }
    if (param_bytes != img.param_bytes || (param_bytes && !params)) {
        set_err(opt, "functor parameters are " + std::to_string(param_bytes) + " bytes, sizeof of the functor is "
                     + std::to_string(img.param_bytes));
        return nullptr;
    }
    if (vector != (img.m > 0)) {
        set_err(opt, vector ? "a scalar functor (no member m) cannot be registered as an mconstraint"
                            : "a vector functor (m = " + std::to_string(img.m) + ") is registered with the _mconstraint forms");
        return nullptr;
    }
    if (tol)
        for (unsigned i = 0; i < ntol; ++i)
            if (!(tol[i] >= 0.0)) {
                set_err(opt, "constraint tolerance must be non-negative (got " + std::to_string(tol[i]) + ")");
                return nullptr;
            }
    auto r = std::make_unique<Record>();
    r->img = h->img;
    r->params.resize((param_bytes + sizeof(Block16) - 1) / sizeof(Block16));
    if (param_bytes) std::memcpy(r->params.data(), params, param_bytes);
    h->records.push_back(std::move(r));
    *ret = NLOPT_SUCCESS;
    return h->records.back().get();
}

nlopt_result scalar_reg(nlopt_opt opt, nlopt_b200_jit h, const void *params, size_t param_bytes, nlopt_b200_dfinish fin, void *fin_data,
                        int role, double tol)
{
    nlopt_result ret;
    Record *r = prepare(opt, h, params, param_bytes, false, role >= 2 ? 1 : 0, &tol, &ret);
    if (!r) return ret;
    r->fin = fin;
    r->fin_data = fin_data;
    const int halo = h->img->halo;
    switch (role) {
    case 0: ret = nlopt_b200_set_min_objective_device2(opt, jit_trampoline2, jit_finish2, r, halo); break;
    case 1: ret = nlopt_b200_set_max_objective_device2(opt, jit_trampoline2, jit_finish2, r, halo); break;
    case 2: ret = nlopt_b200_add_inequality_constraint_device2(opt, jit_trampoline2, jit_finish2, r, tol, halo); break;
    default: ret = nlopt_b200_add_equality_constraint_device2(opt, jit_trampoline2, jit_finish2, r, tol, halo); break;
    }
    if (ret < 0) h->records.pop_back();
    return ret;
}

nlopt_result vector_reg(nlopt_opt opt, nlopt_b200_jit h, const void *params, size_t param_bytes, nlopt_b200_dmfinish fin, void *fin_data,
                        bool equality, const double *tol)
{
    nlopt_result ret;
    const unsigned m = h && h->img ? (unsigned) h->img->m : 0;
    Record *r = prepare(opt, h, params, param_bytes, true, m, tol, &ret);
    if (!r) return ret;
    r->mfin = fin;
    r->fin_data = fin_data;
    const int halo = h->img->halo;
    ret = equality ? nlopt_b200_add_equality_mconstraint_device2(opt, m, jit_mtrampoline2, jit_mfinish2, r, tol, halo)
                   : nlopt_b200_add_inequality_mconstraint_device2(opt, m, jit_mtrampoline2, jit_mfinish2, r, tol, halo);
    if (ret < 0) h->records.pop_back();
    return ret;
}

}  // namespace

extern "C" {

nlopt_b200_jit nlopt_b200_jit_create(const char *source, const char *name, const char *const *options, int noptions)
{
    auto *h = new (std::nothrow) nlopt_b200_jit_s;
    if (!h) return nullptr;
    if (!source || !name || !*name || noptions < 0 || (noptions > 0 && !options)) {
        h->img = std::make_shared<Image>();
        h->img->error = "nlopt_b200_jit_create needs a source, a functor name and noptions >= 0 options";
        return h;
    }
    std::vector<std::string> opts;
    for (int i = 0; i < noptions; ++i) opts.emplace_back(options[i] ? options[i] : "");
    h->img = cached_compile(source, name, opts);
    return h;
}

void nlopt_b200_jit_destroy(nlopt_b200_jit h) { delete h; }

const char *nlopt_b200_jit_errmsg(nlopt_b200_jit h)
{
    if (!h) return "NULL functor handle";
    return h->img->error.empty() ? nullptr : h->img->error.c_str();
}

const char *nlopt_b200_jit_log(nlopt_b200_jit h) { return h ? h->img->log.c_str() : ""; }

int nlopt_b200_jit_info(nlopt_b200_jit h, int *m, int *halo, size_t *param_bytes)
{
    if (!h || !h->img->error.empty()) return -1;
    if (m) *m = h->img->m;
    if (halo) *halo = h->img->halo;
    if (param_bytes) *param_bytes = h->img->param_bytes;
    return 0;
}

const void *nlopt_b200_jit_image(nlopt_b200_jit h, size_t *bytes)
{
    const bool ok = h && h->img->error.empty();
    if (bytes) *bytes = ok ? h->img->cubin.size() : 0;
    return ok ? h->img->cubin.data() : nullptr;
}

nlopt_result nlopt_b200_jit_set_min_objective(nlopt_opt opt, nlopt_b200_jit f, const void *params, size_t param_bytes,
                                              nlopt_b200_dfinish finish, void *finish_data)
{ return scalar_reg(opt, f, params, param_bytes, finish, finish_data, 0, 0.0); }
nlopt_result nlopt_b200_jit_set_max_objective(nlopt_opt opt, nlopt_b200_jit f, const void *params, size_t param_bytes,
                                              nlopt_b200_dfinish finish, void *finish_data)
{ return scalar_reg(opt, f, params, param_bytes, finish, finish_data, 1, 0.0); }
nlopt_result nlopt_b200_jit_add_inequality_constraint(nlopt_opt opt, nlopt_b200_jit fc, const void *params, size_t param_bytes,
                                                      nlopt_b200_dfinish finish, void *finish_data, double tol)
{ return scalar_reg(opt, fc, params, param_bytes, finish, finish_data, 2, tol); }
nlopt_result nlopt_b200_jit_add_equality_constraint(nlopt_opt opt, nlopt_b200_jit h, const void *params, size_t param_bytes,
                                                    nlopt_b200_dfinish finish, void *finish_data, double tol)
{ return scalar_reg(opt, h, params, param_bytes, finish, finish_data, 3, tol); }
nlopt_result nlopt_b200_jit_add_inequality_mconstraint(nlopt_opt opt, nlopt_b200_jit fc, const void *params, size_t param_bytes,
                                                       nlopt_b200_dmfinish finish, void *finish_data, const double *tol)
{ return vector_reg(opt, fc, params, param_bytes, finish, finish_data, false, tol); }
nlopt_result nlopt_b200_jit_add_equality_mconstraint(nlopt_opt opt, nlopt_b200_jit h, const void *params, size_t param_bytes,
                                                     nlopt_b200_dmfinish finish, void *finish_data, const double *tol)
{ return vector_reg(opt, h, params, param_bytes, finish, finish_data, true, tol); }

}  // extern "C"
