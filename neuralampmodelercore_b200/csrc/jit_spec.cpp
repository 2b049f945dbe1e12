// jit_spec.cpp -- see jit_spec.h.  NVRTC is reached through dlopen (no link-time dependency: the library still
// loads, and serves every model through the precompiled kernels, on a host without libnvrtc).
#include "jit_spec.h"
#include "generic_pack.h"

#include <dlfcn.h>
#include <sys/stat.h>
#include <unistd.h>

#include <chrono>
#include <future>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <mutex>
#include <sstream>

namespace namb200
{

namespace
{
// The kernel source, embedded at build time (neuralampmodelercore_b200/_build.py writes wavenet_spec_src.inc from
// wavenet_spec.cuh as a raw string literal).
const char* const kSpecKernelSource =
#include "wavenet_spec_src.inc"
  ;
const char* const kLstmSpecKernelSource =
#include "lstm_spec_src.inc"
  ;
const char* const kLatKernelSource =
#include "wavenet_lat_src.inc"
  ;
const char* const kGenericSpecKernelSource =
#include "wavenet_generic_spec_src.inc"
  ;
const char* const kGenericDescSource =
#include "generic_desc_src.inc"
  ;

// ---- NVRTC through dlopen ------------------------------------------------------------------------------------------
typedef struct _nvrtcProgram* nvrtcProgram;
struct Nvrtc
{
  void* handle = nullptr;
  int (*Version)(int*, int*) = nullptr;
  int (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
  int (*DestroyProgram)(nvrtcProgram*) = nullptr;
  int (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
  int (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
  int (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
  int (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
  int (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string error;
  bool ok() const { return handle != nullptr; }
};

Nvrtc& nvrtc()
{
  static Nvrtc n;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12",
                           "/usr/local/cuda/lib64/libnvrtc.so"};
    for (const char* nm : names)
    {
      n.handle = dlopen(nm, RTLD_NOW | RTLD_LOCAL);
      if (n.handle)
        break;
    }
    if (!n.handle)
    {
      n.error = "libnvrtc.so.12 not found (dlopen)";
      return;
    }
    bool all = true;
    auto sym = [&](const char* s) {
      void* p = dlsym(n.handle, s);
      if (!p)
        all = false;
      return p;
    };
    n.Version = reinterpret_cast<decltype(n.Version)>(sym("nvrtcVersion"));
    n.CreateProgram = reinterpret_cast<decltype(n.CreateProgram)>(sym("nvrtcCreateProgram"));
    n.DestroyProgram = reinterpret_cast<decltype(n.DestroyProgram)>(sym("nvrtcDestroyProgram"));
    n.CompileProgram = reinterpret_cast<decltype(n.CompileProgram)>(sym("nvrtcCompileProgram"));
    n.GetCUBINSize = reinterpret_cast<decltype(n.GetCUBINSize)>(sym("nvrtcGetCUBINSize"));
    n.GetCUBIN = reinterpret_cast<decltype(n.GetCUBIN)>(sym("nvrtcGetCUBIN"));
    n.GetProgramLogSize = reinterpret_cast<decltype(n.GetProgramLogSize)>(sym("nvrtcGetProgramLogSize"));
    n.GetProgramLog = reinterpret_cast<decltype(n.GetProgramLog)>(sym("nvrtcGetProgramLog"));
    n.GetErrorString = reinterpret_cast<decltype(n.GetErrorString)>(sym("nvrtcGetErrorString"));
    if (!all)
    {
      dlclose(n.handle);
      n.handle = nullptr;
      n.error = "libnvrtc lacks an expected entry point";
    }
  });
  return n;
}

// ---- helpers ----------------------------------------------------------------------------------------------------------
uint64_t fnv1a(uint64_t h, const void* data, size_t n)
{
  const unsigned char* p = static_cast<const unsigned char*>(data);
  for (size_t i = 0; i < n; i++)
  {
    h ^= p[i];
    h *= 1099511628211ull;
  }
  return h;
}

// A float as a C++17 hexadecimal literal built from integers only (no locale, exact): [-]0x<24-bit mantissa>p<exp>f
std::string float_literal(float v)
{
  if (v == 0.0f)
    return std::signbit(v) ? "-0.0f" : "0.0f";
  int e = 0;
  const float m = std::frexp(std::fabs(v), &e); // |v| = m * 2^e, m in [0.5, 1)
  const long mi = (long)std::ldexp((double)m, 24); // exact: 24 significant bits
  char buf[64];
  std::snprintf(buf, sizeof buf, "%s0x%lXp%df", v < 0.0f ? "-" : "", mi, e - 24);
  return buf;
}

std::string library_dir()
{
  Dl_info info{};
  if (dladdr(reinterpret_cast<const void*>(&library_dir), &info) && info.dli_fname)
  {
    std::string p = info.dli_fname;
    const size_t s = p.find_last_of('/');
    return s == std::string::npos ? "." : p.substr(0, s);
  }
  return ".";
}

std::string cache_dir()
{
  if (const char* e = std::getenv("NAM_B200_JIT_CACHE"))
    if (*e)
      return e;
  return library_dir() + "/jit_cache";
}

bool read_file(const std::string& path, std::vector<char>& out)
{
  std::ifstream f(path, std::ios::binary);
  if (!f)
    return false;
  f.seekg(0, std::ios::end);
  const std::streamoff n = f.tellg();
  if (n <= 0)
    return false;
  f.seekg(0);
  out.resize((size_t)n);
  f.read(out.data(), n);
  return (bool)f;
}

void write_file_atomic(const std::string& dir, const std::string& name, const std::vector<char>& data)
{
  ::mkdir(dir.c_str(), 0755); // best effort: a read-only install simply never caches
  const std::string tmp = dir + "/." + name + "." + std::to_string((long)::getpid()) + ".tmp";
  {
    std::ofstream f(tmp, std::ios::binary);
    if (!f)
      return;
    f.write(data.data(), (std::streamsize)data.size());
    if (!f)
    {
      ::unlink(tmp.c_str());
      return;
    }
  }
  if (::rename(tmp.c_str(), (dir + "/" + name).c_str()) != 0)
    ::unlink(tmp.c_str());
}

struct CompiledKernel
{
  bool ok = false, from_cache = false;
  std::string why_not;
  std::vector<char> cubin;
  double compile_seconds = 0.0;
};

// header + `#include "<kernel_file>"` -> sm_90a cubin, through the disk cache.  `env_override`: development aid, an
// environment variable that names a file to use instead of the embedded kernel source.
CompiledKernel compile_or_fetch(const std::string& tag, const std::string& header, const char* kernel_file,
                                const char* embedded_source, const char* env_override, const std::vector<std::string>& defines,
                                const std::vector<std::pair<const char*, const char*>>& extra_headers = {})
{
  CompiledKernel r;
  std::string kernel_source = embedded_source;
  if (const char* e = std::getenv(env_override))
  {
    std::vector<char> txt;
    if (*e && read_file(e, txt))
      kernel_source.assign(txt.begin(), txt.end());
  }
  std::string opts_text = "-arch=sm_90a -std=c++17 -default-device";
  for (const std::string& d : defines)
    opts_text += " " + d;
  uint64_t h = 1469598103934665603ull;
  h = fnv1a(h, header.data(), header.size());
  h = fnv1a(h, kernel_source.data(), kernel_source.size());
  for (const auto& eh : extra_headers)
    h = fnv1a(h, eh.second, std::strlen(eh.second));
  h = fnv1a(h, opts_text.data(), opts_text.size());
  char name[96];
  std::snprintf(name, sizeof name, "%s_%016llx.cubin", tag.c_str(), (unsigned long long)h);
  const std::string dir = cache_dir();
  if (read_file(dir + "/" + name, r.cubin))
  {
    r.ok = true;
    r.from_cache = true;
    return r;
  }
  Nvrtc& n = nvrtc();
  if (!n.ok())
  {
    r.why_not = "NVRTC unavailable: " + n.error;
    return r;
  }
  const auto t0 = std::chrono::steady_clock::now();
  const std::string source = header + "\n#include \"" + kernel_file + "\"\n";
  std::vector<const char*> hdr_src = {kernel_source.c_str()}, hdr_name = {kernel_file};
  for (const auto& eh : extra_headers)
  {
    hdr_name.push_back(eh.first);
    hdr_src.push_back(eh.second);
  }
  nvrtcProgram prog = nullptr;
  int rc = n.CreateProgram(&prog, source.c_str(), (tag + "_model.cu").c_str(), (int)hdr_src.size(), hdr_src.data(), hdr_name.data());
  if (rc != 0)
  {
    r.why_not = std::string("nvrtcCreateProgram: ") + n.GetErrorString(rc);
    return r;
  }
  // -default-device: the layer loop is a generic lambda, which NVRTC would otherwise take for a host function
  std::vector<const char*> copts = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo", "-default-device"};
  for (const std::string& d : defines)
    copts.push_back(d.c_str());
  rc = n.CompileProgram(prog, (int)copts.size(), copts.data());
  if (rc != 0)
  {
    size_t ls = 0;
    n.GetProgramLogSize(prog, &ls);
    std::string log(ls, '\0');
    if (ls)
      n.GetProgramLog(prog, &log[0]);
    r.why_not = std::string("nvrtcCompileProgram: ") + n.GetErrorString(rc) + "\n" + log.substr(0, 4000);
    n.DestroyProgram(&prog);
    return r;
  }
  size_t cs = 0;
  rc = n.GetCUBINSize(prog, &cs);
  if (rc == 0 && cs > 0)
  {
    r.cubin.resize(cs);
    rc = n.GetCUBIN(prog, r.cubin.data());
  }
  n.DestroyProgram(&prog);
  if (rc != 0 || cs == 0)
  {
    r.why_not = "nvrtcGetCUBIN failed";
    r.cubin.clear();
    return r;
  }
  r.compile_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  write_file_atomic(dir, name, r.cubin);
  r.ok = true;
  return r;
}

} // namespace

bool spec_eligible(const WaveNetPlan& plan, const SpecGeometry& g, std::string* why_not)
{
  auto no = [&](const std::string& w) {
    if (why_not)
      *why_not = w;
    return false;
  };
  if (!plan.eligible)
    return no("not in the fused family: " + plan.why_not);
  if (plan.n_arrays < 1 || plan.n_arrays > 2)
    return no("more than two layer arrays");
  int pmax = 0;
  for (int a = 0; a < plan.n_arrays; a++)
  {
    pmax = std::max(pmax, plan.cp[a] / 4);
  }
  for (const LayerDesc& L : plan.layers)
    for (float v : {L.ap0, L.ap1, L.ap2, L.ap3})
      if (!std::isfinite(v))
        return no("non-finite activation parameter");
  for (float v : plan.blob)
    if (!std::isfinite(v))
      return no("non-finite weight");
  const size_t smem = (size_t)pmax * (size_t)(plan.max_lookback + g.tile()) * 16;
  if (smem * (size_t)g.min_ctas > 226u * 1024u || smem > 226u * 1024u)
    return no("history window (" + std::to_string(plan.max_lookback) + " columns) + tile do not fit in shared memory");
  return true;
}

std::string spec_header_source(const WaveNetPlan& plan)
{
  std::ostringstream o;
  o << "// generated by jit_spec.cpp: one model, as compile-time data\n"
       "#define NAMB200_SPEC_HEADER_INCLUDED 1\n"
       "namespace spec {\n"
       "struct Layer { int K, dil, act, w_off, ring_off, ring_mask; float ap0, ap1, ap2, ap3; };\n"
       "struct Array { int C, CIN, HOUT, n_layers, layer0, rech_off, head_off, head_kernel, head_dilation, head_ring_off, "
       "head_ring_mask; };\n";
  o << "constexpr int NA = " << plan.n_arrays << ";\n";
  o << "constexpr int NL = " << plan.layers.size() << ";\n";
  o << "constexpr int LS = " << plan.max_lookback << ";\n";
  o << "constexpr float head_scale = " << float_literal(plan.head_scale) << ";\n";
  o << "constexpr Array A[NA] = {\n";
  for (int a = 0; a < plan.n_arrays; a++)
  {
    const ArrayDesc& A = plan.arrays[a];
    const int cin = a == 0 ? 1 : plan.cp[a - 1];
    const int hout = a + 1 == plan.n_arrays ? 1 : plan.cp[a + 1];
    o << "  {" << plan.cp[a] << ", " << cin << ", " << hout << ", " << A.n_layers << ", " << A.layer0 << ", " << A.rech_off
      << ", " << A.head_off << ", " << A.head_kernel << ", " << A.head_dilation << ", " << A.head_ring_off << ", "
      << A.head_ring_mask << "},\n";
  }
  o << "};\nconstexpr Layer L[NL] = {\n";
  for (const LayerDesc& L : plan.layers)
    o << "  {" << L.kernel << ", " << L.dilation << ", " << L.act << ", " << L.w_off << ", " << L.ring_off << ", " << L.ring_mask
      << ", " << float_literal(L.ap0) << ", " << float_literal(L.ap1) << ", " << float_literal(L.ap2) << ", "
      << float_literal(L.ap3) << "},\n";
  o << "};\n// channels (padded) of the array that owns layer li\n"
       "__host__ __device__ constexpr int layer_channels(int li) { int c = A[0].C; for (int a = 0; a < NA; a++) if (li >= A[a].layer0 && li < "
       "A[a].layer0 + A[a].n_layers) c = A[a].C; return c; }\n";
  // the weights as bit patterns (exact, locale-free); wavenet_spec.cuh reads them through spec::w(i), and after full
  // unrolling every index is a constant, so the loads fold into FFMA immediates
  o << "__device__ const unsigned Wb[" << plan.blob.size() << "] = {\n";
  char buf[16];
  for (size_t i = 0; i < plan.blob.size(); i++)
  {
    uint32_t u;
    std::memcpy(&u, &plan.blob[i], 4);
    std::snprintf(buf, sizeof buf, "0x%08Xu,", u);
    o << buf << ((i % 8 == 7) ? "\n" : " ");
  }
  o << "};\n__device__ __forceinline__ float w(const int i) { return __uint_as_float(Wb[i]); }\n}  // namespace spec\n";
  return o.str();
}

SpecBuild build_spec_kernel(const WaveNetPlan& plan, const SpecGeometry& g)
{
  SpecBuild r;
  r.geom = g;
  if (!spec_eligible(plan, g, &r.why_not))
    return r;
  r.staged_cols = plan.max_lookback;
  for (int a = 0; a < plan.n_arrays; a++)
    r.max_planes = std::max(r.max_planes, plan.cp[a] / 4);

  const std::string header = spec_header_source(plan);
  std::vector<std::string> defs = {"-DNAMB200_SPEC_NT=" + std::to_string(g.nt), "-DNAMB200_SPEC_S=" + std::to_string(g.s),
                                   "-DNAMB200_SPEC_MINB=" + std::to_string(g.min_ctas)};
  // second entry point of the same cubin: the short-call variant (nt / 64 streams x 64 frames per CTA) for models
  // without a convolutional head
  r.has_short = g.s == 1 && g.nt % 64 == 0;
  for (int a = 0; a < plan.n_arrays; a++)
    r.has_short = r.has_short && plan.arrays[a].head_kernel == 1;
  // Two programs compiled side by side (NVRTC is re-entrant): the throughput kernel with the 64-frame short-call variant, and the
  // 128- / 256-frame variants -- half the wall time of one program with all four entry points (16 s -> 8 s for a1_standard).
  std::future<CompiledKernel> extra;
  if (r.has_short)
  {
    std::vector<std::string> defs_x = defs;
    defs_x.push_back("-DNAMB200_SPEC_ONLY_EXTRA_SHORT=1");
    defs_x.push_back("-DNAMB200_SPEC_SHORT128_NT=" + std::to_string(128 * g.short128_streams));
    defs_x.push_back("-DNAMB200_SPEC_SHORT256_NT=" + std::to_string(256 * g.short256_streams));
    extra = std::async(std::launch::async, [header, defs_x]() {
      return compile_or_fetch("wavenet_spec_x", header, "wavenet_spec.cuh", kSpecKernelSource, "NAM_B200_SPEC_SOURCE", defs_x);
    });
    defs.push_back("-DNAMB200_SPEC_SHORT_FQ=64");
    defs.push_back("-DNAMB200_SPEC_SHORT_NT=" + std::to_string(64 * g.short_streams));
  }
  const CompiledKernel ck = compile_or_fetch("wavenet_spec", header, "wavenet_spec.cuh", kSpecKernelSource, "NAM_B200_SPEC_SOURCE", defs);
  r.ok = ck.ok;
  r.why_not = ck.why_not;
  r.cubin = ck.cubin;
  r.from_cache = ck.from_cache;
  r.compile_seconds = ck.compile_seconds;
  if (extra.valid())
  {
    const CompiledKernel cx = extra.get();
    if (cx.ok)
    {
      r.cubin_extra = cx.cubin;
      r.from_cache = r.from_cache && cx.from_cache;
      r.compile_seconds = std::max(r.compile_seconds, cx.compile_seconds);
    } // (a failure here only costs the two extra entry points: the long-call kernel takes those calls)
  }
  return r;
}

// shared-memory bytes of wavenet_lat.cuh's Plan<F>: tile + exchange buffer + every (layer, tap) history window
size_t lat_smem_bytes(const WaveNetPlan& plan, int frames)
{
  int pmax = 0;
  for (int a = 0; a < plan.n_arrays; a++)
    pmax = std::max(pmax, plan.cp[a] / 4);
  size_t f4 = (size_t)2 * pmax * frames;
  for (int a = 0; a < plan.n_arrays; a++)
    for (int i = 0; i < plan.arrays[a].n_layers; i++)
    {
      const LayerDesc& L = plan.layers[plan.arrays[a].layer0 + i];
      for (int k = 0; k + 1 < L.kernel; k++)
        f4 += (size_t)(plan.cp[a] / 4) * std::min((L.kernel - 1 - k) * L.dilation, frames);
    }
  return f4 * 16;
}

SpecBuild build_lat_kernel(const WaveNetPlan& plan, int frame_warps)
{
  SpecBuild r;
  // 8 channel groups when every array's (padded) width divides by 8: twice the instruction streams of half the length
  // (wavenet_lat.cuh); $NAM_B200_LAT_GROUPS=4 keeps the 4-group form (A/B)
  int groups = 8;
  for (int a = 0; a < plan.n_arrays; a++)
    if (plan.cp[a] % 8 != 0)
      groups = 4;
  if (const char* e = std::getenv("NAM_B200_LAT_GROUPS"))
    if (std::atoi(e) == 4)
      groups = 4;
  if (32 * groups * frame_warps > 1024)
    groups = 4;
  r.geom.nt = 32 * groups * frame_warps;
  r.geom.s = 1;
  r.geom.min_ctas = 1;
  SpecGeometry tiny; // eligibility of the family (heads, finiteness); the throughput kernel's shared-memory rule does not apply
  tiny.nt = 32;
  tiny.min_ctas = 1;
  std::string why;
  if (!spec_eligible(plan, tiny, &why) && why.find("do not fit") == std::string::npos)
  {
    r.why_not = why;
    return r;
  }
  for (int a = 0; a < plan.n_arrays; a++)
    if (plan.arrays[a].head_kernel != 1)
    {
      r.why_not = "convolutional head (served by the precompiled short-call geometries)";
      return r;
    }
  if (plan.layers.size() > 64)
  {
    r.why_not = "more than 64 layers";
    return r;
  }
  const size_t smem = lat_smem_bytes(plan, 32 * frame_warps);
  if (smem > 200u * 1024u)
  {
    r.why_not = "history windows of a " + std::to_string(32 * frame_warps) + "-frame call do not fit in shared memory";
    return r;
  }
  const CompiledKernel ck = compile_or_fetch("wavenet_lat", spec_header_source(plan), "wavenet_lat.cuh", kLatKernelSource,
                                             "NAM_B200_LAT_SOURCE",
                                             {"-DNAMB200_LAT_FW=" + std::to_string(frame_warps), "-DNAMB200_LAT_GROUPS=" + std::to_string(groups)},
                                             {{"wavenet_spec.cuh", kSpecKernelSource}});
  r.ok = ck.ok;
  r.why_not = ck.why_not;
  r.cubin = ck.cubin;
  r.from_cache = ck.from_cache;
  r.compile_seconds = ck.compile_seconds;
  r.staged_cols = (int)(smem / 16); // (reused: float4 columns of dynamic shared memory)
  r.max_planes = 1;
  return r;
}

// ---- the general kernel, specialised (wavenet_generic_spec.cuh) -------------------------------------------------------
namespace
{
std::string lit(const GMat& m)
{
  std::ostringstream o;
  o << "{" << m.in << ", " << m.out << ", " << m.w_off << ", " << m.b_off << "}";
  return o.str();
}
std::string lit(const GConv& v)
{
  std::ostringstream o;
  o << "{" << v.in << ", " << v.out << ", " << v.kernel << ", " << v.dilation << ", " << v.w_off << ", " << v.b_off << ", "
    << v.ring_off << ", " << v.ring_mask << "}";
  return o.str();
}
std::string lit(const GAct& a)
{
  std::ostringstream o;
  o << "{" << a.type << ", " << float_literal(a.p0) << ", " << float_literal(a.p1) << ", " << float_literal(a.p2) << ", "
    << float_literal(a.p3) << ", " << a.slopes_off << ", " << a.n_slopes << "}";
  return o.str();
}
std::string lit(const GFilm& f)
{
  std::ostringstream o;
  o << "{" << f.active << ", " << f.shift << ", " << f.dim << ", " << lit(f.css) << "}";
  return o.str();
}
std::string lit(const GLayer& L)
{
  std::ostringstream o;
  o << "{" << L.channels << ", " << L.bottleneck << ", " << L.zrows << ", " << L.gating << ", " << L.has_l1x1 << ", " << L.has_h1x1
    << ",\n   " << lit(L.conv) << ", " << lit(L.mixin) << ", " << lit(L.l1x1) << ", " << lit(L.h1x1) << ",\n   " << lit(L.act) << ", "
    << lit(L.sec) << ",\n   {";
  for (int i = 0; i < kGenFilmSites; i++)
    o << (i ? ", " : "") << lit(L.film[i]);
  o << "}}";
  return o.str();
}
std::string lit(const GArray& A)
{
  std::ostringstream o;
  o << "{" << A.input_size << ", " << A.channels << ", " << A.head_out_size << ", " << A.head_size << ", " << A.layer0 << ", "
    << A.n_layers << ", " << lit(A.rechannel) << ", " << lit(A.head) << "}";
  return o.str();
}
std::string lit(const GNet& N)
{
  std::ostringstream o;
  o << "{" << N.in_channels << ", " << N.out_channels << ", " << N.n_arrays << ", " << N.with_head << ", " << N.n_head_convs << ", "
    << float_literal(N.head_scale) << ", " << lit(N.head_act) << ",\n  {";
  for (int i = 0; i < kGenMaxArrays; i++)
    o << (i ? ",\n   " : "") << lit(N.arrays[i]);
  o << "},\n  {";
  for (int i = 0; i < kGenMaxHeadConvs; i++)
    o << (i ? ", " : "") << lit(N.head_convs[i]);
  o << "}}";
  return o.str();
}
bool finite_desc(const GenericPlan& gp)
{
  for (float v : gp.weights)
    if (!std::isfinite(v))
      return false;
  for (const GLayer& L : gp.layers)
    for (float v : {L.act.p0, L.act.p1, L.act.p2, L.act.p3, L.sec.p0, L.sec.p1, L.sec.p2, L.sec.p3})
      if (!std::isfinite(v))
        return false;
  return std::isfinite(gp.net.head_scale) && std::isfinite(gp.cond.head_scale);
}
} // namespace

std::string generic_spec_header_source(const GenericPlan& gp)
{
  std::ostringstream o;
  o << "// generated by jit_spec.cpp: one WaveNet with the reference's full option set, as compile-time data\n"
       "#define NAMB200_GSPEC_HEADER_INCLUDED 1\n#include \"generic_desc.h\"\nnamespace gspec {\nusing namespace namb200;\n";
  o << "constexpr int has_cond = " << (gp.has_cond ? 1 : 0) << ";\n";
  o << "__device__ constexpr GNet net = " << lit(gp.net) << ";\n";
  o << "__device__ constexpr GNet cond = " << lit(gp.has_cond ? gp.cond : GNet{}) << ";\n";
  o << "__device__ constexpr GLayer layers[" << std::max<size_t>(gp.layers.size(), 1) << "] = {\n";
  for (const GLayer& L : gp.layers)
    o << "  " << lit(L) << ",\n";
  if (gp.layers.empty())
    o << "  {}\n";
  o << "};\n__device__ const unsigned Wb[" << std::max<size_t>(gp.weights.size(), 1) << "] = {\n";
  char buf[16];
  for (size_t i = 0; i < gp.weights.size(); i++)
  {
    uint32_t u;
    std::memcpy(&u, &gp.weights[i], 4);
    std::snprintf(buf, sizeof buf, "0x%08Xu,", u);
    o << buf << ((i % 8 == 7) ? "\n" : " ");
  }
  if (gp.weights.empty())
    o << "0u";
  o << "};\n__device__ __forceinline__ float w(const int i) { return __uint_as_float(Wb[i]); }\n}  // namespace gspec\n";
  return o.str();
}

SpecBuild build_generic_spec_kernel(const GenericPlan& gp)
{
  SpecBuild r;
  r.geom.nt = kGenTile;
  if (!gp.eligible)
  {
    r.why_not = "not served by the general kernel: " + gp.why_not;
    return r;
  }
  if (!finite_desc(gp))
  {
    r.why_not = "non-finite weight or activation parameter";
    return r;
  }
  if (gp.weights.size() > 40000)
  {
    r.why_not = "too many weights to unroll (" + std::to_string(gp.weights.size()) + ")";
    return r;
  }
  const CompiledKernel ck = compile_or_fetch("wavenet_generic_spec", generic_spec_header_source(gp), "wavenet_generic_spec.cuh",
                                             kGenericSpecKernelSource, "NAM_B200_GSPEC_SOURCE", {},
                                             {{"generic_desc.h", kGenericDescSource}});
  r.ok = ck.ok;
  r.why_not = ck.why_not;
  r.cubin = ck.cubin;
  r.from_cache = ck.from_cache;
  r.compile_seconds = ck.compile_seconds;
  return r;
}

bool lstm_spec_eligible(const ModelSpec& ms, std::string* why_not)
{
  auto no = [&](const std::string& w) {
    if (why_not)
      *why_not = w;
    return false;
  };
  if (ms.arch != Arch::LSTM)
    return no("not an LSTM");
  const LstmSpec& ls = ms.lstm;
  if (ms.in_channels != 1 || ms.out_channels != 1 || ls.input_size != 1)
    return no("multi-channel LSTM");
  if (ls.num_layers < 1 || ls.num_layers > 4)
    return no("more than four layers");
  long fmas = 0;
  for (int l = 0; l < ls.num_layers; l++)
    fmas += 4L * ls.hidden * ((l == 0 ? ls.input_size : ls.hidden) + ls.hidden);
  if (fmas > 320) // beyond this a lane group per stream (lstm_group.cuh) has the shorter step
    return no("cell too large for one thread per stream (" + std::to_string(fmas) + " FMAs per step)");
  for (const auto& c : ls.cells)
  {
    for (float v : c.w)
      if (!std::isfinite(v))
        return no("non-finite weight");
    for (float v : c.b)
      if (!std::isfinite(v))
        return no("non-finite weight");
  }
  return true;
}

std::string lstm_spec_header_source(const ModelSpec& ms)
{
  const LstmSpec& ls = ms.lstm;
  std::vector<float> blob; // per layer W[4H][I+H] | b[4H]; then head_w[H] | head_b -- the order of nam_b200.cu's blob
  for (const auto& c : ls.cells)
  {
    blob.insert(blob.end(), c.w.begin(), c.w.end());
    blob.insert(blob.end(), c.b.begin(), c.b.end());
  }
  blob.insert(blob.end(), ls.head_w.begin(), ls.head_w.end());
  blob.insert(blob.end(), ls.head_b.begin(), ls.head_b.end());
  std::ostringstream o;
  o << "// generated by jit_spec.cpp: one LSTM, as compile-time data\n"
       "#define NAMB200_LSTM_SPEC_HEADER_INCLUDED 1\n"
       "namespace spec {\n";
  o << "constexpr int H = " << ls.hidden << ";\nconstexpr int L = " << ls.num_layers << ";\nconstexpr int I = " << ls.input_size
    << ";\n";
  o << "__device__ const unsigned Wb[" << blob.size() << "] = {\n";
  char buf[16];
  for (size_t i = 0; i < blob.size(); i++)
  {
    uint32_t u;
    std::memcpy(&u, &blob[i], 4);
    std::snprintf(buf, sizeof buf, "0x%08Xu,", u);
    o << buf << ((i % 8 == 7) ? "\n" : " ");
  }
  o << "};\n__device__ __forceinline__ float w(const int i) { return __uint_as_float(Wb[i]); }\n}  // namespace spec\n";
  return o.str();
}

SpecBuild build_lstm_spec_kernel(const ModelSpec& ms)
{
  SpecBuild r;
  if (!lstm_spec_eligible(ms, &r.why_not))
    return r;
  const CompiledKernel ck =
    compile_or_fetch("lstm_spec", lstm_spec_header_source(ms), "lstm_spec.cuh", kLstmSpecKernelSource, "NAM_B200_LSTM_SPEC_SOURCE", {});
  r.ok = ck.ok;
  r.why_not = ck.why_not;
  r.cubin = ck.cubin;
  r.from_cache = ck.from_cache;
  r.compile_seconds = ck.compile_seconds;
  return r;
}

} // namespace namb200
