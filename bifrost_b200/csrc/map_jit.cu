// map_jit.cu -- the general bfMap: an arbitrary user expression over named
// arrays, compiled at run time with NVRTC for sm_90a and cached.
//
// Replaces src/map.cpp:110-406,630-797 (code generation, NVRTC build, kernel
// cache, launch) and the device headers it embeds (src/Complex.hpp,
// src/ArrayIndexer.cuh, src/IndexArray.cuh, src/ShapeIndexer.cuh) with this
// file's own generator and its own device prelude.  What a user string may
// rely on is kept (python/bifrost/map.py:64-112, test/test_map.py):
//   * array names are the element at the current index, broadcast against the
//     computation shape from the trailing dimension ("c = a + b"), or -- when
//     the string indexes them -- callable views: a(i,j), a(_), a(_, 0),
//     a(_ - a.shape()/2); negative indices count from the end, dimensions of
//     length 1 broadcast;
//   * `_` is the index vector of the current element, axis_names name its
//     components, `<name>_type` is an argument's element type, `_shape` the
//     computation shape;
//   * immutable 1-element system-space arrays are scalars passed by value;
//   * element types: signed char .. unsigned long long, float, double,
//     Complex<float|double|signed char|short|int>, Complex<FourBit> (ci4, real
//     part in the high nibble); Complex has .real/.imag (.x/.y), assign(),
//     conj(), mag2(), mag(), abs(), phase(), mad(), msub(), arithmetic with
//     complex and real operands;
//   * the reference's build flags (--use_fast_math, device as the default
//     execution space).
// Differences, all on the tuning side: shapes and strides are kernel
// PARAMETERS here (one compilation serves every shape of the same rank),
// block_shape / block_axes are accepted and ignored (one flat grid-stride
// loop with the last axis fastest), the cache lives in the process.
//
// libnvrtc and libcuda are dlopen'ed at the first general bfMap call: the
// library itself keeps no link-time dependency on them (it must load on a
// box without a driver), and a missing libnvrtc is reported as
// BF_STATUS_UNSUPPORTED, never papered over.
#include "core.hpp"

#include <dlfcn.h>

#include <cstring>
#include <map>
#include <mutex>
#include <sstream>
#include <string>
#include <vector>

namespace bfb {

// ---------------------------------------------------------------------------
// device prelude (compiled by NVRTC in front of every generated kernel)
// ---------------------------------------------------------------------------
static const char* const kMapPrelude = R"BFM(
typedef signed char int8_t;   typedef unsigned char uint8_t;
typedef short int16_t;        typedef unsigned short uint16_t;
typedef int int32_t;          typedef unsigned int uint32_t;
typedef long long int64_t;    typedef unsigned long long uint64_t;

struct FourBit {};
template<typename T> struct Complex;

namespace bfm {
template<bool B, typename T = void> struct enable_if {};
template<typename T> struct enable_if<true, T> { typedef T type; };
template<typename T> struct is_scalar { enum { value = 0 }; };
#define BFM_SCALAR(T_) template<> struct is_scalar<T_> { enum { value = 1 }; };
BFM_SCALAR(bool) BFM_SCALAR(char) BFM_SCALAR(signed char) BFM_SCALAR(unsigned char) BFM_SCALAR(short)
BFM_SCALAR(unsigned short) BFM_SCALAR(int) BFM_SCALAR(unsigned int) BFM_SCALAR(long) BFM_SCALAR(unsigned long)
BFM_SCALAR(long long) BFM_SCALAR(unsigned long long) BFM_SCALAR(float) BFM_SCALAR(double)
#undef BFM_SCALAR
template<typename T> struct remove_const { typedef T type; };
template<typename T> struct remove_const<const T> { typedef T type; };
}  // namespace bfm

// 4+4-bit complex storage: real part in the high nibble, two's complement
template<> struct alignas(1) Complex<FourBit> {
	typedef signed char real_type;
	signed char real_imag;
	Complex() {}
	explicit Complex(signed char r, signed char i = 0) : real_imag((signed char)(((r & 0xF) << 4) | (i & 0xF))) {}
	template<typename U> Complex(Complex<U> const& c);
	signed char re() const { return (signed char)(real_imag >> 4); }
	signed char im() const { return (signed char)((signed char)(real_imag << 4) >> 4); }
};

template<typename T> struct alignas(2 * sizeof(T)) Complex {
	typedef T real_type;
	union { T x; T real; };
	union { T y; T imag; };
	Complex() {}
	Complex(T r, T i = 0) : x(r), y(i) {}
	template<typename U> Complex(Complex<U> const& c) : x((T)c.x), y((T)c.y) {}
	Complex(Complex<FourBit> const& c) : x((T)c.re()), y((T)c.im()) {}
	Complex& assign(T r, T i) { x = r; y = i; return *this; }
	Complex& operator+=(Complex c) { x += c.x; y += c.y; return *this; }
	Complex& operator-=(Complex c) { x -= c.x; y -= c.y; return *this; }
	Complex& operator*=(Complex c) { T r = x * c.x - y * c.y; T i = x * c.y + y * c.x; x = r; y = i; return *this; }
	Complex& operator/=(Complex c) { T d = c.x * c.x + c.y * c.y; T r = (x * c.x + y * c.y) / d; T i = (y * c.x - x * c.y) / d; x = r; y = i; return *this; }
	Complex& operator*=(T s) { x *= s; y *= s; return *this; }
	Complex& operator/=(T s) { x /= s; y /= s; return *this; }
	Complex operator+() const { return *this; }
	Complex operator-() const { return Complex(-x, -y); }
	Complex conj() const { return Complex(x, -y); }
	T mag2()  const { T a = x * x; a += y * y; return a; }
	T mag()   const { return (T)sqrt((double)mag2()); }
	T abs()   const { return mag(); }
	T phase() const { return (T)atan2((double)y, (double)x); }
	Complex& mad(Complex a, Complex b)  { x += a.x * b.x; x -= a.y * b.y; y += a.x * b.y; y += a.y * b.x; return *this; }
	Complex& msub(Complex a, Complex b) { x -= a.x * b.x; x += a.y * b.y; y -= a.x * b.y; y -= a.y * b.x; return *this; }
	bool operator==(Complex const& c) const { return x == c.x && y == c.y; }
	bool operator!=(Complex const& c) const { return !(*this == c); }
	bool isreal(T tol = (T)1e-6) const { return y / x <= tol; }
};
template<> inline float  Complex<float>::mag()    const { return sqrtf(mag2()); }
template<> inline float  Complex<float>::phase()  const { return atan2f(y, x); }
template<typename U> Complex<FourBit>::Complex(Complex<U> const& c)
	: real_imag((signed char)((((int)c.x & 0xF) << 4) | ((int)c.y & 0xF))) {}

#define BFM_BINARY(op_) \
template<typename T> Complex<T> operator op_(Complex<T> a, Complex<T> b) { a op_##= b; return a; } \
template<typename T, typename U> typename bfm::enable_if<bfm::is_scalar<U>::value, Complex<T> >::type \
operator op_(Complex<T> a, U b) { a op_##= Complex<T>((T)b); return a; } \
template<typename T, typename U> typename bfm::enable_if<bfm::is_scalar<U>::value, Complex<T> >::type \
operator op_(U a, Complex<T> b) { Complex<T> c((T)a); c op_##= b; return c; }
BFM_BINARY(+) BFM_BINARY(-) BFM_BINARY(*) BFM_BINARY(/)
#undef BFM_BINARY
template<typename T> Complex<T> exp(Complex<T> const& a) { T m = (T)::exp((double)a.x); return Complex<T>(m * (T)cos((double)a.y), m * (T)sin((double)a.y)); }
inline Complex<float> rintf(Complex<float> const& c) { return Complex<float>(::rintf(c.x), ::rintf(c.y)); }
inline Complex<float> rint(Complex<float> const& c)  { return Complex<float>(::rintf(c.x), ::rintf(c.y)); }

// ---- index vectors -----------------------------------------------------------
template<int N> struct Index {
	enum { size = N };
	int v[N > 0 ? N : 1];
	int&       operator[](int i)       { return v[i]; }
	int const& operator[](int i) const { return v[i]; }
	Index operator-() const { Index r; for( int d=0; d<N; ++d ) r.v[d] = -v[d]; return r; }
};
#define BFM_INDEX_OP(op_) \
template<int N> Index<N> operator op_(Index<N> const& a, Index<N> const& b) { Index<N> r; for( int d=0; d<N; ++d ) r.v[d] = a.v[d] op_ b.v[d]; return r; } \
template<int N> Index<N> operator op_(Index<N> const& a, int b) { Index<N> r; for( int d=0; d<N; ++d ) r.v[d] = a.v[d] op_ b; return r; } \
template<int N> Index<N> operator op_(int a, Index<N> const& b) { Index<N> r; for( int d=0; d<N; ++d ) r.v[d] = a op_ b.v[d]; return r; }
BFM_INDEX_OP(+) BFM_INDEX_OP(-) BFM_INDEX_OP(*) BFM_INDEX_OP(/) BFM_INDEX_OP(%)
#undef BFM_INDEX_OP

namespace bfm {
struct ArgDesc { void* ptr; int shape[8]; long long stride[8]; };   // strides in elements
// offset of an index vector in an array: array dimension d pairs with index
// component d + max(M - ND, 0); a negative index counts from the end; a
// dimension of length 1 broadcasts
template<int ND, int M>
inline long long offset_of(ArgDesc const& a, Index<M> const& idx) {
	long long off = 0;
	const int shift = M > ND ? M - ND : 0;
#pragma unroll
	for( int d=0; d<(ND < M ? ND : M); ++d ) {
		const int len = a.shape[d];
		int i = idx.v[d + shift];
		i += (i < 0) ? len : 0;
		off += (len != 1) ? (long long)i * a.stride[d] : 0;
	}
	return off;
}
template<int M, int K> inline Index<M + K> join(Index<M> const& a, Index<K> const& b) {
	Index<M + K> r;
	for( int d=0; d<M; ++d ) r.v[d] = a.v[d];
	for( int d=0; d<K; ++d ) r.v[M + d] = b.v[d];
	return r;
}
template<typename... I> inline Index<sizeof...(I)> make_index(I... i) { Index<sizeof...(I)> r = {{ (int)i... }}; return r; }
}  // namespace bfm

// A named array inside the user's expression (advanced form): the element at
// the current index by default, any other element through operator().
template<typename T, int ND> class ArrayView {
	bfm::ArgDesc const& _a;
	long long _dflt;
public:
	typedef T type;
	enum { NDIM = ND };
	template<int M> ArrayView(bfm::ArgDesc const& a, Index<M> const& cur) : _a(a), _dflt(bfm::offset_of<ND>(a, cur)) {}
	ArrayView(ArrayView const&) = delete;
	T* data() const { return (T*)_a.ptr; }
	Index<ND> shape() const { Index<ND> s; for( int d=0; d<ND; ++d ) s.v[d] = _a.shape[d]; return s; }
	int size() const { int n = 1; for( int d=0; d<ND; ++d ) n *= _a.shape[d]; return n; }
	template<int M> T& operator()(Index<M> const& idx) const { return data()[bfm::offset_of<ND>(_a, idx)]; }
	template<int M, typename... I> typename bfm::enable_if<(sizeof...(I) > 0), T&>::type
	operator()(Index<M> const& head, I... tail) const { return (*this)(bfm::join(head, bfm::make_index(tail...))); }
	template<typename I0, typename... I> typename bfm::enable_if<bfm::is_scalar<I0>::value, T&>::type
	operator()(I0 i0, I... i) const { return (*this)(bfm::make_index(i0, i...)); }
	operator T&() const { return data()[_dflt]; }
	T& operator*()  const { return data()[_dflt]; }
	T* operator->() const { return data() + _dflt; }
	template<typename U> ArrayView& operator=(U const& v)  { data()[_dflt] = v; return *this; }
	ArrayView& operator=(ArrayView const& v)               { data()[_dflt] = (T const&)v; return *this; }
	template<typename U> ArrayView& operator+=(U const& v) { data()[_dflt] += v; return *this; }
	template<typename U> ArrayView& operator-=(U const& v) { data()[_dflt] -= v; return *this; }
	template<typename U> ArrayView& operator*=(U const& v) { data()[_dflt] *= v; return *this; }
	template<typename U> ArrayView& operator/=(U const& v) { data()[_dflt] /= v; return *this; }
};
)BFM";

// ---------------------------------------------------------------------------
// NVRTC and the driver API, loaded on demand
// ---------------------------------------------------------------------------
typedef struct _nvrtcProgram* nvrtcProgram_t;
struct JitApi {
	bool ok = false, tried = false;
	std::string why;
	int  (*nvrtcCreateProgram)(nvrtcProgram_t*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
	int  (*nvrtcCompileProgram)(nvrtcProgram_t, int, const char* const*) = nullptr;
	int  (*nvrtcGetCUBINSize)(nvrtcProgram_t, size_t*) = nullptr;
	int  (*nvrtcGetCUBIN)(nvrtcProgram_t, char*) = nullptr;
	int  (*nvrtcGetProgramLogSize)(nvrtcProgram_t, size_t*) = nullptr;
	int  (*nvrtcGetProgramLog)(nvrtcProgram_t, char*) = nullptr;
	int  (*nvrtcDestroyProgram)(nvrtcProgram_t*) = nullptr;
	// driver (only needed to run a kernel, not to compile one)
	bool drv_ok = false, drv_tried = false;
	int  (*cuModuleLoadData)(void**, const void*) = nullptr;
	int  (*cuModuleGetFunction)(void**, void*, const char*) = nullptr;
	int  (*cuModuleUnload)(void*) = nullptr;
	int  (*cuLaunchKernel)(void*, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, void*, void**, void**) = nullptr;
};
static JitApi g_jit;
static std::mutex g_jit_mutex;

template<typename F> static bool load_sym(void* lib, const char* name, F* fn) {
	*fn = (F)dlsym(lib, name);
	return *fn != nullptr;
}
static bool jit_load_nvrtc() {
	if( g_jit.tried ) return g_jit.ok;
	g_jit.tried = true;
	void* lib = nullptr;
	const char* names[] = { "libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so" };
	for( const char* n : names ) if( (lib = dlopen(n, RTLD_NOW | RTLD_LOCAL)) ) break;
	if( !lib ) { g_jit.why = "libnvrtc not found"; return false; }
	g_jit.ok = load_sym(lib, "nvrtcCreateProgram", &g_jit.nvrtcCreateProgram) &&
	           load_sym(lib, "nvrtcCompileProgram", &g_jit.nvrtcCompileProgram) &&
	           load_sym(lib, "nvrtcGetCUBINSize", &g_jit.nvrtcGetCUBINSize) &&
	           load_sym(lib, "nvrtcGetCUBIN", &g_jit.nvrtcGetCUBIN) &&
	           load_sym(lib, "nvrtcGetProgramLogSize", &g_jit.nvrtcGetProgramLogSize) &&
	           load_sym(lib, "nvrtcGetProgramLog", &g_jit.nvrtcGetProgramLog) &&
	           load_sym(lib, "nvrtcDestroyProgram", &g_jit.nvrtcDestroyProgram);
	if( !g_jit.ok ) g_jit.why = "libnvrtc lacks a required symbol";
	return g_jit.ok;
}
static bool jit_load_driver() {
	if( g_jit.drv_tried ) return g_jit.drv_ok;
	g_jit.drv_tried = true;
	void* lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
	if( !lib ) lib = dlopen("libcuda.so", RTLD_NOW | RTLD_LOCAL);
	if( !lib ) return false;
	g_jit.drv_ok = load_sym(lib, "cuModuleLoadData", &g_jit.cuModuleLoadData) &&
	               load_sym(lib, "cuModuleGetFunction", &g_jit.cuModuleGetFunction) &&
	               load_sym(lib, "cuModuleUnload", &g_jit.cuModuleUnload) &&
	               load_sym(lib, "cuLaunchKernel", &g_jit.cuLaunchKernel);
	return g_jit.drv_ok;
}

// ---------------------------------------------------------------------------
// code generation
// ---------------------------------------------------------------------------
static std::string map_ctype(BFdtype dt) {
	if( dtype_veclen(dt) > 1 ) return "";
	switch( dt ) {
	case BF_DTYPE_I8:   return "signed char";
	case BF_DTYPE_I16:  return "short";
	case BF_DTYPE_I32:  return "int";
	case BF_DTYPE_I64:  return "long long";
	case BF_DTYPE_U8:   return "unsigned char";
	case BF_DTYPE_U16:  return "unsigned short";
	case BF_DTYPE_U32:  return "unsigned int";
	case BF_DTYPE_U64:  return "unsigned long long";
	case BF_DTYPE_F32:  return "float";
	case BF_DTYPE_F64:  return "double";
	case BF_DTYPE_CI4:  return "Complex<FourBit>";
	case BF_DTYPE_CI8:  return "Complex<signed char>";
	case BF_DTYPE_CI16: return "Complex<short>";
	case BF_DTYPE_CI32: return "Complex<int>";
	case BF_DTYPE_CF32: return "Complex<float>";
	case BF_DTYPE_CF64: return "Complex<double>";
	default: return "";
	}
}
static bool map_is_scalar_arg(BFarray const* a) {
	// (src/map.cpp:191-194: a 1-element immutable array the host can read)
	return a->ndim == 1 && a->shape[0] == 1 && a->immutable &&
	       (a->space == BF_SPACE_SYSTEM || a->space == BF_SPACE_CUDA_HOST || a->space == BF_SPACE_CUDA_MANAGED);
}
static bool valid_identifier(const char* s) {
	if( !s || !*s || !(isalpha((unsigned char)*s) || *s == '_') ) return false;
	for( const char* q=s; *q; ++q ) if( !(isalnum((unsigned char)*q) || *q == '_') ) return false;
	return true;
}

struct MapSig {
	int ndim = 0;
	std::vector<std::string> axis_names;
	int narg = 0;
	std::vector<std::string> arg_names, ctypes;
	std::vector<int> arg_ndim;
	std::vector<char> arg_const, arg_scalar;
	std::string func, extra, func_name;
};

// Parameter block layout (must match the struct the generated code declares):
//   long long total; int shape[max(ndim,1)] (padded to 8); ArgDesc arg[max(narg,1)]; 16 bytes per scalar slot
static size_t params_shape_off() { return 8; }
static size_t params_args_off(int ndim) { return 8 + round_up<size_t>(4 * (size_t)std::max(ndim, 1), 8); }
static size_t params_scalars_off(int ndim, int narg) { return params_args_off(ndim) + 104 * (size_t)std::max(narg, 1); }
static size_t params_size(int ndim, int narg) { return params_scalars_off(ndim, narg) + 16 * (size_t)std::max(narg, 1); }

static std::string generate_map_source(MapSig const& s, bool basic, std::string* kernel_name) {
	std::ostringstream c;
	*kernel_name = (s.func_name.empty() ? std::string() : s.func_name + "_") + "map_kernel";
	for( char& ch : *kernel_name ) if( !(isalnum((unsigned char)ch) || ch == '_') ) ch = '_';
	c << kMapPrelude << "\n";
	if( !s.extra.empty() ) c << "\n" << s.extra << "\n\n";
	const int nd = std::max(s.ndim, 1), na = std::max(s.narg, 1);
	c << "struct BfmParams { long long total; int shape[" << nd << "]; ";
	if( nd % 2 ) c << "int _pad; ";
	c << "bfm::ArgDesc arg[" << na << "]; unsigned long long scalar[" << na << "][2]; };\n";
	c << "extern \"C\" __global__ void __launch_bounds__(256) " << *kernel_name << "(const __grid_constant__ BfmParams _P) {\n";
	c << "  enum { NDIM = " << s.ndim << " };\n";
	c << "  const int _shape[" << nd << "] = {";
	for( int d=0; d<nd; ++d ) c << (d ? ", " : "") << (d < s.ndim ? "_P.shape[" + std::to_string(d) + "]" : std::string("1"));
	c << "}; (void)_shape[0];\n";
	for( int a=0; a<s.narg; ++a ) {
		c << "  typedef " << s.ctypes[a] << " " << s.arg_names[a] << "_type;\n";
		if( s.arg_scalar[a] )
			c << "  const " << s.ctypes[a] << " " << s.arg_names[a] << " = *(const " << s.ctypes[a] << "*)&_P.scalar[" << a << "][0];\n";
	}
	c << "  for( long long _lin = blockIdx.x * (long long)blockDim.x + threadIdx.x; _lin < _P.total; _lin += (long long)gridDim.x * blockDim.x ) {\n";
	c << "    Index<NDIM> _;\n";
	c << "    { long long _r = _lin;";
	for( int d=s.ndim-1; d>=0; --d ) {
		if( d == 0 ) c << " _.v[0] = (int)_r;";
		else c << " { long long _q = _r / _P.shape[" << d << "]; _.v[" << d << "] = (int)(_r - _q * _P.shape[" << d << "]); _r = _q; }";
	}
	c << " }\n";
	for( int a=0; a<s.narg; ++a ) {
		if( s.arg_scalar[a] ) continue;
		std::string T = s.ctypes[a] + (s.arg_const[a] ? " const" : "");
		if( basic )
			c << "    " << T << "& " << s.arg_names[a] << " = ((" << T << "*)_P.arg[" << a << "].ptr)[bfm::offset_of<" << s.arg_ndim[a]
			  << ">(_P.arg[" << a << "], _)];\n";
		else
			c << "    ArrayView<" << T << ", " << s.arg_ndim[a] << "> " << s.arg_names[a] << "(_P.arg[" << a << "], _);\n";
	}
	for( int d=0; d<s.ndim && d<(int)s.axis_names.size(); ++d )
		if( !s.axis_names[d].empty() ) c << "    const int " << s.axis_names[d] << " = _.v[" << d << "]; (void)" << s.axis_names[d] << ";\n";
	c << "    " << s.func << ";\n";
	c << "  }\n}\n";
	return c.str();
}

static BFstatus nvrtc_compile(std::string const& src, std::string const& name, std::vector<char>* cubin, std::string* log) {
	if( !jit_load_nvrtc() ) { if( log ) *log = g_jit.why; return BF_STATUS_UNSUPPORTED; }
	nvrtcProgram_t prog = nullptr;
	if( g_jit.nvrtcCreateProgram(&prog, src.c_str(), name.c_str(), 0, nullptr, nullptr) != 0 ) return BF_STATUS_INTERNAL_ERROR;
	const char* opts[] = { "--std=c++17", "--gpu-architecture=sm_90a", "--use_fast_math",
	                       "--device-as-default-execution-space", "--restrict", "-w" };
	int rc = g_jit.nvrtcCompileProgram(prog, (int)(sizeof(opts) / sizeof(opts[0])), opts);
	if( log ) {
		size_t n = 0;
		if( g_jit.nvrtcGetProgramLogSize(prog, &n) == 0 && n > 1 ) {
			std::vector<char> buf(n);
			g_jit.nvrtcGetProgramLog(prog, buf.data());
			*log = buf.data();
		}
	}
	BFstatus st = BF_STATUS_SUCCESS;
	if( rc != 0 ) st = BF_STATUS_INVALID_ARGUMENT;      // (the user's expression does not compile: src/map.cpp:376-379)
	else {
		size_t n = 0;
		if( g_jit.nvrtcGetCUBINSize(prog, &n) != 0 || n == 0 ) st = BF_STATUS_INTERNAL_ERROR;
		else { cubin->resize(n); if( g_jit.nvrtcGetCUBIN(prog, cubin->data()) != 0 ) st = BF_STATUS_INTERNAL_ERROR; }
	}
	g_jit.nvrtcDestroyProgram(&prog);
	return st;
}

struct MapKernel {
	std::vector<char> cubin;
	std::string name;
	bool  basic = false;
	void* module = nullptr;    // CUmodule, loaded at first launch (per process; one device context)
	void* function = nullptr;  // CUfunction
	int   device = -1;
};
static std::map<std::string, MapKernel> g_map_cache;

static BFstatus make_sig(int ndim, char const* const* axis_names, int narg, BFarray const* const* args,
                         char const* const* arg_names, char const* func_name, char const* func, char const* extra_code,
                         MapSig* s) {
	s->ndim = ndim; s->narg = narg;
	for( int d=0; d<ndim; ++d ) {
		std::string n = (axis_names && axis_names[d]) ? axis_names[d] : "";
		if( !n.empty() ) BFB_ASSERT(valid_identifier(n.c_str()) && n[0] != '_', BF_STATUS_INVALID_ARGUMENT);
		s->axis_names.push_back(n);
	}
	for( int a=0; a<narg; ++a ) {
		BFB_ASSERT(args[a] && arg_names[a], BF_STATUS_INVALID_POINTER);
		BFB_ASSERT(valid_identifier(arg_names[a]), BF_STATUS_INVALID_ARGUMENT);
		std::string ct = map_ctype(args[a]->dtype);
		BFB_ASSERT(!ct.empty(), BF_STATUS_INVALID_ARGUMENT);
		s->arg_names.push_back(arg_names[a]); s->ctypes.push_back(ct);
		s->arg_ndim.push_back(args[a]->ndim); s->arg_const.push_back(args[a]->immutable ? 1 : 0);
		s->arg_scalar.push_back(map_is_scalar_arg(args[a]) ? 1 : 0);
	}
	s->func = func; s->extra = extra_code ? extra_code : ""; s->func_name = func_name ? func_name : "";
	return BF_STATUS_SUCCESS;
}
static std::string sig_key(MapSig const& s, bool force_advanced) {
	std::ostringstream k;
	k << s.ndim << '|';
	for( auto const& n : s.axis_names ) k << n << ',';
	k << '|';
	for( int a=0; a<s.narg; ++a ) k << s.arg_names[a] << ':' << s.ctypes[a] << ':' << s.arg_ndim[a] << ':' << (int)s.arg_const[a] << ':' << (int)s.arg_scalar[a] << ',';
	k << '|' << force_advanced << '|' << s.func_name << '|' << s.func << '|' << s.extra;
	return k.str();
}

// Broadcast shape of the non-scalar arguments, aligned at the trailing
// dimension (src/map.cpp: broadcast_shapes).
static bool broadcast_shape(int narg, BFarray const* const* args, long* shape, int* ndim) {
	int nd = 0;
	for( int a=0; a<narg; ++a ) if( !map_is_scalar_arg(args[a]) ) nd = std::max(nd, args[a]->ndim);
	if( nd == 0 ) { *ndim = 1; shape[0] = 1; return true; }
	for( int d=0; d<nd; ++d ) shape[d] = 1;
	for( int a=0; a<narg; ++a ) {
		if( map_is_scalar_arg(args[a]) ) continue;
		int off = nd - args[a]->ndim;
		for( int d=0; d<args[a]->ndim; ++d ) {
			long n = args[a]->shape[d];
			if( n == 1 ) continue;
			if( shape[off + d] == 1 ) shape[off + d] = n;
			else if( shape[off + d] != n ) return false;
		}
	}
	*ndim = nd;
	return true;
}

// Compiles (or finds) the kernel for this call.  No device is needed.
static BFstatus map_get_kernel(int ndim, long const* shape_in, char const* const* axis_names, int narg,
                               BFarray const* const* args, char const* const* arg_names, char const* func_name,
                               char const* func, char const* extra_code, bool force_advanced,
                               MapKernel** out, std::string* log) {
	MapSig s;
	BFstatus st = make_sig(ndim, axis_names, narg, args, arg_names, func_name, func, extra_code, &s);
	if( st != BF_STATUS_SUCCESS ) return st;
	std::string key = sig_key(s, force_advanced);
	auto it = g_map_cache.find(key);
	if( it == g_map_cache.end() ) {
		MapKernel k;
		st = BF_STATUS_INVALID_ARGUMENT;
		// the plain-reference form first (names are elements), then the callable
		// views -- the order of src/map.cpp:712-735
		for( int attempt = force_advanced ? 1 : 0; attempt < 2 && st != BF_STATUS_SUCCESS; ++attempt ) {
			std::string src = generate_map_source(s, attempt == 0, &k.name);
			st = nvrtc_compile(src, k.name, &k.cubin, log);
			k.basic = attempt == 0;
			if( st == BF_STATUS_UNSUPPORTED || st == BF_STATUS_INTERNAL_ERROR ) return st;
			if( st != BF_STATUS_SUCCESS && getenv("BF_PRINT_MAP_KERNELS") && attempt == 1 )
				fprintf(stderr, "%s\n---- bfMap: NVRTC log ----\n%s\n", src.c_str(), log ? log->c_str() : "");
		}
		if( st != BF_STATUS_SUCCESS ) return st;
		it = g_map_cache.insert(std::make_pair(key, std::move(k))).first;
	}
	*out = &it->second;
	return BF_STATUS_SUCCESS;
}

BFstatus map_jit(int ndim, long const* shape, char const* const* axis_names, int narg,
                 BFarray const* const* args, char const* const* arg_names, char const* func_name,
                 char const* func, char const* extra_code, int const* block_axes, bool compile_only, int* mode_out) {
	BFB_ASSERT(ndim >= 0 && ndim <= BF_MAX_DIMS && narg >= 0 && narg <= 32, BF_STATUS_INVALID_ARGUMENT);
	BFB_ASSERT(func && (!narg || (args && arg_names)), BF_STATUS_INVALID_POINTER);
	const bool force_advanced = (shape != nullptr && ndim > 0) || block_axes != nullptr;
	long bshape[BF_MAX_DIMS];
	if( !(shape && ndim > 0) ) {
		BFB_ASSERT(broadcast_shape(narg, args, bshape, &ndim), BF_STATUS_INVALID_SHAPE);
	} else memcpy(bshape, shape, ndim * sizeof(long));
	long total = 1;
	for( int d=0; d<ndim; ++d ) { BFB_ASSERT(bshape[d] >= 0 && bshape[d] < (1L << 31), BF_STATUS_INVALID_SHAPE); total *= bshape[d]; }
	std::lock_guard<std::mutex> lock(g_jit_mutex);
	MapKernel* k = nullptr;
	std::string log;
	BFstatus st = BF_STATUS_SUCCESS;
	BFB_TRY(st = map_get_kernel(ndim, shape, axis_names, narg, args, arg_names, func_name, func, extra_code,
	                            force_advanced, &k, &log));
	if( st != BF_STATUS_SUCCESS ) {
		if( getenv("BF_PRINT_MAP_KERNELS") || getenv("BFB_MAP_DEBUG") ) fprintf(stderr, "bfMap: %s\n", log.c_str());
		return st;
	}
	if( mode_out ) *mode_out = k->basic ? 0 : 1;
	if( compile_only || total == 0 ) return BF_STATUS_SUCCESS;

	// ---- parameter block
	std::vector<unsigned char> pb(params_size(ndim, narg), 0);
	*(long long*)&pb[0] = total;
	for( int d=0; d<ndim; ++d ) *(int*)&pb[params_shape_off() + 4 * d] = (int)bshape[d];
	for( int a=0; a<narg; ++a ) {
		BFarray const* A = args[a];
		if( map_is_scalar_arg(A) ) {
			BFB_ASSERT(A->data, BF_STATUS_INVALID_POINTER);
			memcpy(&pb[params_scalars_off(ndim, narg) + 16 * a], A->data, std::min<size_t>(16, (size_t)std::max(1, dtype_nbit(A->dtype) / 8)));
			continue;
		}
		BFB_ASSERT(A->data, BF_STATUS_INVALID_POINTER);
		BFB_ASSERT(space_on_device(A->space), BF_STATUS_INVALID_SPACE);
		const long esz = std::max(1, dtype_nbit(A->dtype) / 8);
		unsigned char* q = &pb[params_args_off(ndim) + 104 * a];
		*(void**)q = A->data;
		for( int d=0; d<A->ndim; ++d ) {
			BFB_ASSERT(A->strides[d] % esz == 0, BF_STATUS_UNSUPPORTED_STRIDE);
			*(int*)(q + 8 + 4 * d) = (int)A->shape[d];
			*(long long*)(q + 40 + 8 * d) = A->strides[d] / esz;
		}
	}
	// ---- load (once per process) and launch on the thread's stream
	BFB_ASSERT(jit_load_driver(), BF_STATUS_DEVICE_ERROR);
	int dev = 0;
	BFB_CUDA(cudaGetDevice(&dev), BF_STATUS_DEVICE_ERROR);
	if( !k->function || k->device != dev ) {
		BFB_CUDA(cudaFree(0), BF_STATUS_DEVICE_ERROR);                  // make sure the primary context is current
		if( k->module ) g_jit.cuModuleUnload(k->module);
		k->module = nullptr; k->function = nullptr;
		BFB_ASSERT(g_jit.cuModuleLoadData(&k->module, k->cubin.data()) == 0, BF_STATUS_DEVICE_ERROR);
		BFB_ASSERT(g_jit.cuModuleGetFunction(&k->function, k->module, k->name.c_str()) == 0, BF_STATUS_DEVICE_ERROR);
		k->device = dev;
	}
	unsigned grid = (unsigned)std::min<long>(div_up<long>(total, 256), 148L * 16);
	void* kargs[1] = { pb.data() };
	BFB_ASSERT(g_jit.cuLaunchKernel(k->function, grid, 1, 1, 256, 1, 1, 0, (void*)thread_stream(), kargs, nullptr) == 0,
	           BF_STATUS_DEVICE_ERROR);
	count_launch();
	return BF_STATUS_SUCCESS;
}

void map_jit_clear_cache() {
	std::lock_guard<std::mutex> lock(g_jit_mutex);
	for( auto& kv : g_map_cache ) if( kv.second.module && g_jit.cuModuleUnload ) g_jit.cuModuleUnload(kv.second.module);
	g_map_cache.clear();
}

} // namespace bfb
