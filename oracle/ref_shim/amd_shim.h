/*
 * amd_shim.h -- the HLSL scalar / vector types, constructors, operators and intrinsics the AMD FidelityFX headers
 * use under A_GPU + A_HLSL, for compiling the REFERENCE's own kernel lines on the host (fsr_ref.cpp, cas_ref.cpp).
 * TEST INFRASTRUCTURE ONLY.  Nothing of the algorithms lives here.  Include inside namespace ref.
 */
// ---- HLSL scalar/vector types as the AMD headers name them (ffx_a.h A_HLSL section) ----
typedef float AF1;
typedef uint32_t AU1;
typedef bool AP1;

struct AF2 {
  float x, y;
  AF2() : x(0), y(0) {}
  AF2(double a, double b) : x((float)a), y((float)b) {}
  explicit AF2(const struct AU2 &u);
};
struct AF3pod { float r, g, b; };
struct AF3 {
  union { struct { float x, y, z; }; struct { float r, g, b; }; };
  AF3() : x(0), y(0), z(0) {}
  AF3(float a, float b_, float c) : x(a), y(b_), z(c) {}
  AF3(const AF3pod &p) : x(p.r), y(p.g), z(p.b) {}
};
struct AF4 {
  union { struct { float x, y, z, w; }; struct { float r, g, b, a; }; AF3pod rgb; };
  AF4() : x(0), y(0), z(0), w(0) {}
  AF4(float a_, float b_, float c, float d) : x(a_), y(b_), z(c), w(d) {}
};
struct AU2 { uint32_t x, y; AU2() : x(0), y(0) {} AU2(uint32_t a, uint32_t b) : x(a), y(b) {} };
struct AU2pod { uint32_t x, y; };
struct AU4 {
  union { struct { uint32_t x, y, z, w; }; struct { AU2pod xy, zw; }; };
};
struct ASU2 {
  int x, y;
  ASU2(int a, int b) : x(a), y(b) {}
  explicit ASU2(const AU2 &u) : x((int)u.x), y((int)u.y) {}
  explicit ASU2(const AF2 &f) : x((int)f.x), y((int)f.y) {}
};
inline AF2::AF2(const AU2 &u) : x((float)u.x), y((float)u.y) {}

#define AF1_(a) ((ref::AF1)(a))
#define AU1_(a) ((ref::AU1)(a))
static inline AF2 AF2_(double a) { return AF2(a, a); }
static inline AF3 AF3_(float a) { return AF3(a, a, a); }
static inline AF4 AF4_(double a) { return AF4((float)a, (float)a, (float)a, (float)a); }
static inline AF1 AF1_AU1(AU1 u) { return ovo_u2f(u); }
static inline AU1 AU1_AF1(AF1 f) { return ovo_f2u(f); }
static inline AF2 AF2_AU2(const AU2pod &u) { AF2 r; r.x = ovo_u2f(u.x); r.y = ovo_u2f(u.y); return r; }

// ---- HLSL operators / intrinsics with D3D semantics (NaN-ignoring min/max, saturate(NaN)=0) ----
static inline AF2 operator+(AF2 a, AF2 b) { return AF2(a.x + b.x, a.y + b.y); }
static inline AF2 operator-(AF2 a, AF2 b) { return AF2(a.x - b.x, a.y - b.y); }
static inline AF2 operator*(AF2 a, AF2 b) { return AF2(a.x * b.x, a.y * b.y); }
static inline AF2 &operator-=(AF2 &a, AF2 b) { a.x -= b.x; a.y -= b.y; return a; }
static inline AF2 &operator*=(AF2 &a, AF2 b) { a.x *= b.x; a.y *= b.y; return a; }
static inline AF3 operator*(AF3 a, AF3 b) { return AF3(a.x * b.x, a.y * b.y, a.z * b.z); }
static inline AF3 operator*(AF3 a, float b) { return AF3(a.x * b, a.y * b, a.z * b); }
static inline AF3 &operator+=(AF3 &a, AF3 b) { a.x += b.x; a.y += b.y; a.z += b.z; return a; }
static inline AF4 operator*(AF4 a, AF4 b) { return AF4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
static inline AF4 operator+(AF4 a, AF4 b) { return AF4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
static inline ASU2 operator+(ASU2 a, ASU2 b) { return ASU2(a.x + b.x, a.y + b.y); }
// min / max / saturate are the checker's pinned rule (ovr_glue.h ovo_min / ovo_max / ovo_sat), not libm's
static inline float min(float a, float b) { return ovo_min(a, b); }
static inline float max(float a, float b) { return ovo_max(a, b); }
static inline float abs(float a) { return fabsf(a); }
static inline float clamp(float x, float lo, float hi) { return ovo_min(ovo_max(x, lo), hi); }
static inline AF2 floor(AF2 a) { return AF2(floorf(a.x), floorf(a.y)); }
static inline AF3 min(AF3 a, AF3 b) { return AF3(ovo_min(a.x, b.x), ovo_min(a.y, b.y), ovo_min(a.z, b.z)); }
static inline AF3 max(AF3 a, AF3 b) { return AF3(ovo_max(a.x, b.x), ovo_max(a.y, b.y), ovo_max(a.z, b.z)); }
// ffx_a.h:1141,1143,1166,1168,1196,1206 (A_HLSL definitions; one-line wrappers around the intrinsics)
static inline AF1 AMax3F1(AF1 x, AF1 y, AF1 z) { return max(x, max(y, z)); }
static inline AF1 AMin3F1(AF1 x, AF1 y, AF1 z) { return min(x, min(y, z)); }
static inline AF3 AMax3F3(AF3 x, AF3 y, AF3 z) { return max(x, max(y, z)); }
static inline AF3 AMin3F3(AF3 x, AF3 y, AF3 z) { return min(x, min(y, z)); }
static inline AF1 ARcpF1(AF1 x) { return 1.0f / x; }                 // rcp(x)
static inline AF1 ASatF1(AF1 x) { return ovo_sat(x); }               // saturate(x)

