// Mesh renderer: the reference's overlay of the recovered meshes on the photo (utils/render.py:175 render_meshes,
// reached from demo.py:340-346 overlay_human_meshes, app.py and Trainer.evaluate's visu_to_save), which the reference
// runs through pyrender / OpenGL.  Here it is a z-buffer rasterizer over the meshes the engine leaves on the device.
//
// One call renders B views.  A view has its own intrinsics, an optional world->camera [R|t] (OpenCV convention) and a
// background image; person p is drawn into every view whose image is person_image[p].  Four launches, no host sync:
//   1. prep     clears the 64-bit key buffer and the big-triangle queue; with smooth shading, one thread per
//               (person, vertex) sums the angle-weighted face normals of its faces through a CSR built at create
//               (fixed order: no float atomics).
//   2. raster   one thread per (view, person, face): transform, back-face cull, near-plane clip for the bounding box,
//               coverage of the pixel centres, atomicMin of key = (z bits) << 32 | person << fbits | face.  A
//               triangle whose box exceeds kBigArea pixels goes to a queue instead.
//   3. big      one CTA per queued triangle (persistent grid), its threads striding over the box.
//   4. shade    one thread per output pixel: decode the key, perspective-correct barycentrics, pyrender's
//               metallic-roughness shading, the reference's 3x3 foreground smoothing and alpha blend, uint8 out.
//
// Coverage is "2-D homogeneous" rasterization: for the ray d = ((x+0.5-cx)/fx, (y+0.5-cy)/fy, 1) of a pixel centre,
// the edge opposite vertex k has e_k = d . (p_j x p_i) (camera-space vertices, (k, i, j) cyclic); a front-facing
// triangle covers the pixel when every e_k >= 0, with the top-left rule on e_k == 0, and the ray meets it at
// znear <= z <= zfar.  This is exact clipping against the near plane without building clipped polygons (they are built
// only for the bounding box).  e_k / sum(e) are the barycentrics of the ray's hit point, i.e. the perspective-correct
// screen-space barycentrics.  Each shared edge is evaluated in one canonical vertex order and negated for the other
// triangle, so the two triangles see exactly opposite values and the tie rule gives every pixel to one of them.
#include <algorithm>
#include <vector>

#include "common.cuh"

using namespace mhmr;

namespace {

constexpr float kZNear = 0.05f;  // pyrender IntrinsicsCamera defaults [3P-memory]
constexpr float kZFar = 100.f;
constexpr unsigned long long kEmpty = ~0ull;
constexpr int kBigArea = 256;      // bounding-box pixels above which a triangle is rasterized by a whole CTA
constexpr int kQueueCap = 1 << 20; // queued triangles; when full, a thread rasterizes its triangle itself
constexpr float kPi = 3.14159265358979f;

struct Cam {
  float fx, fy, cx, cy;
  float R[9], t[3];
};

__device__ __forceinline__ Cam load_cam(const float* K, const float* pose, int b) {
  Cam c;
  const float* k = K + 9 * b;
  c.fx = k[0]; c.cx = k[2]; c.fy = k[4]; c.cy = k[5];
  if (pose) {
    const float* q = pose + 12 * b;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      c.R[3 * r] = q[4 * r]; c.R[3 * r + 1] = q[4 * r + 1]; c.R[3 * r + 2] = q[4 * r + 2]; c.t[r] = q[4 * r + 3];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 9; ++i) c.R[i] = (i % 4 == 0) ? 1.f : 0.f;
    c.t[0] = c.t[1] = c.t[2] = 0.f;
  }
  return c;
}

__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
  return make_float3(fmaf(a.y, b.z, -a.z * b.y), fmaf(a.z, b.x, -a.x * b.z), fmaf(a.x, b.y, -a.y * b.x));
}
__device__ __forceinline__ float3 normalize3(float3 a) {
  const float n2 = dot3(a, a);
  const float s = n2 > 0.f ? rsqrtf(n2) : 0.f;
  return make_float3(a.x * s, a.y * s, a.z * s);
}

__device__ __forceinline__ float3 rotate(const Cam& c, float3 v) {
  return make_float3(fmaf(c.R[0], v.x, fmaf(c.R[1], v.y, c.R[2] * v.z)),
                     fmaf(c.R[3], v.x, fmaf(c.R[4], v.y, c.R[5] * v.z)),
                     fmaf(c.R[6], v.x, fmaf(c.R[7], v.y, c.R[8] * v.z)));
}

__device__ __forceinline__ float3 load3(const float* p) { return make_float3(p[0], p[1], p[2]); }

__device__ __forceinline__ float3 to_cam(const Cam& c, const float* v) {
  const float3 r = rotate(c, load3(v));
  return make_float3(r.x + c.t[0], r.y + c.t[1], r.z + c.t[2]);
}

struct Tri {
  float3 p[3];  // camera-space vertices
  float3 m[3];  // m[k]: edge plane opposite vertex k (through the camera centre), e_k = d . m[k] > 0 inside
  int x0, x1, y0, y1;
};

// Transforms, culls and sets up the face; false when nothing of it can be visible.  The bounding box is that of the
// near-clipped polygon, widened by a pixel (coverage itself is decided per pixel by tri_cover).
__device__ __forceinline__ bool tri_setup(const float* vp, const int* fc, const Cam& c, int W, int H, Tri& T) {
  const int id[3] = {fc[0], fc[1], fc[2]};
#pragma unroll
  for (int k = 0; k < 3; ++k) T.p[k] = to_cam(c, vp + 3 * id[k]);
  // GL's default front face is counter-clockwise in the window; for vertices in front of the camera that is
  // (p1 - p0) x (p2 - p0) . p0 < 0 in OpenCV camera coordinates.  Back faces and degenerate faces are culled.
  const float3 n = cross3(sub3(T.p[1], T.p[0]), sub3(T.p[2], T.p[0]));
  if (!(dot3(n, T.p[0]) < 0.f)) return false;
  const float zmax = fmaxf(T.p[0].z, fmaxf(T.p[1].z, T.p[2].z));
  const float zmin = fminf(T.p[0].z, fminf(T.p[1].z, T.p[2].z));
  if (!(zmax >= kZNear) || !(zmin <= kZFar)) return false;
  float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
  auto add = [&](float3 q) {
    const float u = fmaf(c.fx, q.x / q.z, c.cx), v = fmaf(c.fy, q.y / q.z, c.cy);
    umin = fminf(umin, u); umax = fmaxf(umax, u); vmin = fminf(vmin, v); vmax = fmaxf(vmax, v);
  };
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float3 a = T.p[k], b = T.p[(k + 1) % 3];
    if (a.z >= kZNear) add(a);
    if ((a.z >= kZNear) != (b.z >= kZNear)) {
      const float s = (kZNear - a.z) / (b.z - a.z);
      add(make_float3(fmaf(s, b.x - a.x, a.x), fmaf(s, b.y - a.y, a.y), kZNear));
    }
  }
  if (!(umin <= umax) || !(vmin <= vmax)) return false;
  umin = fmaxf(umin, -2.f); vmin = fmaxf(vmin, -2.f);
  umax = fminf(umax, W + 2.f); vmax = fminf(vmax, H + 2.f);
  T.x0 = max(0, __float2int_rd(umin - 0.5f) - 1); T.x1 = min(W - 1, __float2int_ru(umax - 0.5f) + 1);
  T.y0 = max(0, __float2int_rd(vmin - 0.5f) - 1); T.y1 = min(H - 1, __float2int_ru(vmax - 0.5f) + 1);
  if (T.x0 > T.x1 || T.y0 > T.y1) return false;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int i = (k + 1) % 3, j = (k + 2) % 3;
    // canonical edge plane (lower vertex id first): (p_hi - p_lo) x p_lo = p_hi x p_lo
    const bool fwd = id[i] < id[j];
    const float3 lo = fwd ? T.p[i] : T.p[j], hi = fwd ? T.p[j] : T.p[i];
    const float3 cm = cross3(sub3(hi, lo), lo);
    T.m[k] = fwd ? cm : make_float3(-cm.x, -cm.y, -cm.z);  // p_j x p_i
  }
  return true;
}

// Top-left rule: an edge owns the pixels exactly on it when its inward gradient (m.x / fx, m.y / fy) points right,
// or straight down (y grows downwards).  Opposite orientations of one edge never both own it.
__device__ __forceinline__ bool owns(float3 m) { return m.x > 0.f || (m.x == 0.f && m.y > 0.f); }

__device__ __forceinline__ bool tri_cover(const Tri& T, float dx, float dy, float (&e)[3], float& z) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    e[k] = fmaf(T.m[k].x, dx, fmaf(T.m[k].y, dy, T.m[k].z));
    if (e[k] < 0.f || (e[k] == 0.f && !owns(T.m[k]))) return false;
  }
  const float s = e[0] + e[1] + e[2];
  if (!(s > 0.f)) return false;
  z = fmaf(e[0], T.p[0].z, fmaf(e[1], T.p[1].z, e[2] * T.p[2].z)) / s;
  return z >= kZNear && z <= kZFar;
}

__device__ __forceinline__ float ray_x(const Cam& c, int x) { return __fdiv_rn(x + 0.5f - c.cx, c.fx); }
__device__ __forceinline__ float ray_y(const Cam& c, int y) { return __fdiv_rn(y + 0.5f - c.cy, c.fy); }

__device__ __forceinline__ void write_key(unsigned long long* keys, float z, unsigned int low) {
  const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(z)) << 32) | low;
  if (key < *reinterpret_cast<volatile unsigned long long*>(keys)) atomicMin(keys, key);
}

struct Params {
  int views, H, W, P, F, V, fbits, smooth;
  const int* faces;
  const int* csr_ptr;
  const int* csr_ent;
  const float* verts;
  const int* person_image;
  const int* view_image;
  const int* count;
  const float* K;
  const float* pose;
  float* normals;
  unsigned long long* keys;
  int2* queue;
  int* queue_count;
};

__device__ __forceinline__ int person_count(const Params& a) { return min(max(*a.count, 0), a.P); }

// ---- 1. clear + vertex normals ----------------------------------------------------------------------------------
// trimesh's vertex normals [3P-memory]: unit face normals weighted by the face's corner angle at the vertex, summed,
// then normalised; a zero sum stays zero.
__global__ void render_prep_kernel(Params a) {
  const long long npix = static_cast<long long>(a.views) * a.H * a.W;
  const int np = a.smooth ? person_count(a) : 0;
  const long long total = npix + static_cast<long long>(np) * a.V;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.queue_count = 0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += stride) {
    if (i < npix) {
      a.keys[i] = kEmpty;
      continue;
    }
    const long long j = i - npix;
    const int p = static_cast<int>(j / a.V), v = static_cast<int>(j % a.V);
    const float* vp = a.verts + static_cast<size_t>(p) * a.V * 3;
    float3 acc = make_float3(0.f, 0.f, 0.f);
    for (int q = a.csr_ptr[v]; q < a.csr_ptr[v + 1]; ++q) {
      const int ent = a.csr_ent[q], f = ent / 3, corner = ent % 3;
      const int* fc = a.faces + 3 * f;
      const float3 p0 = load3(vp + 3 * fc[corner]), p1 = load3(vp + 3 * fc[(corner + 1) % 3]),
                   p2 = load3(vp + 3 * fc[(corner + 2) % 3]);
      const float3 fn = cross3(sub3(p1, p0), sub3(p2, p0));  // same orientation for every corner
      const float3 u = sub3(p1, p0), w = sub3(p2, p0);
      const float ang = atan2f(sqrtf(dot3(fn, fn)), dot3(u, w));
      const float3 un = normalize3(fn);
      acc.x = fmaf(ang, un.x, acc.x); acc.y = fmaf(ang, un.y, acc.y); acc.z = fmaf(ang, un.z, acc.z);
    }
    const float3 n = normalize3(acc);
    float* out = a.normals + (static_cast<size_t>(p) * a.V + v) * 3;
    out[0] = n.x; out[1] = n.y; out[2] = n.z;
  }
}

// ---- 2. per-face rasterization ----------------------------------------------------------------------------------
__device__ __forceinline__ void raster_box(const Params& a, const Tri& T, const Cam& c, int b, unsigned int low,
                                           int start, int step) {
  const int bw = T.x1 - T.x0 + 1, n = bw * (T.y1 - T.y0 + 1);
  unsigned long long* keys = a.keys + static_cast<size_t>(b) * a.H * a.W;
  for (int i = start; i < n; i += step) {
    const int x = T.x0 + i % bw, y = T.y0 + i / bw;
    float e[3], z;
    if (tri_cover(T, ray_x(c, x), ray_y(c, y), e, z)) write_key(keys + static_cast<size_t>(y) * a.W + x, z, low);
  }
}

__global__ void __launch_bounds__(128) render_raster_kernel(Params a) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y / a.P, p = blockIdx.y % a.P;
  if (p >= person_count(a) || a.person_image[p] != a.view_image[b] || f >= a.F) return;
  const Cam c = load_cam(a.K, a.pose, b);
  if (!(c.fx > 0.f) || !(c.fy > 0.f)) return;
  Tri T;
  if (!tri_setup(a.verts + static_cast<size_t>(p) * a.V * 3, a.faces + 3 * f, c, a.W, a.H, T)) return;
  const int area = (T.x1 - T.x0 + 1) * (T.y1 - T.y0 + 1);
  if (area > kBigArea) {
    const int slot = atomicAdd(a.queue_count, 1);
    if (slot < kQueueCap) {
      a.queue[slot] = make_int2(blockIdx.y, f);
      return;
    }
  }
  raster_box(a, T, c, b, (static_cast<unsigned int>(p) << a.fbits) | f, 0, 1);
}

// ---- 3. queued large triangles: one CTA each --------------------------------------------------------------------
__global__ void __launch_bounds__(256) render_raster_big_kernel(Params a) {
  const int nq = min(*a.queue_count, kQueueCap);
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const int2 ent = a.queue[q];
    const int b = ent.x / a.P, p = ent.x % a.P, f = ent.y;
    const Cam c = load_cam(a.K, a.pose, b);
    Tri T;
    if (!tri_setup(a.verts + static_cast<size_t>(p) * a.V * 3, a.faces + 3 * f, c, a.W, a.H, T)) continue;
    raster_box(a, T, c, b, (static_cast<unsigned int>(p) << a.fbits) | f, threadIdx.x, blockDim.x);
  }
}

// ---- 4. shading + composite -------------------------------------------------------------------------------------
struct Shade {
  const unsigned char* images;
  const float* colors;
  float alpha, intensity, metallic, roughness;
  unsigned char* overlay;
  float* depth;
  int* person;
};

// pyrender's metallic-roughness fragment shader (the glTF reference BRDF) for one white directional light along the
// camera's viewing direction, plus the scene's ambient term, gamma 2.2 and the 8-bit readback [3P-memory].
__device__ __forceinline__ float3 shade_pbr(float3 n, float3 v, float3 base, float intensity, float metallic,
                                            float roughness) {
  const float min_r = 0.04f;
  const float r = fminf(fmaxf(roughness, min_r), 1.f), m = fminf(fmaxf(metallic, 0.f), 1.f);
  const float3 l = make_float3(0.f, 0.f, -1.f);
  const float3 h = normalize3(make_float3(l.x + v.x, l.y + v.y, l.z + v.z));
  const float nl = fminf(fmaxf(dot3(n, l), 0.001f), 1.f);
  const float nv = fminf(fmaxf(fabsf(dot3(n, v)), 0.001f), 1.f);
  const float nh = fminf(fmaxf(dot3(n, h), 0.f), 1.f);
  const float vh = fminf(fmaxf(dot3(v, h), 0.f), 1.f);
  const float k = (r + 1.f) * (r + 1.f) / 8.f;
  const float G = nv / (nv * (1.f - k) + k) * (nl / (nl * (1.f - k) + k));
  const float a2 = (r * r) * (r * r);
  const float fd = nh * nh * (a2 - 1.f) + 1.f;
  const float D = a2 / (kPi * fd * fd);
  const float fres = powf(fminf(fmaxf(1.f - vh, 0.f), 1.f), 5.f);
  const float bc[3] = {base.x, base.y, base.z};
  float out[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float f0 = min_r + (bc[ch] - min_r) * m;
    const float cdiff = bc[ch] * (1.f - min_r) * (1.f - m);
    const float F = f0 + (1.f - f0) * fres;
    const float diffuse = (1.f - F) * cdiff / kPi;
    const float spec = F * G * D / (4.f * nl * nv + 0.001f);
    const float col = nl * intensity * (diffuse + spec) + 0.3f * bc[ch];  // ambient_light 0.3 x base colour
    out[ch] = fminf(fmaxf(powf(col, 1.f / 2.2f), 0.f), 1.f);
  }
  return make_float3(out[0], out[1], out[2]);
}

__global__ void __launch_bounds__(256) render_shade_kernel(Params a, Shade s) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long hw = static_cast<long long>(a.H) * a.W;
  if (i >= a.views * hw) return;
  const int b = static_cast<int>(i / hw), pix = static_cast<int>(i % hw), y = pix / a.W, x = pix % a.W;
  const unsigned long long* keys = a.keys + b * hw;
  const unsigned long long key = keys[pix];
  const unsigned char* bg = s.images + (static_cast<size_t>(a.view_image[b]) * hw + pix) * 3;
  unsigned char* out = s.overlay + i * 3;
  if (key == kEmpty) {  // fg = 0: the blend returns the photo exactly
    out[0] = bg[0]; out[1] = bg[1]; out[2] = bg[2];
    if (s.depth) s.depth[i] = 0.f;
    if (s.person) s.person[i] = -1;
    return;
  }
  int nfg = 0;  // the reference's conv2d(fg, 2/9, bias -1, zero padding), times fg, clamped at 0
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const int yy = y + dy, xx = x + dx;
      if (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W) nfg += keys[yy * a.W + xx] != kEmpty;
    }
  const float fg = fmaxf(fmaf(static_cast<float>(nfg), 2.f / 9.f, -1.f), 0.f);
  const unsigned int low = static_cast<unsigned int>(key);
  const int p = static_cast<int>(low >> a.fbits), f = static_cast<int>(low & ((1u << a.fbits) - 1u));
  const float z = __uint_as_float(static_cast<unsigned int>(key >> 32));
  const Cam c = load_cam(a.K, a.pose, b);
  const float* vp = a.verts + static_cast<size_t>(p) * a.V * 3;
  const int* fc = a.faces + 3 * f;
  Tri T;
  tri_setup(vp, fc, c, a.W, a.H, T);
  const float rx = ray_x(c, x), ry = ray_y(c, y);
  float e[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) e[k] = fmaf(T.m[k].x, rx, fmaf(T.m[k].y, ry, T.m[k].z));
  const float inv = 1.f / (e[0] + e[1] + e[2]);
  float3 n;
  if (a.smooth) {
    float3 acc = make_float3(0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float3 vn = load3(a.normals + (static_cast<size_t>(p) * a.V + fc[k]) * 3);
      const float w = e[k] * inv;
      acc.x = fmaf(w, vn.x, acc.x); acc.y = fmaf(w, vn.y, acc.y); acc.z = fmaf(w, vn.z, acc.z);
    }
    n = normalize3(rotate(c, acc));
  } else {
    n = normalize3(cross3(sub3(T.p[1], T.p[0]), sub3(T.p[2], T.p[0])));
  }
  const float3 v = normalize3(make_float3(-rx * z, -ry * z, -z));
  const float* col = s.colors + 3 * p;
  const float3 rgb = shade_pbr(n, v, make_float3(col[0], col[1], col[2]), s.intensity, s.metallic, s.roughness);
  const float rgbv[3] = {rgb.x, rgb.y, rgb.z};
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float r8 = rintf(rgbv[ch] * 255.f);
    const float im = static_cast<float>(bg[ch]);
    const float o = fg * (s.alpha * r8 + (1.f - s.alpha) * im) + (1.f - fg) * im;
    out[ch] = static_cast<unsigned char>(fminf(fmaxf(o, 0.f), 255.f));
  }
  if (s.depth) s.depth[i] = z;
  if (s.person) s.person[i] = p;
}

}  // namespace

struct mhmr_render {
  int F = 0, V = 0, fbits = 0, nnz = 0;
  int* faces = nullptr;
  int* csr_ptr = nullptr;
  int* csr_ent = nullptr;
  int2* queue = nullptr;
  int* queue_count = nullptr;
  unsigned long long* keys = nullptr;
  size_t key_cap = 0;
  float* normals = nullptr;
  size_t normal_cap = 0;
  ~mhmr_render() {
    for (void* p : {static_cast<void*>(faces), static_cast<void*>(csr_ptr), static_cast<void*>(csr_ent),
                    static_cast<void*>(queue), static_cast<void*>(queue_count), static_cast<void*>(keys),
                    static_cast<void*>(normals)})
      if (p) cudaFree(p);
  }
};

namespace {

template <typename T>
int grow(T** buf, size_t* cap, size_t n) {
  if (n <= *cap) return MHMR_OK;
  if (*buf) MHMR_CUDA_CHECK(cudaFree(*buf));  // cudaFree waits for work still using the old buffer
  *buf = nullptr;
  *cap = 0;
  MHMR_CUDA_CHECK(cudaMalloc(buf, n * sizeof(T)));
  *cap = n;
  return MHMR_OK;
}

int render_build(mhmr_render* h, const int32_t* faces, cudaStream_t st) {
  const int F = h->F, V = h->V;
  std::vector<int32_t> hf(3ll * F);
  MHMR_CUDA_CHECK(cudaMemcpy(hf.data(), faces, 12ll * F, cudaMemcpyDefault));
  for (int32_t v : hf) MHMR_REQUIRE(v >= 0 && v < V, "face vertex index outside [0, num_verts)");
  // vertex -> incident (face, corner) entries, faces in increasing order
  std::vector<int32_t> ptr(V + 1, 0), ent(3ll * F);
  for (int32_t v : hf) ++ptr[v + 1];
  for (int v = 0; v < V; ++v) ptr[v + 1] += ptr[v];
  std::vector<int32_t> fill(ptr.begin(), ptr.end() - 1);
  for (int i = 0; i < 3 * F; ++i) ent[fill[hf[i]]++] = i;
  MHMR_CUDA_CHECK(cudaMalloc(&h->faces, 12ll * F));
  MHMR_CUDA_CHECK(cudaMalloc(&h->csr_ptr, 4ll * (V + 1)));
  MHMR_CUDA_CHECK(cudaMalloc(&h->csr_ent, 12ll * F));
  MHMR_CUDA_CHECK(cudaMalloc(&h->queue, sizeof(int2) * kQueueCap));
  MHMR_CUDA_CHECK(cudaMalloc(&h->queue_count, sizeof(int)));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(h->faces, hf.data(), 12ll * F, cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(h->csr_ptr, ptr.data(), 4ll * (V + 1), cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(h->csr_ent, ent.data(), 12ll * F, cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaStreamSynchronize(st));  // the host vectors go out of scope
  return MHMR_OK;
}

}  // namespace

extern "C" {

int mhmr_render_create(const int32_t* faces, int num_faces, int num_verts, void* stream, mhmr_render** out) {
  MHMR_REQUIRE(out != nullptr, "null output handle");
  *out = nullptr;
  MHMR_REQUIRE(faces != nullptr, "null faces");
  MHMR_REQUIRE(num_faces >= 1 && num_verts >= 3, "need at least one face and three vertices");
  int fbits = 0;
  while ((1ll << fbits) < num_faces) ++fbits;
  MHMR_REQUIRE(fbits <= 24, "at most 2^24 faces (the depth key keeps 32 bits for person and face)");
  auto* h = new mhmr_render();
  h->F = num_faces; h->V = num_verts; h->fbits = fbits; h->nnz = 3 * num_faces;
  const int rc = render_build(h, faces, static_cast<cudaStream_t>(stream));
  if (rc != MHMR_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return MHMR_OK;
}

int mhmr_render_destroy(mhmr_render* h) {
  delete h;
  return MHMR_OK;
}

int mhmr_render_info(const mhmr_render* h, int* num_faces, int* num_verts, int* face_bits) {
  MHMR_REQUIRE(h != nullptr, "null renderer");
  if (num_faces) *num_faces = h->F;
  if (num_verts) *num_verts = h->V;
  if (face_bits) *face_bits = h->fbits;
  return MHMR_OK;
}

int mhmr_render_forward(mhmr_render* h, const mhmr_render_args* a, void* stream) {
  MHMR_REQUIRE(h != nullptr && a != nullptr, "null renderer or arguments");
  MHMR_REQUIRE(a->views >= 1 && a->H >= 1 && a->W >= 1, "views, H and W must be positive");
  MHMR_REQUIRE(a->max_persons >= 1, "max_persons must be positive");
  MHMR_REQUIRE(static_cast<long long>(a->max_persons) <= (1ll << (32 - h->fbits)),
               "max_persons does not fit the depth key next to the face index");
  MHMR_REQUIRE(static_cast<long long>(a->views) * a->max_persons <= 65535, "views x max_persons exceeds 65535");
  MHMR_REQUIRE(a->images && a->view_image && a->K && a->verts && a->person_image && a->count && a->colors &&
                   a->overlay,
               "null argument");
  MHMR_REQUIRE(a->alpha >= 0.f && a->alpha <= 1.f, "alpha must lie in [0, 1]");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t npix = static_cast<size_t>(a->views) * a->H * a->W;
  if (grow(&h->keys, &h->key_cap, npix) != MHMR_OK) return MHMR_ERR_CUDA;
  if (a->smooth && grow(&h->normals, &h->normal_cap, static_cast<size_t>(a->max_persons) * h->V * 3) != MHMR_OK)
    return MHMR_ERR_CUDA;
  Params p;
  p.views = a->views; p.H = a->H; p.W = a->W; p.P = a->max_persons; p.F = h->F; p.V = h->V; p.fbits = h->fbits;
  p.smooth = a->smooth ? 1 : 0;
  p.faces = h->faces; p.csr_ptr = h->csr_ptr; p.csr_ent = h->csr_ent;
  p.verts = a->verts; p.person_image = a->person_image; p.view_image = a->view_image; p.count = a->count;
  p.K = a->K; p.pose = a->pose; p.normals = h->normals; p.keys = h->keys; p.queue = h->queue;
  p.queue_count = h->queue_count;
  Shade s;
  s.images = a->images; s.colors = a->colors; s.alpha = a->alpha; s.intensity = a->intensity;
  s.metallic = a->metallic; s.roughness = a->roughness; s.overlay = a->overlay; s.depth = a->depth;
  s.person = a->person;
  const int sms = device_sm_count();
  const size_t prep_work = npix + (a->smooth ? static_cast<size_t>(a->max_persons) * h->V : 0);
  const int prep_blocks = static_cast<int>(std::min<size_t>((prep_work + 255) / 256, static_cast<size_t>(sms) * 16));
  render_prep_kernel<<<prep_blocks, 256, 0, st>>>(p);
  MHMR_CUDA_CHECK(cudaGetLastError());
  render_raster_kernel<<<dim3((h->F + 127) / 128, a->views * a->max_persons), 128, 0, st>>>(p);
  MHMR_CUDA_CHECK(cudaGetLastError());
  render_raster_big_kernel<<<sms * 8, 256, 0, st>>>(p);
  MHMR_CUDA_CHECK(cudaGetLastError());
  render_shade_kernel<<<static_cast<unsigned>((npix + 255) / 256), 256, 0, st>>>(p, s);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // extern "C"
