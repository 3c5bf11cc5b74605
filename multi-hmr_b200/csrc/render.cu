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

// ---- props: extra meshes of other topologies in the same z-buffer ------------------------------------------------
// Prop j is mesh P + j of the key.  Its topology's faces and CSR sit in the handle's concatenated topology arrays;
// the per-prop offsets travel by value.
struct Props {
  int n, total_faces, total_verts;
  int face_off[MHMR_RENDER_MAX_PROPS], nf[MHMR_RENDER_MAX_PROPS];   // into faces (in faces), of the topology
  int ptr_off[MHMR_RENDER_MAX_PROPS], nv[MHMR_RENDER_MAX_PROPS];    // into csr_ptr, vertices of the topology
  int vert_off[MHMR_RENDER_MAX_PROPS], fsum[MHMR_RENDER_MAX_PROPS]; // into verts / normals; faces of props < j
  const int* faces;
  const int* csr_ptr;
  const int* csr_ent;
  const float* verts;
  const float* colors;
  const unsigned char* visible;
  float* normals;
};

__device__ __forceinline__ int prop_of_vertex(const Props& q, int i) {
  int j = 0;
  while (j + 1 < q.n && q.vert_off[j + 1] <= i) ++j;
  return j;
}

__device__ __forceinline__ int prop_of_face(const Props& q, int i) {
  int j = 0;
  while (j + 1 < q.n && q.fsum[j + 1] <= i) ++j;
  return j;
}

// Vertex normals of the props, as render_prep_kernel computes the persons'.
__global__ void render_prop_normals_kernel(Props q) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= q.total_verts) return;
  const int j = prop_of_vertex(q, i), v = i - q.vert_off[j];
  const float* vp = q.verts + static_cast<size_t>(q.vert_off[j]) * 3;
  const int* faces = q.faces + 3ll * q.face_off[j];
  const int* ptr = q.csr_ptr + q.ptr_off[j];
  float3 acc = make_float3(0.f, 0.f, 0.f);
  for (int e = ptr[v]; e < ptr[v + 1]; ++e) {
    const int ent = q.csr_ent[e], f = ent / 3, corner = ent % 3;
    const int* fc = faces + 3 * f;
    const float3 p0 = load3(vp + 3 * fc[corner]), p1 = load3(vp + 3 * fc[(corner + 1) % 3]),
                 p2 = load3(vp + 3 * fc[(corner + 2) % 3]);
    const float3 fn = cross3(sub3(p1, p0), sub3(p2, p0));
    const float3 u = sub3(p1, p0), w = sub3(p2, p0);
    const float ang = atan2f(sqrtf(dot3(fn, fn)), dot3(u, w));
    const float3 un = normalize3(fn);
    acc.x = fmaf(ang, un.x, acc.x); acc.y = fmaf(ang, un.y, acc.y); acc.z = fmaf(ang, un.z, acc.z);
  }
  const float3 n = normalize3(acc);
  float* out = q.normals + static_cast<size_t>(i) * 3;
  out[0] = n.x; out[1] = n.y; out[2] = n.z;
}

// One CTA per (prop face, view): props are few faces, often large on screen (a glyph next to the camera).
__global__ void __launch_bounds__(128) render_prop_raster_kernel(Params a, Props q) {
  const int b = blockIdx.y, j = prop_of_face(q, blockIdx.x), f = blockIdx.x - q.fsum[j];
  if (q.visible && !q.visible[static_cast<size_t>(b) * q.n + j]) return;
  const Cam c = load_cam(a.K, a.pose, b);
  if (!(c.fx > 0.f) || !(c.fy > 0.f)) return;
  Tri T;
  if (!tri_setup(q.verts + static_cast<size_t>(q.vert_off[j]) * 3, q.faces + 3ll * (q.face_off[j] + f), c, a.W, a.H,
                 T))
    return;
  raster_box(a, T, c, b, (static_cast<unsigned int>(a.P + j) << a.fbits) | f, threadIdx.x, blockDim.x);
}

// ---- 4. shading + composite -------------------------------------------------------------------------------------
struct Shade {
  const unsigned char* images;
  const float* colors;
  float alpha, intensity, metallic, roughness;
  unsigned char* overlay;
  float* depth;
  int* person;
  const float* view_alpha;      // kExtra only: per-view alpha, or null
  const int* view_background;   // kExtra only: per-view background image, or null
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

// kExtra: props, per-view alpha and backgrounds (mhmr_render_forward_extra); without, the one-topology path.
template <bool kExtra>
__global__ void __launch_bounds__(256) render_shade_kernel(Params a, Shade s, Props q) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long hw = static_cast<long long>(a.H) * a.W;
  if (i >= a.views * hw) return;
  const int b = static_cast<int>(i / hw), pix = static_cast<int>(i % hw), y = pix / a.W, x = pix % a.W;
  const unsigned long long* keys = a.keys + b * hw;
  const unsigned long long key = keys[pix];
  const int bg_image = kExtra && s.view_background ? s.view_background[b] : a.view_image[b];
  const float alpha = kExtra && s.view_alpha ? s.view_alpha[b] : s.alpha;
  const unsigned char* bg = s.images + (static_cast<size_t>(bg_image) * hw + pix) * 3;
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
  const float* vn_base = a.normals + static_cast<size_t>(p) * a.V * 3;
  const float* col = s.colors + 3 * p;
  if (kExtra && p >= a.P) {
    const int j = p - a.P;
    vp = q.verts + static_cast<size_t>(q.vert_off[j]) * 3;
    fc = q.faces + 3ll * (q.face_off[j] + f);
    vn_base = q.normals + static_cast<size_t>(q.vert_off[j]) * 3;
    col = q.colors + 3 * j;
  }
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
      const float3 vn = load3(vn_base + static_cast<size_t>(fc[k]) * 3);
      const float w = e[k] * inv;
      acc.x = fmaf(w, vn.x, acc.x); acc.y = fmaf(w, vn.y, acc.y); acc.z = fmaf(w, vn.z, acc.z);
    }
    n = normalize3(rotate(c, acc));
  } else {
    n = normalize3(cross3(sub3(T.p[1], T.p[0]), sub3(T.p[2], T.p[0])));
  }
  const float3 v = normalize3(make_float3(-rx * z, -ry * z, -z));
  const float3 rgb = shade_pbr(n, v, make_float3(col[0], col[1], col[2]), s.intensity, s.metallic, s.roughness);
  const float rgbv[3] = {rgb.x, rgb.y, rgb.z};
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float r8 = rintf(rgbv[ch] * 255.f);
    const float im = static_cast<float>(bg[ch]);
    const float o = fg * (alpha * r8 + (1.f - alpha) * im) + (1.f - fg) * im;
    out[ch] = static_cast<unsigned char>(fminf(fmaxf(o, 0.f), 255.f));
  }
  if (s.depth) s.depth[i] = z;
  if (s.person) s.person[i] = p;
}

// ---- view poses of the demo (demo.py:160-241, utils/render.py:329-448) ------------------------------------------
constexpr int kPoseThreads = 256;
constexpr int kMaxPosePersons = 4096;

__device__ void put_pose(float* out, const double (&R)[9], const double (&t)[3]) {
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) out[4 * r + k] = static_cast<float>(R[3 * r + k]);
    out[4 * r + 3] = static_cast<float>(t[r]);
  }
}

// utils/render.py:lookAt with up (0, -1, 0) and normalisation v / (|v| + 1e-13), then OPENCV_TO_OPENGL @ view:
// rows x, -y, z_forward of the camera frame and t = -R eye.
__device__ void look_at(const double (&eye)[3], const double (&at)[3], float* out) {
  auto normalize = [](double (&v)[3]) {
    const double l = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]) + 1e-13;
    v[0] = v[0] / l; v[1] = v[1] / l; v[2] = v[2] / l;
  };
  double z[3] = {at[0] - eye[0], at[1] - eye[1], at[2] - eye[2]};
  normalize(z);
  const double up[3] = {0.0, -1.0, 0.0};
  double x[3] = {z[1] * up[2] - up[1] * z[2], z[2] * up[0] - up[2] * z[0], z[0] * up[1] - up[0] * z[1]};
  normalize(x);
  const double y[3] = {x[1] * z[2] - z[1] * x[2], x[2] * z[0] - z[2] * x[0], x[0] * z[1] - z[0] * x[1]};
  const double R[9] = {x[0], x[1], x[2], -y[0], -y[1], -y[2], z[0], z[1], z[2]};
  double t[3];
  for (int r = 0; r < 3; ++r) t[r] = -(R[3 * r] * eye[0] + R[3 * r + 1] * eye[1] + R[3 * r + 2] * eye[2]);
  put_pose(out, R, t);
}

struct PoseArgs {
  int images, P, V, n_frames, side, vpi;
  double angle_range;
  const int* count;
  const int* person_image;
  const float* verts;
  const float* transl_pelvis;
  const float* transl;
  float* pose;
  unsigned char* nonempty;
  int* rank;
};

// One CTA per image.  Each thread takes persons p strided and counts, over all persons q of the image, those listed
// before p (its rank: list order, or stable by transl z) and those with a smaller pelvis depth (its slot in the
// sorted depths, ties by index): O(n^2 / threads) per image, no serial sort.  All threads then sum the first
// person's vertices in fp64, strided, and reduce in a fixed-order tree: the centroid is bitwise repeatable.
__global__ void __launch_bounds__(kPoseThreads) render_pose_kernel(PoseArgs a) {
  extern __shared__ double sh[];  // [3][kPoseThreads] partial sums, then [P] sorted depths
  __shared__ int s_first, s_cnt;
  double* zs = sh + 3 * kPoseThreads;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = min(max(*a.count, 0), a.P);
  if (b == 0)
    for (int p = tid; p < a.P; p += blockDim.x)
      if (p >= n || a.person_image[p] < 0 || a.person_image[p] >= a.images) a.rank[p] = -1;
  if (tid == 0) {
    s_first = -1;
    s_cnt = 0;
  }
  __syncthreads();
  for (int p = tid; p < n; p += blockDim.x) {
    if (a.person_image[p] != b) continue;
    const float zp = a.transl ? a.transl[3 * p + 2] : 0.f;
    const float tp = a.transl_pelvis ? a.transl_pelvis[3 * p + 2] : 0.f;
    int r = 0, slot = 0;
    for (int q = 0; q < n; ++q) {
      if (a.person_image[q] != b) continue;
      if (a.transl) {
        const float zq = a.transl[3 * q + 2];
        r += zq < zp || (zq == zp && q < p);
      } else {
        r += q < p;
      }
      if (a.transl_pelvis) {
        const float tq = a.transl_pelvis[3 * q + 2];
        slot += tq < tp || (tq == tp && q < p);
      }
    }
    a.rank[p] = r;
    if (r == 0) s_first = p;  // the ranks of an image are a permutation: one writer
    if (a.transl_pelvis) zs[slot] = static_cast<double>(tp);
    atomicAdd(&s_cnt, 1);
  }
  __syncthreads();
  if (tid == 0) a.nonempty[b] = s_cnt > 0 ? 1 : 0;
  const int first = s_first, cnt = s_cnt;
  double acc[3] = {0.0, 0.0, 0.0};
  if (first >= 0) {
    const float* vp = a.verts + static_cast<size_t>(first) * a.V * 3;
    for (int v = tid; v < a.V; v += blockDim.x)
      for (int k = 0; k < 3; ++k) acc[k] += static_cast<double>(vp[3 * v + k]);
  }
  for (int k = 0; k < 3; ++k) sh[k * kPoseThreads + tid] = acc[k];
  __syncthreads();
  for (int s = kPoseThreads / 2; s > 0; s >>= 1) {
    if (tid < s)
      for (int k = 0; k < 3; ++k) sh[k * kPoseThreads + tid] += sh[k * kPoseThreads + tid + s];
    __syncthreads();
  }
  if (tid != 0) return;
  float* out = a.pose + static_cast<size_t>(b) * a.vpi * 12;
  const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, zero[3] = {0, 0, 0};
  for (int w = 0; w < a.vpi; ++w) put_pose(out + 12 * w, I, zero);
  if (cnt == 0) return;
  const double c[3] = {sh[0] / a.V, sh[kPoseThreads] / a.V, sh[2 * kPoseThreads] / a.V};
  int w = 1;
  if (a.n_frames >= 2) {
    const double kDeg = 3.141592653589793 / 180.0;  // np.deg2rad
    for (int sweep = 0; sweep < 3; ++sweep) {
      const double range = sweep == 1 ? -a.angle_range : a.angle_range;
      for (int i = 0; i < a.n_frames; ++i, ++w) {
        const double th = range * i / (a.n_frames - 1) * kDeg, co = cos(th), si = sin(th);
        double R[9];
        if (sweep < 2) {
          const double Ry[9] = {co, 0, si, 0, 1, 0, -si, 0, co};
          for (int k = 0; k < 9; ++k) R[k] = Ry[k];
        } else {
          const double Rx[9] = {1, 0, 0, 0, co, -si, 0, si, co};
          for (int k = 0; k < 9; ++k) R[k] = Rx[k];
        }
        double t[3];
        for (int r = 0; r < 3; ++r) t[r] = c[r] - (R[3 * r] * c[0] + R[3 * r + 1] * c[1] + R[3 * r + 2] * c[2]);
        put_pose(out + 12 * w, R, t);
      }
    }
  }
  if (a.side) {
    const double zt = (cnt % 2) ? zs[cnt / 2] : (zs[cnt / 2 - 1] + zs[cnt / 2]) / 2.0;  // np.median
    const double e0[3] = {2.0, -1.0, -2.0}, t0[3] = {0.0, 0.0, 3.0};
    const double e1[3] = {2.2 * zt, 0.0, zt}, e2[3] = {0.0, -2.0 * zt, zt - 0.001}, tz[3] = {0.0, 0.0, zt};
    look_at(e0, t0, out + 12 * w);
    look_at(e1, tz, out + 12 * (w + 1));
    look_at(e2, tz, out + 12 * (w + 2));
  }
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
  // extra topologies: faces (local indices) and CSR back to back; per topology, host offsets
  int* topo_faces = nullptr;
  int* topo_ptr = nullptr;
  int* topo_ent = nullptr;
  float* prop_normals = nullptr;
  size_t prop_normal_cap = 0;
  std::vector<int> topo_face_off, topo_nf, topo_ptr_off, topo_nv;
  ~mhmr_render() {
    for (void* p : {static_cast<void*>(faces), static_cast<void*>(csr_ptr), static_cast<void*>(csr_ent),
                    static_cast<void*>(queue), static_cast<void*>(queue_count), static_cast<void*>(keys),
                    static_cast<void*>(normals), static_cast<void*>(topo_faces), static_cast<void*>(topo_ptr),
                    static_cast<void*>(topo_ent), static_cast<void*>(prop_normals)})
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

// vertex -> incident (face, corner) entries, faces in increasing order; ptr values offset by `base`
void build_csr(const int32_t* hf, int F, int V, int base, std::vector<int32_t>& ptr, std::vector<int32_t>& ent) {
  const size_t p0 = ptr.size(), e0 = ent.size();
  ptr.resize(p0 + V + 1, 0);
  ent.resize(e0 + 3ll * F);
  for (int i = 0; i < 3 * F; ++i) ++ptr[p0 + hf[i] + 1];
  for (int v = 0; v < V; ++v) ptr[p0 + v + 1] += ptr[p0 + v];
  std::vector<int32_t> fill(ptr.begin() + p0, ptr.begin() + p0 + V);
  for (int i = 0; i < 3 * F; ++i) ent[e0 + fill[hf[i]]++] = i;
  for (size_t i = p0; i < ptr.size(); ++i) ptr[i] += base;
}

int render_build_topologies(mhmr_render* h, const int32_t* topo_faces, int total_faces, cudaStream_t st) {
  std::vector<int32_t> hf(3ll * total_faces), ptr, ent;
  MHMR_CUDA_CHECK(cudaMemcpy(hf.data(), topo_faces, 12ll * total_faces, cudaMemcpyDefault));
  for (size_t t = 0; t < h->topo_nf.size(); ++t) {
    const int32_t* f = hf.data() + 3ll * h->topo_face_off[t];
    for (int i = 0; i < 3 * h->topo_nf[t]; ++i)
      MHMR_REQUIRE(f[i] >= 0 && f[i] < h->topo_nv[t], "topology face vertex index outside [0, its num_verts)");
    h->topo_ptr_off.push_back(static_cast<int>(ptr.size()));
    build_csr(f, h->topo_nf[t], h->topo_nv[t], static_cast<int>(ent.size()), ptr, ent);
  }
  MHMR_CUDA_CHECK(cudaMalloc(&h->topo_faces, 12ll * total_faces));
  MHMR_CUDA_CHECK(cudaMalloc(&h->topo_ptr, 4ll * ptr.size()));
  MHMR_CUDA_CHECK(cudaMalloc(&h->topo_ent, 4ll * ent.size()));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(h->topo_faces, hf.data(), 12ll * total_faces, cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(h->topo_ptr, ptr.data(), 4ll * ptr.size(), cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaMemcpyAsync(h->topo_ent, ent.data(), 4ll * ent.size(), cudaMemcpyHostToDevice, st));
  MHMR_CUDA_CHECK(cudaStreamSynchronize(st));
  return MHMR_OK;
}

int render_build(mhmr_render* h, const int32_t* faces, cudaStream_t st) {
  const int F = h->F, V = h->V;
  std::vector<int32_t> hf(3ll * F);
  MHMR_CUDA_CHECK(cudaMemcpy(hf.data(), faces, 12ll * F, cudaMemcpyDefault));
  for (int32_t v : hf) MHMR_REQUIRE(v >= 0 && v < V, "face vertex index outside [0, num_verts)");
  std::vector<int32_t> ptr, ent;
  build_csr(hf.data(), F, V, 0, ptr, ent);
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

int mhmr_render_create_topologies(const int32_t* faces, int num_faces, int num_verts, int num_topologies,
                                  const int32_t* topo_faces, const int32_t* topo_num_faces,
                                  const int32_t* topo_num_verts, void* stream, mhmr_render** out) {
  MHMR_REQUIRE(out != nullptr, "null output handle");
  *out = nullptr;
  MHMR_REQUIRE(faces != nullptr, "null faces");
  MHMR_REQUIRE(num_faces >= 1 && num_verts >= 3, "need at least one face and three vertices");
  MHMR_REQUIRE(num_topologies >= 0, "negative topology count");
  MHMR_REQUIRE(num_topologies == 0 || (topo_faces && topo_num_faces && topo_num_verts), "null topology argument");
  long long max_faces = num_faces, total = 0;
  for (int t = 0; t < num_topologies; ++t) {
    MHMR_REQUIRE(topo_num_faces[t] >= 1 && topo_num_verts[t] >= 3,
                 "a topology needs at least one face and three vertices");
    max_faces = std::max<long long>(max_faces, topo_num_faces[t]);
    total += topo_num_faces[t];
  }
  MHMR_REQUIRE(total < (1ll << 31) / 3, "too many topology faces");
  int fbits = 0;
  while ((1ll << fbits) < max_faces) ++fbits;
  MHMR_REQUIRE(fbits <= 24, "at most 2^24 faces (the depth key keeps 32 bits for mesh and face)");
  auto* h = new mhmr_render();
  h->F = num_faces; h->V = num_verts; h->fbits = fbits; h->nnz = 3 * num_faces;
  for (int t = 0, off = 0; t < num_topologies; off += topo_num_faces[t++]) {
    h->topo_face_off.push_back(off);
    h->topo_nf.push_back(topo_num_faces[t]);
    h->topo_nv.push_back(topo_num_verts[t]);
  }
  int rc = render_build(h, faces, static_cast<cudaStream_t>(stream));
  if (rc == MHMR_OK && num_topologies > 0)
    rc = render_build_topologies(h, topo_faces, static_cast<int>(total), static_cast<cudaStream_t>(stream));
  if (rc != MHMR_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return MHMR_OK;
}

int mhmr_render_create(const int32_t* faces, int num_faces, int num_verts, void* stream, mhmr_render** out) {
  return mhmr_render_create_topologies(faces, num_faces, num_verts, 0, nullptr, nullptr, nullptr, stream, out);
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

int mhmr_render_forward_extra(mhmr_render* h, const mhmr_render_args* a, const mhmr_render_extra* e,
                              void* stream) {
  MHMR_REQUIRE(h != nullptr && a != nullptr, "null renderer or arguments");
  MHMR_REQUIRE(a->views >= 1 && a->H >= 1 && a->W >= 1, "views, H and W must be positive");
  MHMR_REQUIRE(a->max_persons >= 1, "max_persons must be positive");
  const int nprops = e ? e->num_props : 0;
  MHMR_REQUIRE(nprops >= 0 && nprops <= MHMR_RENDER_MAX_PROPS, "at most MHMR_RENDER_MAX_PROPS props");
  MHMR_REQUIRE(static_cast<long long>(a->max_persons) + nprops <= (1ll << (32 - h->fbits)),
               "max_persons does not fit the depth key next to the face index");
  Props q{};
  if (nprops > 0) {
    MHMR_REQUIRE(e->prop_topology && e->prop_verts && e->prop_colors, "null prop argument");
    q.n = nprops;
    for (int j = 0; j < nprops; ++j) {
      const int t = e->prop_topology[j];
      MHMR_REQUIRE(t >= 0 && t < static_cast<int>(h->topo_nf.size()), "prop topology outside the handle's");
      q.face_off[j] = h->topo_face_off[t]; q.nf[j] = h->topo_nf[t];
      q.ptr_off[j] = h->topo_ptr_off[t]; q.nv[j] = h->topo_nv[t];
      q.vert_off[j] = q.total_verts; q.fsum[j] = q.total_faces;
      q.total_verts += q.nv[j]; q.total_faces += q.nf[j];
    }
    q.faces = h->topo_faces; q.csr_ptr = h->topo_ptr; q.csr_ent = h->topo_ent;
    q.verts = e->prop_verts; q.colors = e->prop_colors; q.visible = e->prop_visible;
  }
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
  if (nprops > 0 && a->smooth &&
      grow(&h->prop_normals, &h->prop_normal_cap, static_cast<size_t>(q.total_verts) * 3) != MHMR_OK)
    return MHMR_ERR_CUDA;
  q.normals = h->prop_normals;
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
  s.view_alpha = e ? e->view_alpha : nullptr;
  s.view_background = e ? e->view_background : nullptr;
  const int sms = device_sm_count();
  const size_t prep_work = npix + (a->smooth ? static_cast<size_t>(a->max_persons) * h->V : 0);
  const int prep_blocks = static_cast<int>(std::min<size_t>((prep_work + 255) / 256, static_cast<size_t>(sms) * 16));
  render_prep_kernel<<<prep_blocks, 256, 0, st>>>(p);
  MHMR_CUDA_CHECK(cudaGetLastError());
  render_raster_kernel<<<dim3((h->F + 127) / 128, a->views * a->max_persons), 128, 0, st>>>(p);
  MHMR_CUDA_CHECK(cudaGetLastError());
  if (nprops > 0) {
    if (a->smooth) {
      render_prop_normals_kernel<<<(q.total_verts + 255) / 256, 256, 0, st>>>(q);
      MHMR_CUDA_CHECK(cudaGetLastError());
    }
    render_prop_raster_kernel<<<dim3(q.total_faces, a->views), 128, 0, st>>>(p, q);
    MHMR_CUDA_CHECK(cudaGetLastError());
  }
  render_raster_big_kernel<<<sms * 8, 256, 0, st>>>(p);
  MHMR_CUDA_CHECK(cudaGetLastError());
  const unsigned shade_blocks = static_cast<unsigned>((npix + 255) / 256);
  if (e)
    render_shade_kernel<true><<<shade_blocks, 256, 0, st>>>(p, s, q);
  else
    render_shade_kernel<false><<<shade_blocks, 256, 0, st>>>(p, s, q);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

int mhmr_render_forward(mhmr_render* h, const mhmr_render_args* a, void* stream) {
  return mhmr_render_forward_extra(h, a, nullptr, stream);
}

int mhmr_render_view_poses(const mhmr_render_pose_args* a, void* stream) {
  MHMR_REQUIRE(a != nullptr, "null arguments");
  MHMR_REQUIRE(a->images >= 1 && a->max_persons >= 1 && a->num_verts >= 1,
               "images, max_persons and num_verts must be positive");
  MHMR_REQUIRE(a->max_persons <= kMaxPosePersons, "at most 4096 persons");
  MHMR_REQUIRE(a->n_frames == 0 || a->n_frames >= 2, "n_frames must be 0 (no orbit) or at least 2");
  MHMR_REQUIRE(a->n_frames <= 10000, "n_frames above 10000");
  MHMR_REQUIRE(a->count && a->person_image && a->verts && a->pose && a->nonempty && a->rank, "null argument");
  MHMR_REQUIRE(!a->side || a->transl_pelvis, "the side views need transl_pelvis");
  PoseArgs p;
  p.images = a->images; p.P = a->max_persons; p.V = a->num_verts; p.n_frames = a->n_frames;
  p.side = a->side ? 1 : 0;
  p.vpi = 1 + 3 * a->n_frames + 3 * p.side;
  p.angle_range = a->angle_range;
  p.count = a->count; p.person_image = a->person_image; p.verts = a->verts; p.transl_pelvis = a->transl_pelvis;
  p.transl = a->transl; p.pose = a->pose; p.nonempty = a->nonempty; p.rank = a->rank;
  const size_t smem = sizeof(double) * (3 * kPoseThreads + a->max_persons);
  if (smem > 48 * 1024)
    MHMR_CUDA_CHECK(cudaFuncSetAttribute(render_pose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem)));
  render_pose_kernel<<<a->images, kPoseThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
  MHMR_CUDA_CHECK(cudaGetLastError());
  return MHMR_OK;
}

}  // extern "C"
