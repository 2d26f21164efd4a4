// TEST INFRASTRUCTURE: CPU restatement of the world raycast (include/b2d.h b2d_raycast) that the device kernels are
// compared with.  shape_raycast of src/edyn/collision/raycast.cpp for sphere / box / capsule / plane, plus the
// brute-force world query over every body.  Built by tests/raycast_support.py with g++ -ffp-contract=off, so it can be
// compared with the reference and with the device (-fmad=false) bit for bit.
#include "../../oracle/ora_math.hpp"
#include <cstring>

using namespace ora;

namespace {

enum : uint32_t { SH_SPHERE = 0, SH_CAPSULE = 2, SH_BOX = 3, SH_PLANE = 6, SH_NONE = 255 };
constexpr uint32_t RAY_FEATURE_NONE = 0xFFFFFFFFu, RAY_CAPSULE_SIDE = 2u, RAY_MISS = 0xFFFFFFFFu;
struct shape { uint32_t kind; scalar p[4]; };
struct ray_result { bool hit = false; scalar fraction = SCALAR_MAX; vec3 normal{0, 0, 0}; uint32_t feature = RAY_FEATURE_NONE; };

vec3 box_face_normal(size_t f) {                                   // box_shape.cpp:185-196
    static const vec3 n[6] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
    return n[f];
}
void capsule_vertices(const shape &c, vec3 pos, quat orn, vec3 out[2]) {    // shapes/capsule_shape.hpp:21-27
    vec3 ax{0, 0, 0}; ax[(size_t)c.p[2]] = 1;
    vec3 dir = rotate(orn, ax);
    out[0] = pos + dir * c.p[1];
    out[1] = pos - dir * c.p[1];
}
vec3 v3(const float *p) { return {p[0], p[1], p[2]}; }
quat q4(const float *p) { return {p[0], p[1], p[2], p[3]}; }
shape mk_shape(uint32_t kind, const float *p) { shape s; s.kind = kind; for (int i = 0; i < 4; ++i) s.p[i] = p[i]; return s; }

// The reference's fraction / normal / feature, no clamping to [0, 1]; the one change is the capsule hemisphere normal,
// taken at the hit fraction from the hemisphere centre (the reference uses lerp(p0, p1, u_in) - pos, raycast.cpp:217-218).

static bool ray_sphere(vec3 p0, vec3 p1, vec3 pos, scalar radius, scalar &t) {      // geom.cpp:1276-1305
    vec3 d = p1 - p0, m = p0 - pos;
    scalar a = dot(d, d), b = dot(m, d), c = dot(m, m) - radius * radius;
    if (c > 0 && b > 0) return false;
    scalar discr = b * b - a * c;
    if (discr < 0) return false;
    t = (-b - std::sqrt(discr)) / a;
    t = std::max(scalar(0), t);
    return true;
}
static bool line_line(vec3 p1, vec3 q1, vec3 p2, vec3 q2, scalar &s, scalar &t) {   // geom.cpp:46-70
    vec3 d1 = q1 - p1, d2 = q2 - p2, r = p1 - p2;
    scalar a = dot(d1, d1), b = dot(d1, d2), c = dot(d1, r), e = dot(d2, d2), f = dot(d2, r);
    scalar d = a * e - b * b;
    if (!(d > EPS)) return false;
    scalar d_inv = scalar(1) / d;
    s = (b * f - c * e) * d_inv;
    t = (a * f - b * c) * d_inv;
    return true;
}
static vec3 unit(vec3 v) { return v / length(v); }                                  // vector3.hpp:231-235

static ray_result shape_raycast(const shape &sh, vec3 pos, quat orn, vec3 p0, vec3 p1) {
    ray_result r;
    if (sh.kind == SH_SPHERE) {                                                    // raycast.cpp:182-195
        scalar t;
        if (!ray_sphere(p0, p1, pos, sh.p[0], t)) return r;
        r.hit = true; r.fraction = t; r.normal = unit(lerp(p0, p1, t) - pos);
    } else if (sh.kind == SH_BOX) {                                                // raycast.cpp:58-109
        vec3 a = to_object(p0, pos, orn), b = to_object(p1, pos, orn), dir = b - a;
        scalar t_min = -SCALAR_MAX, t_max = SCALAR_MAX;
        size_t face = SIZE_MAX;
        for (size_t i = 0; i < 3; ++i) {
            scalar he = sh.p[i];
            if (std::abs(dir[i]) < EPS) {
                if (std::abs(a[i]) > he) return r;
            } else {
                scalar d_inv = scalar(1) / dir[i];
                scalar t1 = (-he - a[i]) * d_inv, t2 = (he - a[i]) * d_inv;
                if (t1 > t2) std::swap(t1, t2);
                if (t1 > t_min) face = i * 2 + (a[i] > 0 ? 0 : 1);
                t_min = std::max(t_min, t1);
                t_max = std::min(t_max, t2);
                if (t_min > t_max) return r;
            }
        }
        if (face == SIZE_MAX) return r;                                            // get_face_normal(SIZE_MAX) in the reference
        r.hit = true; r.fraction = t_min; r.normal = rotate(orn, box_face_normal(face)); r.feature = uint32_t(face);
    } else if (sh.kind == SH_CAPSULE) {                                            // raycast.cpp:197-257
        scalar radius = sh.p[0];
        vec3 v[2]; capsule_vertices(sh, pos, orn, v);                             // = the cylinder's vertices, geom.cpp:1241-1245
        vec3 cap_dir = v[1] - v[0];
        size_t hemi;
        scalar s, t;
        if (!line_line(v[0], v[1], p0, p1, s, t)) {                                // parallel_directions, geom.cpp:1248-1250
            hemi = dot(p0 - pos, cap_dir) < 0 ? 0 : 1;
        } else {
            scalar radius_sqr = radius * radius;
            vec3 n = lerp(p0, p1, t) - lerp(v[0], v[1], s);
            scalar dist_sqr = length_sqr(n);
            if (dist_sqr > radius_sqr) return r;
            vec3 d = p1 - p0, e = v[1] - v[0];
            scalar dd = dot(d, d), ee = dot(e, e), de = dot(d, e);
            scalar delta_sqr = (radius_sqr - dist_sqr) * ee / (dd * ee - de * de);
            scalar u_in = t - std::sqrt(delta_sqr);
            vec3 x = lerp(p0, p1, u_in);
            scalar pr0 = dot(x - v[0], cap_dir), pr1 = dot(x - v[1], cap_dir);
            if (pr0 > 0 && pr1 < 0) {
                r.hit = true; r.fraction = u_in; r.normal = n / std::sqrt(dist_sqr); r.feature = RAY_CAPSULE_SIDE;
                return r;
            }
            hemi = pr0 < 0 ? 0 : 1;
        }
        scalar f;
        if (!ray_sphere(p0, p1, v[hemi], radius, f)) return r;
        r.hit = true; r.fraction = f; r.normal = unit(lerp(p0, p1, f) - v[hemi]); r.feature = uint32_t(hemi);
    } else if (sh.kind == SH_PLANE) {                                              // raycast.cpp:356-378
        vec3 n{sh.p[0], sh.p[1], sh.p[2]};
        vec3 c = n * sh.p[3];
        scalar d = dot(p1 - p0, n), e = dot(c - p0, n);
        if (std::abs(d) < EPS) {
            if (!(std::abs(e) < EPS)) return r;
            r.fraction = 0;
        } else {
            r.fraction = e / d;
        }
        r.hit = true; r.normal = n;
    }
    return r;
}

} // namespace

extern "C" {

// shape_raycast of one shape: out4 = fraction, normal; *feature.  Returns 1 if the reference reports a result.
int ora_shape_raycast(uint32_t kind, const float *p, const float *pos, const float *orn, const float *p0, const float *p1,
                      float *out4, uint32_t *feature) {
    ray_result r = shape_raycast(mk_shape(kind, p), v3(pos), q4(orn), v3(p0), v3(p1));
    out4[0] = r.fraction; out4[1] = r.normal.x; out4[2] = r.normal.y; out4[3] = r.normal.z; *feature = r.feature;
    return r.hit ? 1 : 0;
}
// The world raycast as a brute force over nb bodies (pos 3, orn 4, shape kind, shape params 4 per body; kind 255 = no
// shape / removed): hits with 0 <= f <= 1, smallest f, equal fractions to the smaller id; zero-length and non-finite
// segments hit nothing.
void ora_world_raycast(uint32_t nb, const float *pos, const float *orn, const uint32_t *shape_kind, const float *params,
                       uint32_t n, const float *p0, const float *p1, const uint32_t *ignore_body, const uint32_t *ignore_list,
                       uint32_t nignore, uint32_t *body, float *fraction, float *normal, uint32_t *feature) {
    for (uint32_t i = 0; i < n; ++i) {
        vec3 a = v3(p0 + 3 * i), b = v3(p1 + 3 * i);
        uint32_t best = RAY_MISS; ray_result br;
        bool finite = true;
        for (size_t k = 0; k < 3; ++k) finite = finite && std::isfinite(a[k]) && std::isfinite(b[k]);
        if (finite && !(a.x == b.x && a.y == b.y && a.z == b.z)) {
            for (uint32_t j = 0; j < nb; ++j) {
                if (shape_kind[j] == SH_NONE || (ignore_body && ignore_body[i] == j)) continue;
                bool skip = false;
                for (uint32_t k = 0; k < nignore; ++k) skip = skip || ignore_list[k] == j;
                if (skip) continue;
                ray_result r = shape_raycast(mk_shape(shape_kind[j], params + 4 * j), v3(pos + 3 * j), q4(orn + 4 * j), a, b);
                if (!r.hit || !(r.fraction >= 0 && r.fraction <= 1)) continue;
                if (best == RAY_MISS || r.fraction < br.fraction) { best = j; br = r; }
            }
        }
        body[i] = best; fraction[i] = br.fraction;
        normal[3 * i] = br.normal.x; normal[3 * i + 1] = br.normal.y; normal[3 * i + 2] = br.normal.z; feature[i] = br.feature;
    }
}

} // extern "C"
