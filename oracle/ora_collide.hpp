// TEST INFRASTRUCTURE -- CPU oracle (see ora_math.hpp header).
// Narrowphase restatement: closest-feature contact generation for the primitive pairs
// the hot-path scope covers (SURVEY.md section 8a rows N2/N3).
#pragma once
#include "ora_math.hpp"

namespace ora {

// Values follow the reference's shape_index order (include/edyn/shapes/shapes.hpp:23-37).
enum shape_kind : uint32_t { SH_SPHERE = 0, SH_CAPSULE = 2, SH_BOX = 3, SH_PLANE = 6, SH_NONE = 255 };
// include/edyn/collision/contact_normal_attachment.hpp:16-20
enum attachment : uint32_t { ATT_NONE = 0, ATT_A = 1, ATT_B = 2 };

// sphere: p = {r}; capsule: p = {r, half_length, axis(0/1/2)}; box: p = half extents;
// plane: p = {nx, ny, nz, constant}.
struct shape { uint32_t kind; scalar p[4]; };

struct cpoint {            // collision_result::collision_point, collision_result.hpp:14-21 (features omitted)
    vec3 pivotA, pivotB, normal;
    scalar distance;
    uint32_t att;
};
struct cresult {           // collision_result.hpp:37-50
    size_t num = 0;
    cpoint pt[4];
};
struct cctx {              // collision_context, collide.hpp:11-27
    vec3 posA; quat ornA; aabb bbA;
    vec3 posB; quat ornB; aabb bbB;
    scalar threshold;
};

constexpr size_t MAX_CONTACTS = 4;                    // config/constants.hpp:9
constexpr scalar COLLISION_THRESHOLD = scalar(0.01);  // :15
constexpr scalar BREAKING_THRESHOLD = scalar(0.02);   // :21
constexpr scalar MERGING_THRESHOLD = scalar(0.01);    // :27
constexpr scalar CACHING_THRESHOLD = scalar(0.04);    // :34
constexpr scalar FEATURE_TOL = scalar(0.005);         // :56 support_feature_tolerance

enum insert_type { INS_NONE, INS_SIMILAR, INS_REPLACE, INS_APPEND };
struct insert_res { insert_type type; size_t index; };

// geometry helpers (src/edyn/math/geom.cpp)
void plane_space(vec3 n, vec3 &p, vec3 &q);
size_t intersect_line_aabb(vec2 p0, vec2 p1, vec2 bmin, vec2 bmax, scalar &s0, scalar &s1);
scalar closest_point_segment(vec3 q0, vec3 q1, vec3 p, scalar &t, vec3 &q);
scalar closest_point_segment_segment(vec3 p1, vec3 q1, vec3 p2, vec3 q2, scalar &s, scalar &t,
                                     vec3 &c1, vec3 &c2, size_t *num_points = nullptr,
                                     scalar *sp = nullptr, scalar *tp = nullptr,
                                     vec3 *c1p = nullptr, vec3 *c2p = nullptr);
// collinear (optional, merge tests): which branch of the collinear three-point case decided, 0-3 = d0, d1, d2, shortest edge
insert_res insertion_point_index(const vec3 *points, size_t count, size_t &num_points, vec3 new_point, int *collinear = nullptr);
void maybe_add_point(cresult &r, const cpoint &np);

// box feature helpers (src/edyn/shapes/box_shape.cpp)
enum box_feature { BF_VERTEX, BF_EDGE, BF_FACE };
void box_support_feature(vec3 he, vec3 dir, box_feature &f, size_t &idx, scalar &proj, scalar tol);

// shape AABBs (src/edyn/util/aabb_util.cpp)
aabb shape_aabb(const shape &sh, vec3 pos, quat orn);

// dispatch (src/edyn/util/collision_util.cpp:440-475 minus the registry lookups)
void collide(const shape &a, const shape &b, const cctx &ctx, cresult &r);
// Full detect_collision incl. the AABB early-out of collision_util.cpp:444-474.
void detect_collision(const shape &a, const shape &b, vec3 posA, quat ornA, const aabb &bbA,
                      vec3 posB, quat ornB, const aabb &bbB, cresult &r);

} // namespace ora
