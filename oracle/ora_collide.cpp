// TEST INFRASTRUCTURE -- CPU oracle (see ora_math.hpp header).
// Each function cites the reference file:line (relative to /root/reference) it restates.
#include "ora_collide.hpp"
#include <array>

namespace ora {

// ---------------------------------------------------------------- geom.cpp helpers

// src/edyn/math/geom.cpp:730-754
void plane_space(vec3 n, vec3 &p, vec3 &q) {
    if (std::abs(n.z) > HALF_SQRT2) {
        scalar a = n.y * n.y + n.z * n.z;
        scalar k = scalar(1) / std::sqrt(a);
        p.x = 0; p.y = -n.z * k; p.z = n.y * k;
        q.x = a * k; q.y = -n.x * p.z; q.z = n.x * p.y;
    } else {
        scalar a = n.x * n.x + n.y * n.y;
        scalar k = scalar(1) / std::sqrt(a);
        p.x = -n.y * k; p.y = n.x * k; p.z = 0;
        q.x = -n.z * p.y; q.y = n.z * p.x; q.z = a * k;
    }
}

// src/edyn/math/geom.cpp:12-22
scalar closest_point_segment(vec3 q0, vec3 q1, vec3 p, scalar &t, vec3 &q) {
    vec3 v = q1 - q0;
    vec3 w = p - q0;
    scalar a = dot(w, v);
    scalar b = dot(v, v);
    t = clamp_unit(a / b);
    q = q0 + v * t;
    return length_sqr(p - q);
}

// src/edyn/math/geom.cpp:36-45
static scalar closest_point_line(vec3 q0, vec3 dir, vec3 p, scalar &t, vec3 &r) {
    vec3 w = p - q0;
    scalar a = dot(w, dir);
    scalar b = dot(dir, dir);
    t = a / b;
    r = q0 + dir * t;
    return length_sqr(p - r);
}

// src/edyn/math/geom.cpp:73-170
scalar closest_point_segment_segment(vec3 p1, vec3 q1, vec3 p2, vec3 q2, scalar &s, scalar &t,
                                     vec3 &c1, vec3 &c2, size_t *num_points,
                                     scalar *sp, scalar *tp, vec3 *c1p, vec3 *c2p) {
    const vec3 d1 = q1 - p1;
    const vec3 d2 = q2 - p2;
    const vec3 r = p1 - p2;
    const scalar a = dot(d1, d1);
    const scalar e = dot(d2, d2);
    const scalar f = dot(d2, r);

    if (a <= EPS && e <= EPS) {
        s = t = 0;
        c1 = p1; c2 = p2;
        return length_sqr(c1 - c2);
    }
    if (a <= EPS) {
        s = 0;
        t = f / e;
        t = clamp_unit(t);
    } else {
        scalar c = dot(d1, r);
        if (e <= EPS) {
            t = 0;
            s = clamp_unit(-c / a);
        } else {
            const scalar b = dot(d1, d2);
            const scalar denom = a * e - b * b;
            if (denom > EPS) {
                s = clamp_unit((b * f - c * e) / denom);
                if (num_points != nullptr) *num_points = 1;
            } else if (num_points != nullptr) {
                vec3 r1 = p1 - q2;
                scalar f1 = dot(d1, r1);
                scalar a_inv = 1 / a;
                s = clamp_unit(std::min(-c * a_inv, -f1 * a_inv));
                *sp = clamp_unit(std::max(-c * a_inv, -f1 * a_inv));
                vec3 r2 = p2 - q1;
                scalar f2 = dot(d2, r2);
                scalar e_inv = 1 / e;
                t = clamp_unit(std::min(-f * e_inv, -f2 * e_inv));
                *tp = clamp_unit(std::max(-f * e_inv, -f2 * e_inv));
                if (std::abs(s - *sp) > EPS) {
                    *num_points = 2;
                    *c1p = p1 + d1 * *sp;
                    *c2p = p2 + d2 * *tp;
                } else {
                    *num_points = 1;
                }
            } else {
                s = 0;
            }
            const scalar tnom = b * s + f;
            if (tnom < 0) {
                t = 0;
                s = clamp_unit(-c / a);
            } else if (tnom > e) {
                t = 1;
                s = clamp_unit((b - c) / a);
            } else {
                t = tnom / e;
            }
        }
    }
    c1 = p1 + d1 * s;
    c2 = p2 + d2 * t;
    return length_sqr(c1 - c2);
}

// src/edyn/math/geom.cpp:1044-1138
size_t intersect_line_aabb(vec2 p0, vec2 p1, vec2 bmin, vec2 bmax, scalar &s0, scalar &s1) {
    size_t n = 0;
    vec2 d = p1 - p0;
    vec2 e = bmin - p0;
    vec2 f = bmax - p0;
    if (std::abs(d.x) < EPS) {
        if (e.x <= 0 && f.x >= 0) { s0 = e.y / d.y; s1 = f.y / d.y; n = 2; }
        return n;
    }
    if (std::abs(d.y) < EPS) {
        if (e.y <= 0 && f.y >= 0) { s0 = e.x / d.x; s1 = f.x / d.x; n = 2; }
        return n;
    }
    { // left edge
        scalar t = e.x / d.x;
        scalar qy = p0.y + d.y * t;
        if (qy >= bmin.y && qy < bmax.y) { s0 = t; ++n; }
    }
    { // right edge
        scalar t = f.x / d.x;
        scalar qy = p0.y + d.y * t;
        if (qy > bmin.y && qy <= bmax.y) {
            if (n == 0) { s0 = t; ++n; }
            else if (std::abs(t - s0) > EPS) { s1 = t; ++n; }
        }
    }
    if (n == 2) return n;
    { // bottom edge
        scalar t = e.y / d.y;
        scalar qx = p0.x + d.x * t;
        if (qx >= bmin.x && qx < bmax.x) {
            if (n == 0) { s0 = t; ++n; }
            else if (std::abs(t - s0) > EPS) { s1 = t; ++n; }
        }
    }
    if (n == 2) return n;
    { // top edge
        scalar t = f.y / d.y;
        scalar qx = p0.x + d.x * t;
        if (qx > bmin.x && qx <= bmax.x) {
            if (n == 0) { s0 = t; ++n; }
            else if (std::abs(t - s0) > EPS) { s1 = t; ++n; }
        }
    }
    return n;
}

// include/edyn/math/geom.hpp:330-348 (N = 4)
static bool point_in_quad_prism(const vec3 v[4], vec3 normal, vec3 point) {
    for (size_t i = 0; i < 4; ++i) {
        size_t j = (i + 1) % 4;
        vec3 d = v[j] - v[i];
        vec3 t = cross(d, normal);
        if (dot(point - v[i], t) > EPS) return false;
    }
    return true;
}

// src/edyn/math/triangle.cpp:7-26
static bool point_in_triangle(const vec3 v[3], vec3 normal, vec3 p) {
    vec3 e0 = v[1] - v[0], e1 = v[2] - v[1], e2 = v[0] - v[2];
    vec3 q0 = p - v[0], q1 = p - v[1], q2 = p - v[2];
    vec3 en0 = cross(e0, normal), en1 = cross(e1, normal), en2 = cross(e2, normal);
    scalar d0 = dot(en0, q0), d1 = dot(en1, q1), d2 = dot(en2, q2);
    return (d0 > -EPS && d1 > -EPS && d2 > -EPS) || (d0 < EPS && d1 < EPS && d2 < EPS);
}

// src/edyn/math/geom.cpp:847-856
static scalar manifold_score(vec3 p0, vec3 p1, vec3 p2, vec3 p3) {
    vec3 c0 = cross(p0 - p1, p0 - p2);
    vec3 c1 = cross(p0 - p2, p0 - p3);
    vec3 c2 = cross(p0 - p3, p0 - p1);
    vec3 c3 = cross(p1 - p2, p2 - p3);
    return length_sqr(c0) + length_sqr(c1) + length_sqr(c2) + length_sqr(c3);
}

// src/edyn/math/geom.cpp:857-985
insert_res insertion_point_index(const vec3 *points, size_t count, size_t &num_points, vec3 new_point, int *collinear) {
    const scalar max_dist_similar_sqr = MERGING_THRESHOLD * MERGING_THRESHOLD;
    if (num_points == 0) return {INS_APPEND, num_points++};
    if (num_points == 1) {
        if (distance_sqr(new_point, points[0]) > max_dist_similar_sqr) return {INS_APPEND, num_points++};
        return {INS_SIMILAR, 0};
    }
    if (num_points == 2) {
        if (length_sqr(cross(new_point - points[0], new_point - points[1])) > EPS) {
            return {INS_APPEND, num_points++};
        }
        scalar d0 = distance_sqr(new_point, points[0]);
        scalar d1 = distance_sqr(new_point, points[1]);
        scalar cur = distance_sqr(points[0], points[1]);
        if (d0 > cur && d0 > d1) return {d1 < max_dist_similar_sqr ? INS_SIMILAR : INS_REPLACE, 1};
        if (d1 > cur && d1 > d0) return {d0 < max_dist_similar_sqr ? INS_SIMILAR : INS_REPLACE, 0};
        return {INS_NONE, count};
    }
    if (num_points == 3) {
        vec3 verts[3] = {points[0], points[1], points[2]};
        vec3 normal = cross(points[0] - points[1], points[1] - points[2]);
        if (try_normalize(normal)) {
            if (std::abs(dot(new_point - points[0], normal)) < EPS && point_in_triangle(verts, normal, new_point)) {
                return {INS_NONE, count};
            }
            return {INS_APPEND, num_points++};
        }
        scalar d0 = dot(points[1] - points[0], points[2] - points[0]);
        if (d0 > 0 && d0 < 1) { if (collinear) *collinear = 0; return {INS_REPLACE, 1}; }
        scalar d1 = dot(points[0] - points[1], points[2] - points[1]);
        if (d1 > 0 && d1 < 1) { if (collinear) *collinear = 1; return {INS_REPLACE, 0}; }
        scalar d2 = dot(points[2] - points[0], points[1] - points[0]);
        if (d2 > 0 && d2 < 1) { if (collinear) *collinear = 2; return {INS_REPLACE, 2}; }
        if (collinear) *collinear = 3;
        scalar ds[3] = {distance_sqr(points[0], points[1]), distance_sqr(points[1], points[2]),
                        distance_sqr(points[2], points[0])};
        size_t mi = SIZE_MAX; scalar md = SCALAR_MAX;
        for (size_t i = 0; i < 3; ++i) if (ds[i] < md) { md = ds[i]; mi = i; }
        return {INS_REPLACE, mi};
    }
    scalar scores[4];
    scores[0] = manifold_score(new_point, points[1], points[2], points[3]);
    scores[1] = manifold_score(new_point, points[0], points[2], points[3]);
    scores[2] = manifold_score(new_point, points[0], points[1], points[3]);
    scores[3] = manifold_score(new_point, points[0], points[1], points[2]);
    scalar max_score = manifold_score(points[0], points[1], points[2], points[3]);
    size_t max_idx = SIZE_MAX;
    for (size_t i = 0; i < 4; ++i) if (scores[i] > max_score) { max_score = scores[i]; max_idx = i; }
    if (max_idx < MAX_CONTACTS) {
        return {distance_sqr(points[max_idx], new_point) < max_dist_similar_sqr ? INS_SIMILAR : INS_REPLACE, max_idx};
    }
    return {INS_NONE, count};
}

// src/edyn/collision/collision_result.cpp:12-33
void maybe_add_point(cresult &r, const cpoint &np) {
    vec3 pivots[4];
    for (size_t i = 0; i < r.num; ++i) pivots[i] = r.pt[i].pivotA;
    insert_res res = insertion_point_index(pivots, 4, r.num, np.pivotA);
    if (res.type == INS_NONE) {
        for (size_t i = 0; i < r.num; ++i) pivots[i] = r.pt[i].pivotB;
        res = insertion_point_index(pivots, 4, r.num, np.pivotB);
    }
    if (res.type != INS_NONE) r.pt[res.index] = np;
}
static void add_point(cresult &r, const cpoint &np) { r.pt[r.num++] = np; }   // collision_result.cpp:6-10

// src/edyn/math/geom.cpp:987-996
static vec3 closest_point_box_outside(vec3 he, vec3 p) {
    vec3 c = p;
    c.x = std::min(he.x, c.x); c.x = std::max(-he.x, c.x);
    c.y = std::min(he.y, c.y); c.y = std::max(-he.y, c.y);
    c.z = std::min(he.z, c.z); c.z = std::max(-he.z, c.z);
    return c;
}
// src/edyn/math/geom.cpp:998-1042 -- NB: returns the LAST `dist`, not `min_dist`, as the reference does.
static scalar closest_point_box_inside(vec3 he, vec3 p, vec3 &closest, vec3 &normal) {
    scalar dist = he.x - p.x;
    scalar min_dist = dist;
    closest = {he.x, p.y, p.z}; normal = {1, 0, 0};
    dist = he.x + p.x;
    if (dist < min_dist) { min_dist = dist; closest = {-he.x, p.y, p.z}; normal = {-1, 0, 0}; }
    dist = he.y - p.y;
    if (dist < min_dist) { min_dist = dist; closest = {p.x, he.y, p.z}; normal = {0, 1, 0}; }
    dist = he.y + p.y;
    if (dist < min_dist) { min_dist = dist; closest = {p.x, -he.y, p.z}; normal = {0, -1, 0}; }
    dist = he.z - p.z;
    if (dist < min_dist) { min_dist = dist; closest = {p.x, p.y, he.z}; normal = {0, 0, 1}; }
    dist = he.z + p.z;
    if (dist < min_dist) { min_dist = dist; closest = {p.x, p.y, -he.z}; normal = {0, 0, -1}; }
    return dist;
}

// ---------------------------------------------------------------- box_shape.cpp helpers

static const size_t BOX_EDGE_IDX[24] = {0,1, 1,2, 2,3, 3,0, 4,5, 5,6, 6,7, 7,4, 0,4, 1,7, 2,6, 3,5};  // box_shape.hpp:22-35
static const size_t BOX_FACE_IDX[24] = {0,1,2,3, 4,5,6,7, 0,3,5,4, 1,7,6,2, 0,4,7,1, 3,2,6,5};        // box_shape.hpp:37-44

static vec3 box_vertex(vec3 he, size_t i) {                     // box_shape.cpp:115-128
    static const vec3 mult[8] = {{1,1,1},{1,-1,1},{1,-1,-1},{1,1,-1},{-1,1,1},{-1,1,-1},{-1,-1,-1},{-1,-1,1}};
    return he * mult[i];
}
static vec3 box_support_point(vec3 he, vec3 dir) {               // util/shape_util.cpp:40-46
    return {dir.x > 0 ? he.x : -he.x, dir.y > 0 ? he.y : -he.y, dir.z > 0 ? he.z : -he.z};
}
static scalar box_support_projection(vec3 he, vec3 pos, quat orn, vec3 dir) {   // box_shape.cpp:24-28
    vec3 ld = rotate(conjugate(orn), dir);
    vec3 pt = box_support_point(he, ld);
    return dot(pos, dir) + dot(pt, ld);
}
static size_t box_edge_index(size_t v0, size_t v1) {             // box_shape.cpp:228-242
    for (size_t i = 0; i < 12; ++i) {
        size_t a = BOX_EDGE_IDX[i * 2], b = BOX_EDGE_IDX[i * 2 + 1];
        if ((a == v0 && b == v1) || (b == v0 && a == v1)) return i;
    }
    return SIZE_MAX;
}
static size_t box_support_face(vec3 dir) {                       // box_shape.cpp:244-252
    size_t m = max_index_abs(dir);
    return dir[m] < 0 ? m * 2 + 1 : m * 2;
}
// box_shape.cpp:30-96
void box_support_feature(vec3 he, vec3 dir, box_feature &feature, size_t &feature_index, scalar &projection, scalar threshold) {
    size_t face = box_support_face(dir);
    scalar proj[4];
    projection = -SCALAR_MAX;
    size_t vidx[4];
    size_t indices[4];
    size_t count = 1;
    size_t max_i = 0;
    for (size_t i = 0; i < 4; ++i) {
        size_t vi = BOX_FACE_IDX[face * 4 + i];
        vidx[i] = vi;
        scalar p = dot(box_vertex(he, vi), dir);
        proj[i] = p;
        if (p > projection) { projection = p; indices[0] = i; max_i = i; }
    }
    for (size_t i = 0; i < 4; ++i) {
        if (i != max_i && proj[i] > projection - threshold) indices[count++] = i;
    }
    if (count == 1) {
        feature = BF_VERTEX; feature_index = vidx[indices[0]];
    } else if (count == 2) {
        feature = BF_EDGE; feature_index = box_edge_index(vidx[indices[0]], vidx[indices[1]]);
    } else if (count == 3) {
        feature = BF_EDGE;
        scalar p0 = proj[indices[0]], p1 = proj[indices[1]], p2 = proj[indices[2]];
        if (p0 <= p1 && p0 <= p2) feature_index = box_edge_index(vidx[indices[1]], vidx[indices[2]]);
        else if (p1 <= p0 && p1 <= p2) feature_index = box_edge_index(vidx[indices[0]], vidx[indices[2]]);
        else feature_index = box_edge_index(vidx[indices[0]], vidx[indices[1]]);
    } else {
        feature = BF_FACE; feature_index = face;
    }
}
// box_shape.cpp:98-105
static void box_support_feature_w(vec3 he, vec3 pos, quat orn, vec3 axis_pos, vec3 axis_dir,
                                  box_feature &f, size_t &idx, scalar &proj, scalar tol) {
    vec3 ld = rotate(conjugate(orn), axis_dir);
    box_support_feature(he, ld, f, idx, proj, tol);
    proj += dot(pos - axis_pos, axis_dir);
}
static vec3 box_face_normal(size_t f) {                           // box_shape.cpp:178-188
    static const vec3 n[6] = {{1,0,0},{-1,0,0},{0,1,0},{0,-1,0},{0,0,1},{0,0,-1}};
    return n[f];
}
static vec3 box_face_tangent(size_t f) {                          // box_shape.cpp:163-175
    static const vec3 t[6] = {{0,0,1},{0,0,-1},{1,0,0},{-1,0,0},{0,1,0},{0,-1,0}};
    return t[f];
}
static void box_face_world(vec3 he, size_t f, vec3 pos, quat orn, vec3 out[4]) {   // box_shape.cpp:143-161
    for (size_t i = 0; i < 4; ++i) out[i] = to_world(box_vertex(he, BOX_FACE_IDX[f * 4 + i]), pos, orn);
}
static void box_edge_world(vec3 he, size_t e, vec3 pos, quat orn, vec3 out[2]) {   // box_shape.cpp:130-141
    out[0] = to_world(box_vertex(he, BOX_EDGE_IDX[e * 2]), pos, orn);
    out[1] = to_world(box_vertex(he, BOX_EDGE_IDX[e * 2 + 1]), pos, orn);
}
static vec3 box_face_center(vec3 he, size_t f, vec3 pos, quat orn) {               // box_shape.cpp:194-198
    vec3 n = rotate(orn, box_face_normal(f));
    return pos + n * he[f / 2];
}
static mat3 box_face_basis(size_t f, quat orn) {                                    // box_shape.cpp:200-205
    vec3 y = box_face_normal(f), x = box_face_tangent(f), z = cross(x, y);
    return mat3_columns(rotate(orn, x), rotate(orn, y), rotate(orn, z));
}
static vec2 box_face_half_extents(vec3 he, size_t f) {                              // box_shape.cpp:207-217
    if (f == 0 || f == 1) return {he.z, he.y};
    if (f == 2 || f == 3) return {he.x, he.z};
    return {he.y, he.x};
}

// ---------------------------------------------------------------- aabb_util.cpp

aabb shape_aabb(const shape &sh, vec3 pos, quat orn) {
    switch (sh.kind) {
    case SH_SPHERE: {                                   // util/aabb_util.cpp:65-70
        scalar r = sh.p[0];
        return {{pos.x - r, pos.y - r, pos.z - r}, {pos.x + r, pos.y + r, pos.z + r}};
    }
    case SH_CAPSULE: {                                  // util/aabb_util.cpp:81-88
        vec3 ax{0, 0, 0}; ax[(size_t)sh.p[2]] = 1;
        vec3 dir = rotate(orn, ax);
        vec3 v = dir * sh.p[1];
        vec3 p0 = pos - v, p1 = pos + v;
        vec3 off{sh.p[0], sh.p[0], sh.p[0]};
        return {vmin(p0, p1) - off, vmax(p0, p1) + off};
    }
    case SH_BOX: {                                      // util/aabb_util.cpp:42-63
        aabb bb{pos, pos};
        mat3 basis = to_mat3(orn);
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
            scalar e = basis.row[i][j] * -sh.p[j];
            scalar f = -e;
            if (e < f) { bb.min[i] += e; bb.max[i] += f; }
            else { bb.min[i] += f; bb.max[i] += e; }
        }
        return bb;
    }
    case SH_PLANE: {                                    // util/aabb_util.cpp:9-40
        const scalar H = 99999;
        vec3 n{sh.p[0], sh.p[1], sh.p[2]};
        vec3 umin{-1, -1, -1}, umax{1, 1, 1};
        if (n == vec3{1, 0, 0}) umax.x = 0;
        else if (n == vec3{-1, 0, 0}) umin.x = 0;
        else if (n == vec3{0, 1, 0}) umax.y = 0;
        else if (n == vec3{0, -1, 0}) umin.y = 0;
        else if (n == vec3{0, 0, 1}) umax.z = 0;
        else if (n == vec3{0, 0, -1}) umin.z = 0;
        vec3 pw = n * sh.p[3];
        return {umin * H + pw, umax * H + pw};
    }
    default: return {pos, pos};
    }
}

// ---------------------------------------------------------------- collide_*.cpp

static void capsule_vertices(const shape &c, vec3 pos, quat orn, vec3 out[2]) {    // shapes/capsule_shape.hpp:21-27
    vec3 ax{0, 0, 0}; ax[(size_t)c.p[2]] = 1;
    vec3 dir = rotate(orn, ax);
    out[0] = pos + dir * c.p[1];
    out[1] = pos - dir * c.p[1];
}
static scalar capsule_support_projection(const vec3 v[2], scalar radius, vec3 dir) {   // util/shape_util.cpp:297-300
    return std::max(dot(v[0], dir), dot(v[1], dir)) + radius;
}

// collision/collide/collide_sphere_sphere.cpp:5-27
static void sphere_sphere(const shape &A, const shape &B, const cctx &c, cresult &r) {
    vec3 d = c.posA - c.posB;
    scalar dist_sqr = length_sqr(d);
    scalar rr = A.p[0] + B.p[0] + c.threshold;
    if (dist_sqr > rr * rr) return;
    scalar dist = std::sqrt(dist_sqr);
    vec3 dn = dist > EPS ? d / dist : vec3{1, 0, 0};
    vec3 rA = -dn * A.p[0];
    rA = rotate(conjugate(c.ornA), rA);
    vec3 rB = dn * B.p[0];
    rB = rotate(conjugate(c.ornB), rB);
    add_point(r, {rA, rB, dn, dist - A.p[0] - B.p[0], ATT_NONE});
}

// collision/collide/collide_sphere_plane.cpp:5-20
static void sphere_plane(const shape &S, const shape &P, const cctx &c, cresult &r) {
    vec3 normal{P.p[0], P.p[1], P.p[2]};
    vec3 center = normal * P.p[3];
    vec3 d = c.posA - center;
    scalar l = dot(normal, d);
    if (l > S.p[0]) return;
    vec3 pivotA = rotate(conjugate(c.ornA), -normal * S.p[0]);
    vec3 pivotB = rotate(conjugate(c.ornB), d - normal * l - center);
    add_point(r, {pivotA, pivotB, normal, l - S.p[0], ATT_B});
}

// collision/collide/collide_box_plane.cpp:7-56
static void box_plane(const shape &Bx, const shape &P, const cctx &c, cresult &r) {
    vec3 he{Bx.p[0], Bx.p[1], Bx.p[2]};
    vec3 n{P.p[0], P.p[1], P.p[2]};
    vec3 center = n * P.p[3];
    box_feature fA; size_t fiA; scalar projA;
    box_support_feature_w(he, c.posA, c.ornA, center, -n, fA, fiA, projA, FEATURE_TOL);
    scalar distance = -projA;
    if (distance > c.threshold) return;
    vec3 verts[4]; size_t nv = 0;
    switch (fA) {
    case BF_VERTEX: verts[0] = box_vertex(he, fiA); nv = 1; break;
    case BF_EDGE: verts[0] = box_vertex(he, BOX_EDGE_IDX[fiA * 2]); verts[1] = box_vertex(he, BOX_EDGE_IDX[fiA * 2 + 1]); nv = 2; break;
    case BF_FACE: for (size_t i = 0; i < 4; ++i) verts[i] = box_vertex(he, BOX_FACE_IDX[fiA * 4 + i]); nv = 4; break;
    }
    cpoint pt{};
    pt.normal = n; pt.distance = distance; pt.att = ATT_B;
    for (size_t i = 0; i < nv; ++i) {
        pt.pivotA = verts[i];
        vec3 pAw = to_world(pt.pivotA, c.posA, c.ornA);
        vec3 pBw = project_plane(pAw, center, n);
        pt.pivotB = to_object(pBw, c.posB, c.ornB);
        pt.distance = dot(pAw - pBw, n);
        add_point(r, pt);
    }
}

// collision/collide/collide_capsule_plane.cpp:6-38
static void capsule_plane(const shape &C, const shape &P, const cctx &c, cresult &r) {
    vec3 n{P.p[0], P.p[1], P.p[2]};
    vec3 center = n * P.p[3];
    vec3 cv[2]; capsule_vertices(C, c.posA, c.ornA, cv);
    scalar proj[2] = {dot(cv[0] - center, n), dot(cv[1] - center, n)};
    for (int i = 0; i < 2; ++i) {
        scalar distance = proj[i] - C.p[0];
        if (distance > c.threshold) continue;
        vec3 vertex = cv[i];
        vec3 pAw = vertex - n * C.p[0];
        vec3 pivotA = to_object(pAw, c.posA, c.ornA);
        vec3 pivotB = project_plane(vertex, center, n);   // left in world space, as the reference does (:35-36)
        add_point(r, {pivotA, pivotB, n, distance, ATT_B});
    }
}

// collision/collide/collide_sphere_box.cpp:7-55
static void sphere_box(const shape &S, const shape &Bx, const cctx &c, cresult &r) {
    vec3 he{Bx.p[0], Bx.p[1], Bx.p[2]};
    const quat ornB_conj = conjugate(c.ornB);
    const vec3 posA_in_B = rotate(ornB_conj, c.posA - c.posB);
    const quat ornA_in_B = ornB_conj * c.ornA;
    vec3 closest = closest_point_box_outside(he, posA_in_B);
    vec3 normalB = posA_in_B - closest;
    scalar d_sqr = length_sqr(normalB);
    scalar min_dist = S.p[0] + c.threshold;
    if (d_sqr > min_dist * min_dist) return;
    scalar center_distance;
    uint32_t att = ATT_NONE;
    if (d_sqr <= EPS) {
        center_distance = -closest_point_box_inside(he, posA_in_B, closest, normalB);
        att = ATT_B;
    } else {
        center_distance = std::sqrt(d_sqr);
        normalB /= center_distance;
        if (std::abs(normalB.x) > scalar(1) - EPS || std::abs(normalB.y) > scalar(1) - EPS ||
            std::abs(normalB.z) > scalar(1) - EPS) att = ATT_B;
    }
    vec3 pivotA_in_B = posA_in_B - normalB * S.p[0];
    vec3 pivotA = to_object(pivotA_in_B, posA_in_B, ornA_in_B);
    vec3 normal = rotate(c.ornB, normalB);
    add_point(r, {pivotA, closest, normal, center_distance - S.p[0], att});
}

// collision/collide/collide_capsule_capsule.cpp:7-81
static void capsule_capsule(const shape &A, const shape &B, const cctx &c, cresult &r) {
    vec3 vA[2], vB[2];
    capsule_vertices(A, c.posA, c.ornA, vA);
    capsule_vertices(B, c.posB, c.ornB, vB);
    scalar s[2], t[2]; vec3 cA[2], cB[2]; size_t np = 0;
    scalar dist_sqr = closest_point_segment_segment(vA[0], vA[1], vB[0], vB[1], s[0], t[0], cA[0], cB[0], &np,
                                                    &s[1], &t[1], &cA[1], &cB[1]);
    scalar min_dist = A.p[0] + B.p[0] + c.threshold;
    if (dist_sqr > min_dist * min_dist) return;
    vec3 normal; scalar distance;
    if (dist_sqr > EPS) {
        scalar dist = std::sqrt(dist_sqr);
        normal = (cA[0] - cB[0]) / dist;
        distance = dist - A.p[0] - B.p[0];
    } else {
        vec3 axA = vA[1] - vA[0], axB = vB[1] - vB[0];
        normal = cross(axA, axB);
        if (dot(c.posA - c.posB, normal) < 0) normal *= -1;
        if (!try_normalize(normal)) normal = {0, 1, 0};
        distance = -(A.p[0] + B.p[0]);
    }
    cpoint pt{}; pt.normal = normal; pt.distance = distance; pt.att = ATT_NONE;
    for (size_t i = 0; i < np; ++i) {
        vec3 pAw = cA[i] - normal * A.p[0];
        vec3 pBw = cB[i] + normal * B.p[0];
        pt.pivotA = to_object(pAw, c.posA, c.ornA);
        pt.pivotB = to_object(pBw, c.posB, c.ornB);
        add_point(r, pt);
    }
}

// collision/collide/collide_capsule_sphere.cpp:10-52
static void capsule_sphere(const shape &C, const shape &S, const cctx &c, cresult &r) {
    vec3 cv[2]; capsule_vertices(C, c.posA, c.ornA, cv);
    vec3 closest; scalar t;
    scalar dist_sqr = closest_point_segment(cv[0], cv[1], c.posB, t, closest);
    scalar min_dist = C.p[0] + S.p[0] + c.threshold;
    if (dist_sqr > min_dist * min_dist) return;
    vec3 normal = closest - c.posB;
    scalar nls = length_sqr(normal);
    scalar distance;
    if (nls > EPS) {
        scalar nl = std::sqrt(nls);
        normal /= nl;
        distance = nl - C.p[0] - S.p[0];
    } else {
        normal = quat_z(c.ornA);
        distance = -(C.p[0] + S.p[0]);
    }
    cpoint pt{};
    vec3 normalB = rotate(conjugate(c.ornB), normal);
    vec3 pAw = closest - normal * C.p[0];
    pt.pivotA = to_object(pAw, c.posA, c.ornA);
    pt.pivotB = normalB * S.p[0];
    pt.normal = normal; pt.distance = distance; pt.att = ATT_NONE;
    add_point(r, pt);
}

// collision/collide/collide_capsule_box.cpp:14-213
static void capsule_box(const shape &C, const shape &Bx, const cctx &c, cresult &r) {
    vec3 he{Bx.p[0], Bx.p[1], Bx.p[2]};
    const vec3 posA{0, 0, 0};
    const quat ornA = c.ornA;
    const vec3 posB = c.posB - c.posA;
    const quat ornB = c.ornB;
    vec3 cv[2]; capsule_vertices(C, posA, ornA, cv);
    const vec3 axes[3] = {quat_x(ornB), quat_y(ornB), quat_z(ornB)};
    scalar distance = -SCALAR_MAX, projection_box = -SCALAR_MAX;
    vec3 sep{0, 0, 0};
    for (size_t i = 0; i < 3; ++i) {
        vec3 dir = axes[i];
        if (dot(posA - posB, dir) < 0) dir = -dir;
        scalar projA = -capsule_support_projection(cv, C.p[0], -dir);
        scalar projB = dot(posB, dir) + he[i];
        scalar dist = projA - projB;
        if (dist > distance) { distance = dist; projection_box = projB; sep = dir; }
    }
    for (size_t i = 0; i < 12; ++i) {
        vec3 ev[2]; box_edge_world(he, i, posB, ornB, ev);
        scalar s, t; vec3 cA, cB;
        closest_point_segment_segment(ev[0], ev[1], cv[0], cv[1], s, t, cA, cB);
        vec3 dir = cA - cB;
        if (!try_normalize(dir)) continue;
        if (dot(posA - posB, dir) < 0) dir *= -1;
        scalar projA = -capsule_support_projection(cv, C.p[0], -dir);
        scalar projB = box_support_projection(he, posB, ornB, dir);
        scalar dist = projA - projB;
        if (dist > distance) { distance = dist; projection_box = projB; sep = dir; }
    }
    if (distance > c.threshold) return;
    scalar pcv[2] = {dot(cv[0], sep), dot(cv[1], sep)};
    bool is_edge = std::abs(pcv[0] - pcv[1]) < FEATURE_TOL;
    vec3 origin_box = sep * projection_box;
    scalar fdistB; box_feature fB; size_t fiB;
    box_support_feature_w(he, posB, ornB, origin_box, sep, fB, fiB, fdistB, FEATURE_TOL);
    cpoint pt{}; pt.normal = sep; pt.distance = distance;
    switch (fB) {
    case BF_FACE: {
        vec3 fv[4]; box_face_world(he, fiB, posB, ornB, fv);
        pt.att = ATT_B;
        if (is_edge) {
            for (int k = 0; k < 2; ++k) {
                vec3 pA = cv[k];
                if (point_in_quad_prism(fv, sep, pA)) {
                    pt.pivotA = to_object(pA - sep * C.p[0], posA, ornA);
                    vec3 pBw = project_plane(pA, origin_box, sep);
                    pt.pivotB = to_object(pBw, posB, ornB);
                    add_point(r, pt);
                }
            }
            if (r.num == 2) return;
            vec3 fc = box_face_center(he, fiB, posB, ornB);
            mat3 fb = box_face_basis(fiB, ornB);
            vec2 hx = box_face_half_extents(he, fiB);
            vec3 o0 = to_object(cv[0], fc, fb), o1 = to_object(cv[1], fc, fb);
            vec2 p0{o0.x, o0.z}, p1{o1.x, o1.z};
            scalar s[2];
            size_t np = intersect_line_aabb(p0, p1, -hx, hx, s[0], s[1]);
            for (size_t i = 0; i < np; ++i) {
                if (s[i] < 0 || s[i] > 1) continue;
                vec3 ep = lerp(cv[0], cv[1], s[i]);
                vec3 fp = project_plane(ep, fc, sep);
                pt.pivotA = to_object(ep - sep * C.p[0], posA, ornA);
                pt.pivotB = to_object(fp, posB, ornB);
                add_point(r, pt);
            }
        } else {
            vec3 ccv = pcv[0] < pcv[1] ? cv[0] : cv[1];
            vec3 pAw = ccv - sep * C.p[0];
            vec3 pBw = project_plane(pAw, origin_box, sep);
            pt.pivotA = to_object(pAw, posA, ornA);
            pt.pivotB = to_object(pBw, posB, ornB);
            add_point(r, pt);
        }
        break;
    }
    case BF_EDGE: {
        vec3 ev[2]; box_edge_world(he, fiB, posB, ornB, ev);
        pt.att = ATT_NONE;
        if (is_edge) {
            scalar s[2], t[2]; vec3 cA[2], cB[2]; size_t np = 0;
            closest_point_segment_segment(cv[0], cv[1], ev[0], ev[1], s[0], t[0], cA[0], cB[0], &np,
                                          &s[1], &t[1], &cA[1], &cB[1]);
            for (size_t i = 0; i < np; ++i) {
                pt.pivotA = to_object(cA[i] - sep * C.p[0], posA, ornA);
                pt.pivotB = to_object(cB[i], posB, ornB);
                add_point(r, pt);
            }
        } else {
            vec3 ccv = pcv[0] < pcv[1] ? cv[0] : cv[1];
            vec3 edir = ev[1] - ev[0];
            vec3 pBw; scalar t;
            closest_point_line(ev[0], edir, ccv, t, pBw);
            pt.pivotB = to_object(pBw, posB, ornB);
            pt.pivotA = to_object(ccv - sep * C.p[0], posA, ornA);
            add_point(r, pt);
        }
        break;
    }
    case BF_VERTEX: {
        pt.pivotB = box_vertex(he, fiB);
        vec3 pBw = to_world(pt.pivotB, posB, ornB);
        vec3 pAw = pBw + sep * distance;
        pt.pivotA = to_object(pAw, posA, ornA);
        pt.att = ATT_NONE;
        add_point(r, pt);
        break;
    }
    }
}

// collision/collide/collide_box_box.cpp:14-266
static void box_box(const shape &A, const shape &B, const cctx &c, cresult &r) {
    vec3 heA{A.p[0], A.p[1], A.p[2]}, heB{B.p[0], B.p[1], B.p[2]};
    const vec3 posA = c.posA, posB = c.posB;
    const quat ornA = c.ornA, ornB = c.ornB;
    vec3 axA[3] = {quat_x(ornA), quat_y(ornA), quat_z(ornA)};
    vec3 axB[3] = {quat_x(ornB), quat_y(ornB), quat_z(ornB)};
    scalar distance = -SCALAR_MAX;
    vec3 sep{0, 0, 0};
    for (size_t i = 0; i < 3; ++i) {
        vec3 dir = axA[i];
        if (dot(posA - posB, dir) < 0) dir = -dir;
        scalar projA = dot(posA, dir) - heA[i];
        scalar projB = box_support_projection(heB, posB, ornB, dir);
        scalar dist = projA - projB;
        if (dist > distance) { distance = dist; sep = dir; }
    }
    for (size_t i = 0; i < 3; ++i) {
        vec3 dir = axB[i];
        if (dot(posA - posB, dir) < 0) dir = -dir;
        scalar projA = -box_support_projection(heA, posA, ornA, -dir);
        scalar projB = dot(posB, dir) + heB[i];
        scalar dist = projA - projB;
        if (dist > distance) { distance = dist; sep = dir; }
    }
    for (size_t i = 0; i < 3; ++i) for (size_t j = 0; j < 3; ++j) {
        vec3 dir = cross(axA[i], axB[j]);
        scalar dls = length_sqr(dir);
        if (!(dls > EPS)) continue;
        dir /= std::sqrt(dls);
        if (dot(posA - posB, dir) < 0) dir *= -1;
        scalar projA = -box_support_projection(heA, posA, ornA, -dir);
        scalar projB = box_support_projection(heB, posB, ornB, dir);
        scalar dist = projA - projB;
        if (dist > distance) { distance = dist; sep = dir; }
    }
    if (distance > c.threshold) return;

    box_feature fA, fB; size_t fiA, fiB; scalar prA, prB;
    box_support_feature_w(heA, posA, ornA, vec3{0, 0, 0}, -sep, fA, fiA, prA, FEATURE_TOL);
    box_support_feature_w(heB, posB, ornB, vec3{0, 0, 0}, sep, fB, fiB, prB, FEATURE_TOL);

    cpoint pt{}; pt.normal = sep; pt.distance = distance; pt.att = ATT_NONE;

    if (fA == BF_FACE && fB == BF_FACE) {
        vec3 fvA[4], fvB[4];
        box_face_world(heA, fiA, posA, ornA, fvA);
        vec3 fnA = rotate(ornA, box_face_normal(fiA));
        box_face_world(heB, fiB, posB, ornB, fvB);
        vec3 fnB = rotate(ornB, box_face_normal(fiB));
        pt.att = ATT_B;
        for (size_t i = 0; i < 4; ++i) {
            if (point_in_quad_prism(fvA, fnA, fvB[i])) {
                vec3 pf = project_plane(fvB[i], fvA[0], fnA);
                pt.pivotA = to_object(pf, posA, ornA);
                pt.pivotB = to_object(fvB[i], posB, ornB);
                maybe_add_point(r, pt);
            }
        }
        for (size_t i = 0; i < 4; ++i) {
            if (point_in_quad_prism(fvB, fnB, fvA[i])) {
                vec3 pf = project_plane(fvA[i], fvB[0], fnB);
                pt.pivotA = to_object(fvA[i], posA, ornA);
                pt.pivotB = to_object(pf, posB, ornB);
                maybe_add_point(r, pt);
            }
        }
        if (r.num < 4) {
            vec3 fc = box_face_center(heA, fiA, posA, ornA);
            mat3 fb = box_face_basis(fiA, ornA);
            vec2 hx = box_face_half_extents(heA, fiA);
            for (size_t j = 0; j < 4; ++j) {
                vec3 b0w = fvB[j], b1w = fvB[(j + 1) % 4];
                vec3 b0 = to_object(b0w, fc, fb), b1 = to_object(b1w, fc, fb);
                vec2 p0{b0.x, b0.z}, p1{b1.x, b1.z};
                scalar s[2];
                size_t np = intersect_line_aabb(p0, p1, -hx, hx, s[0], s[1]);
                for (size_t k = 0; k < np; ++k) {
                    if (s[k] < 0 || s[k] > 1) continue;
                    vec3 q1 = lerp(b0w, b1w, s[k]);
                    vec3 q0 = project_plane(q1, fc, fnA);
                    pt.pivotA = to_object(q0, posA, ornA);
                    pt.pivotB = to_object(q1, posB, ornB);
                    maybe_add_point(r, pt);
                }
            }
        }
    } else if ((fA == BF_FACE && fB == BF_EDGE) || (fB == BF_FACE && fA == BF_EDGE)) {
        const bool faceA = fA == BF_FACE;
        vec3 fn = faceA ? rotate(ornA, box_face_normal(fiA)) : rotate(ornB, box_face_normal(fiB));
        vec3 fv[4], ev[2];
        if (faceA) { box_face_world(heA, fiA, posA, ornA, fv); box_edge_world(heB, fiB, posB, ornB, ev); }
        else { box_face_world(heB, fiB, posB, ornB, fv); box_edge_world(heA, fiA, posA, ornA, ev); }
        pt.att = faceA ? ATT_A : ATT_B;
        for (int i = 0; i < 2; ++i) {
            if (point_in_quad_prism(fv, fn, ev[i])) {
                vec3 pf = project_plane(ev[i], fv[0], fn);
                pt.pivotA = faceA ? to_object(pf, posA, ornA) : to_object(ev[i], posA, ornA);
                pt.pivotB = faceA ? to_object(ev[i], posB, ornB) : to_object(pf, posB, ornB);
                add_point(r, pt);
            }
        }
        if (r.num < 2) {
            vec3 fc = faceA ? box_face_center(heA, fiA, posA, ornA) : box_face_center(heB, fiB, posB, ornB);
            mat3 fb = faceA ? box_face_basis(fiA, ornA) : box_face_basis(fiB, ornB);
            vec2 hx = faceA ? box_face_half_extents(heA, fiA) : box_face_half_extents(heB, fiB);
            vec3 e0 = to_object(ev[0], fc, fb), e1 = to_object(ev[1], fc, fb);
            vec2 p0{e0.x, e0.z}, p1{e1.x, e1.z};
            scalar s[2];
            size_t np = intersect_line_aabb(p0, p1, -hx, hx, s[0], s[1]);
            for (size_t i = 0; i < np; ++i) {
                if (s[i] < 0 || s[i] > 1) continue;
                vec3 ep = lerp(ev[0], ev[1], s[i]);
                vec3 fp = project_plane(ep, fc, sep);
                pt.pivotA = to_object(faceA ? fp : ep, posA, ornA);
                pt.pivotB = to_object(faceA ? ep : fp, posB, ornB);
                add_point(r, pt);
            }
        }
    } else if (fA == BF_EDGE && fB == BF_EDGE) {
        scalar s[2], t[2]; vec3 p0[2], p1[2]; size_t np = 0;
        vec3 eA[2], eB[2];
        box_edge_world(heA, fiA, posA, ornA, eA);
        box_edge_world(heB, fiB, posB, ornB, eB);
        closest_point_segment_segment(eA[0], eA[1], eB[0], eB[1], s[0], t[0], p0[0], p1[0], &np,
                                      &s[1], &t[1], &p0[1], &p1[1]);
        pt.att = ATT_NONE;
        for (size_t i = 0; i < np; ++i) {
            pt.pivotA = to_object(p0[i], posA, ornA);
            pt.pivotB = to_object(p1[i], posB, ornB);
            add_point(r, pt);
        }
    } else if (fA == BF_FACE && fB == BF_VERTEX) {
        pt.pivotB = box_vertex(heB, fiB);
        pt.pivotA = to_world(pt.pivotB, posB, ornB) + sep * distance;
        pt.pivotA = to_object(pt.pivotA, posA, ornA);
        pt.att = ATT_A;
        add_point(r, pt);
    } else if (fB == BF_FACE && fA == BF_VERTEX) {
        pt.pivotA = box_vertex(heA, fiA);
        pt.pivotB = to_world(pt.pivotA, posA, ornA) - sep * distance;
        pt.pivotB = to_object(pt.pivotB, posB, ornB);
        pt.att = ATT_B;
        add_point(r, pt);
    }
}

// ---------------------------------------------------------------- dispatch

static cctx swapped(const cctx &c) { return {c.posB, c.ornB, c.bbB, c.posA, c.ornA, c.bbA, c.threshold}; }  // collide.hpp:21-25
static void swap_result(cresult &r) {            // collision_result.hpp:23-46
    for (size_t i = 0; i < r.num; ++i) {
        cpoint &p = r.pt[i];
        std::swap(p.pivotA, p.pivotB);
        p.normal *= -1;
        if (p.att == ATT_A) p.att = ATT_B; else if (p.att == ATT_B) p.att = ATT_A;
    }
}

typedef void (*collide_fn)(const shape &, const shape &, const cctx &, cresult &);
static collide_fn lookup(uint32_t a, uint32_t b) {
    if (a == SH_SPHERE && b == SH_SPHERE) return sphere_sphere;
    if (a == SH_SPHERE && b == SH_PLANE) return sphere_plane;
    if (a == SH_SPHERE && b == SH_BOX) return sphere_box;
    if (a == SH_BOX && b == SH_PLANE) return box_plane;
    if (a == SH_BOX && b == SH_BOX) return box_box;
    if (a == SH_CAPSULE && b == SH_PLANE) return capsule_plane;
    if (a == SH_CAPSULE && b == SH_CAPSULE) return capsule_capsule;
    if (a == SH_CAPSULE && b == SH_SPHERE) return capsule_sphere;
    if (a == SH_CAPSULE && b == SH_BOX) return capsule_box;
    return nullptr;
}

void collide(const shape &a, const shape &b, const cctx &ctx, cresult &r) {
    if (collide_fn f = lookup(a.kind, b.kind)) { f(a, b, ctx, r); return; }
    if (collide_fn f = lookup(b.kind, a.kind)) {       // swap_collide, collide.hpp:369-374
        f(b, a, swapped(ctx), r);
        swap_result(r);
    }
    // plane-plane: undefined / no points (collide.hpp:70-74)
}

void detect_collision(const shape &a, const shape &b, vec3 posA, quat ornA, const aabb &bbA,
                      vec3 posB, quat ornB, const aabb &bbB, cresult &r) {
    const vec3 offset = vec3{1, 1, 1} * -BREAKING_THRESHOLD;     // collision_util.cpp:444
    r.num = 0;
    if (intersect(inset(bbA, offset), bbB)) {
        cctx ctx{posA, ornA, bbA, posB, ornB, bbB, COLLISION_THRESHOLD};
        collide(a, b, ctx, r);
    }
}

} // namespace ora
