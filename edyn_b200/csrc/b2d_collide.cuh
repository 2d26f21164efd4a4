// Device narrowphase: closest-feature contact generation for sphere / capsule / box / plane pairs and
// the persistent-manifold merge, one manifold per thread.  Replaces edyn::narrowphase's inner loop
// (reference src/edyn/util/collision_util.cpp:440-475 detect_collision -> collision/collide/collide_*.cpp,
// include/edyn/util/collision_util.hpp:105-276 process_collision).  Thresholds and tie-breaking follow
// the reference exactly so the contact sets match; file:line cited per function.
#pragma once
#include "b2d_math.cuh"

namespace b2d {

constexpr int SH_SPHERE = 0, SH_CAPSULE = 2, SH_BOX = 3, SH_PLANE = 6, SH_NONE = 255;
constexpr unsigned ATT_NONE = 0, ATT_A = 1, ATT_B = 2;
constexpr int MAX_CONTACTS = 4;                    // config/constants.hpp:9
constexpr float COLLISION_THRESHOLD = 0.01f;       // :15
constexpr float BREAKING_THRESHOLD = 0.02f;        // :21
constexpr float MERGING_THRESHOLD = 0.01f;         // :27
constexpr float CACHING_THRESHOLD = 0.04f;         // :34
constexpr float FEATURE_TOL = 0.005f;              // :56

struct CPoint { v3 pivotA, pivotB, normal; float distance; unsigned att; };
struct CResult { int num; CPoint pt[4]; };
struct CCtx { v3 posA; q4 ornA; v3 posB; q4 ornB; float threshold; };

enum { INS_NONE = 0, INS_SIMILAR = 1, INS_REPLACE = 2, INS_APPEND = 3 };
enum { BF_VERTEX = 0, BF_EDGE = 1, BF_FACE = 2 };

// shapes/box_shape.hpp:22-44, box_shape.cpp:115-128,163-188
__constant__ signed char c_box_vsign[8][3] = {{1,1,1},{1,-1,1},{1,-1,-1},{1,1,-1},{-1,1,1},{-1,1,-1},{-1,-1,-1},{-1,-1,1}};
__constant__ unsigned char c_box_edge[24] = {0,1, 1,2, 2,3, 3,0, 4,5, 5,6, 6,7, 7,4, 0,4, 1,7, 2,6, 3,5};
__constant__ unsigned char c_box_face[24] = {0,1,2,3, 4,5,6,7, 0,3,5,4, 1,7,6,2, 0,4,7,1, 3,2,6,5};
__constant__ signed char c_face_normal[6][3] = {{1,0,0},{-1,0,0},{0,1,0},{0,-1,0},{0,0,1},{0,0,-1}};
__constant__ signed char c_face_tangent[6][3] = {{0,0,1},{0,0,-1},{1,0,0},{-1,0,0},{0,1,0},{0,-1,0}};

// ---------------------------------------------------------------- src/edyn/math/geom.cpp

B2D_D void plane_space(v3 n, v3 &p, v3 &q) {       // geom.cpp:730-754
    if (fabsf(n.z) > HALF_SQRT2) {
        float a = n.y * n.y + n.z * n.z;
        float k = 1.0f / sqrtf(a);
        p.x = 0; p.y = -n.z * k; p.z = n.y * k;
        q.x = a * k; q.y = -n.x * p.z; q.z = n.x * p.y;
    } else {
        float a = n.x * n.x + n.y * n.y;
        float k = 1.0f / sqrtf(a);
        p.x = -n.y * k; p.y = n.x * k; p.z = 0;
        q.x = -n.z * p.y; q.y = n.z * p.x; q.z = a * k;
    }
}

B2D_D float closest_point_segment(v3 q0, v3 q1, v3 p, float &t, v3 &q) {    // geom.cpp:12-22
    v3 v = q1 - q0, w = p - q0;
    float a = dot(w, v), b = dot(v, v);
    t = clamp_unit(a / b);
    q = q0 + v * t;
    return length_sqr(p - q);
}
B2D_D float closest_point_line(v3 q0, v3 dir, v3 p, float &t, v3 &r) {      // geom.cpp:36-45
    v3 w = p - q0;
    float a = dot(w, dir), b = dot(dir, dir);
    t = a / b;
    r = q0 + dir * t;
    return length_sqr(p - r);
}

// geom.cpp:73-170.  want2: the caller passed num_points / second-solution pointers.
__device__ __noinline__ float closest_point_segment_segment(v3 p1, v3 q1, v3 p2, v3 q2, float &s, float &t, v3 &c1, v3 &c2,
                                                            bool want2, int &num_points, float &sp, float &tp, v3 &c1p, v3 &c2p) {
    const v3 d1 = q1 - p1, d2 = q2 - p2, r = p1 - p2;
    const float a = dot(d1, d1), e = dot(d2, d2), f = dot(d2, r);
    if (a <= EPS && e <= EPS) {
        s = t = 0; c1 = p1; c2 = p2;
        return length_sqr(c1 - c2);
    }
    if (a <= EPS) {
        s = 0; t = f / e; t = clamp_unit(t);
    } else {
        float c = dot(d1, r);
        if (e <= EPS) {
            t = 0; s = clamp_unit(-c / a);
        } else {
            const float b = dot(d1, d2);
            const float denom = a * e - b * b;
            if (denom > EPS) {
                s = clamp_unit((b * f - c * e) / denom);
                if (want2) num_points = 1;
            } else if (want2) {
                v3 r1 = p1 - q2;
                float f1 = dot(d1, r1);
                float a_inv = 1.0f / a;
                s = clamp_unit(fminf(-c * a_inv, -f1 * a_inv));
                sp = clamp_unit(fmaxf(-c * a_inv, -f1 * a_inv));
                v3 r2 = p2 - q1;
                float f2 = dot(d2, r2);
                float e_inv = 1.0f / e;
                t = clamp_unit(fminf(-f * e_inv, -f2 * e_inv));
                tp = clamp_unit(fmaxf(-f * e_inv, -f2 * e_inv));
                if (fabsf(s - sp) > EPS) {
                    num_points = 2;
                    c1p = p1 + d1 * sp;
                    c2p = p2 + d2 * tp;
                } else {
                    num_points = 1;
                }
            } else {
                s = 0;
            }
            const float tnom = b * s + f;
            if (tnom < 0) { t = 0; s = clamp_unit(-c / a); }
            else if (tnom > e) { t = 1; s = clamp_unit((b - c) / a); }
            else { t = tnom / e; }
        }
    }
    c1 = p1 + d1 * s;
    c2 = p2 + d2 * t;
    return length_sqr(c1 - c2);
}

// geom.cpp:1044-1138
__device__ __noinline__ int intersect_line_aabb(v2 p0, v2 p1, v2 bmin, v2 bmax, float &s0, float &s1) {
    int n = 0;
    v2 d = p1 - p0, e = bmin - p0, f = bmax - p0;
    if (fabsf(d.x) < EPS) {
        if (e.x <= 0 && f.x >= 0) { s0 = e.y / d.y; s1 = f.y / d.y; n = 2; }
        return n;
    }
    if (fabsf(d.y) < EPS) {
        if (e.y <= 0 && f.y >= 0) { s0 = e.x / d.x; s1 = f.x / d.x; n = 2; }
        return n;
    }
    { float t = e.x / d.x; float qy = p0.y + d.y * t;
      if (qy >= bmin.y && qy < bmax.y) { s0 = t; ++n; } }
    { float t = f.x / d.x; float qy = p0.y + d.y * t;
      if (qy > bmin.y && qy <= bmax.y) { if (n == 0) { s0 = t; ++n; } else if (fabsf(t - s0) > EPS) { s1 = t; ++n; } } }
    if (n == 2) return n;
    { float t = e.y / d.y; float qx = p0.x + d.x * t;
      if (qx >= bmin.x && qx < bmax.x) { if (n == 0) { s0 = t; ++n; } else if (fabsf(t - s0) > EPS) { s1 = t; ++n; } } }
    if (n == 2) return n;
    { float t = f.y / d.y; float qx = p0.x + d.x * t;
      if (qx > bmin.x && qx <= bmax.x) { if (n == 0) { s0 = t; ++n; } else if (fabsf(t - s0) > EPS) { s1 = t; ++n; } } }
    return n;
}

B2D_D bool point_in_quad_prism(const v3 *v, v3 normal, v3 point) {          // geom.hpp:330-348, N = 4
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
        int j = (i + 1) & 3;
        v3 d = v[j] - v[i];
        v3 t = cross(d, normal);
        if (dot(point - v[i], t) > EPS) return false;
    }
    return true;
}
B2D_D bool point_in_triangle(v3 v0, v3 v1, v3 v2, v3 normal, v3 p) {        // math/triangle.cpp:7-26
    v3 e0 = v1 - v0, e1 = v2 - v1, e2 = v0 - v2;
    v3 q0 = p - v0, q1 = p - v1, q2 = p - v2;
    float d0 = dot(cross(e0, normal), q0), d1 = dot(cross(e1, normal), q1), d2 = dot(cross(e2, normal), q2);
    return (d0 > -EPS && d1 > -EPS && d2 > -EPS) || (d0 < EPS && d1 < EPS && d2 < EPS);
}
B2D_D float manifold_score(v3 p0, v3 p1, v3 p2, v3 p3) {                    // geom.cpp:847-856
    v3 c0 = cross(p0 - p1, p0 - p2), c1 = cross(p0 - p2, p0 - p3), c2 = cross(p0 - p3, p0 - p1), c3 = cross(p1 - p2, p2 - p3);
    return length_sqr(c0) + length_sqr(c1) + length_sqr(c2) + length_sqr(c3);
}

// geom.cpp:857-985.  Returns the insertion type, writes the index; may increment num_points (append).  The points
// come by value (p0..p3; those at and past num_points are not read), so that the manifold merge inlines this with its
// points in registers; the collide functions call it out of line through insertion_point_index below.
B2D_D int insertion_index(v3 p0, v3 p1, v3 p2, v3 p3, int &num_points, v3 np, int &index) {
    const float sim = MERGING_THRESHOLD * MERGING_THRESHOLD;
    if (num_points == 0) { index = num_points++; return INS_APPEND; }
    if (num_points == 1) {
        if (distance_sqr(np, p0) > sim) { index = num_points++; return INS_APPEND; }
        index = 0; return INS_SIMILAR;
    }
    if (num_points == 2) {
        if (length_sqr(cross(np - p0, np - p1)) > EPS) { index = num_points++; return INS_APPEND; }
        float d0 = distance_sqr(np, p0), d1 = distance_sqr(np, p1), cur = distance_sqr(p0, p1);
        if (d0 > cur && d0 > d1) { index = 1; return d1 < sim ? INS_SIMILAR : INS_REPLACE; }
        if (d1 > cur && d1 > d0) { index = 0; return d0 < sim ? INS_SIMILAR : INS_REPLACE; }
        index = 4; return INS_NONE;
    }
    if (num_points == 3) {
        v3 normal = cross(p0 - p1, p1 - p2);
        if (try_normalize(normal)) {
            if (fabsf(dot(np - p0, normal)) < EPS && point_in_triangle(p0, p1, p2, normal, np)) {
                index = 4; return INS_NONE;
            }
            index = num_points++; return INS_APPEND;
        }
        float d0 = dot(p1 - p0, p2 - p0);
        if (d0 > 0 && d0 < 1) { index = 1; return INS_REPLACE; }
        float d1 = dot(p0 - p1, p2 - p1);
        if (d1 > 0 && d1 < 1) { index = 0; return INS_REPLACE; }
        float d2 = dot(p2 - p0, p1 - p0);
        if (d2 > 0 && d2 < 1) { index = 2; return INS_REPLACE; }
        float ds0 = distance_sqr(p0, p1), ds1 = distance_sqr(p1, p2), ds2 = distance_sqr(p2, p0);
        int mi = -1; float md = SCALAR_MAX;
        if (ds0 < md) { md = ds0; mi = 0; }
        if (ds1 < md) { md = ds1; mi = 1; }
        if (ds2 < md) { md = ds2; mi = 2; }
        index = mi; return INS_REPLACE;       // mi == -1 only for NaN input, as SIZE_MAX in the reference
    }
    float sc0 = manifold_score(np, p1, p2, p3);
    float sc1 = manifold_score(np, p0, p2, p3);
    float sc2 = manifold_score(np, p0, p1, p3);
    float sc3 = manifold_score(np, p0, p1, p2);
    float max_score = manifold_score(p0, p1, p2, p3);
    int mi = -1;
    if (sc0 > max_score) { max_score = sc0; mi = 0; }
    if (sc1 > max_score) { max_score = sc1; mi = 1; }
    if (sc2 > max_score) { max_score = sc2; mi = 2; }
    if (sc3 > max_score) { max_score = sc3; mi = 3; }
    if (mi >= 0) {
        const v3 pm = mi == 0 ? p0 : mi == 1 ? p1 : mi == 2 ? p2 : p3;
        index = mi; return distance_sqr(pm, np) < sim ? INS_SIMILAR : INS_REPLACE;
    }
    index = 4; return INS_NONE;
}
__device__ __noinline__ int insertion_point_index(const v3 *points, int &num_points, v3 np, int &index) {
    const int n = num_points;
    return insertion_index(n > 0 ? points[0] : np, n > 1 ? points[1] : np, n > 2 ? points[2] : np, n > 3 ? points[3] : np,
                           num_points, np, index);
}

B2D_D void add_point(CResult &r, const CPoint &p) { r.pt[r.num++] = p; }     // collision_result.cpp:6-10
__device__ __noinline__ void maybe_add_point(CResult &r, const CPoint &np) {   // collision_result.cpp:12-33
    v3 piv[4];
    for (int i = 0; i < r.num; ++i) piv[i] = r.pt[i].pivotA;
    int idx;
    int type = insertion_point_index(piv, r.num, np.pivotA, idx);
    if (type == INS_NONE) {
        for (int i = 0; i < r.num; ++i) piv[i] = r.pt[i].pivotB;
        type = insertion_point_index(piv, r.num, np.pivotB, idx);
    }
    if (type != INS_NONE && idx >= 0 && idx < 4) r.pt[idx] = np;
}

B2D_D v3 closest_point_box_outside(v3 he, v3 p) {       // geom.cpp:987-996
    v3 c = p;
    c.x = fminf(he.x, c.x); c.x = fmaxf(-he.x, c.x);
    c.y = fminf(he.y, c.y); c.y = fmaxf(-he.y, c.y);
    c.z = fminf(he.z, c.z); c.z = fmaxf(-he.z, c.z);
    return c;
}
// geom.cpp:998-1042 -- returns the LAST `dist` computed (not the minimum), exactly as the reference does.
B2D_D float closest_point_box_inside(v3 he, v3 p, v3 &closest, v3 &normal) {
    float dist = he.x - p.x;
    float min_dist = dist;
    closest = mk3(he.x, p.y, p.z); normal = mk3(1, 0, 0);
    dist = he.x + p.x;
    if (dist < min_dist) { min_dist = dist; closest = mk3(-he.x, p.y, p.z); normal = mk3(-1, 0, 0); }
    dist = he.y - p.y;
    if (dist < min_dist) { min_dist = dist; closest = mk3(p.x, he.y, p.z); normal = mk3(0, 1, 0); }
    dist = he.y + p.y;
    if (dist < min_dist) { min_dist = dist; closest = mk3(p.x, -he.y, p.z); normal = mk3(0, -1, 0); }
    dist = he.z - p.z;
    if (dist < min_dist) { min_dist = dist; closest = mk3(p.x, p.y, he.z); normal = mk3(0, 0, 1); }
    dist = he.z + p.z;
    if (dist < min_dist) { min_dist = dist; closest = mk3(p.x, p.y, -he.z); normal = mk3(0, 0, -1); }
    return dist;
}

// ---------------------------------------------------------------- src/edyn/shapes/box_shape.cpp

B2D_D v3 box_vertex(v3 he, int i) { return mk3(he.x * (float)c_box_vsign[i][0], he.y * (float)c_box_vsign[i][1], he.z * (float)c_box_vsign[i][2]); }
B2D_D v3 box_support_point(v3 he, v3 d) { return mk3(d.x > 0 ? he.x : -he.x, d.y > 0 ? he.y : -he.y, d.z > 0 ? he.z : -he.z); }   // util/shape_util.cpp:40-46
B2D_D float box_support_projection(v3 he, v3 pos, q4 orn, v3 dir) {          // box_shape.cpp:24-28
    v3 ld = rotate(conjugate(orn), dir);
    v3 pt = box_support_point(he, ld);
    return dot(pos, dir) + dot(pt, ld);
}
B2D_D int box_edge_index(int v0, int v1) {                                    // box_shape.cpp:228-242
    for (int i = 0; i < 12; ++i) {
        int a = c_box_edge[i * 2], b = c_box_edge[i * 2 + 1];
        if ((a == v0 && b == v1) || (b == v0 && a == v1)) return i;
    }
    return 0;   // unreachable for vertices of one face (the reference asserts)
}
B2D_D v3 face_normal(int f) { return mk3(c_face_normal[f][0], c_face_normal[f][1], c_face_normal[f][2]); }
B2D_D v3 face_tangent(int f) { return mk3(c_face_tangent[f][0], c_face_tangent[f][1], c_face_tangent[f][2]); }

// box_shape.cpp:30-96
__device__ __noinline__ void box_support_feature(v3 he, v3 dir, int &feature, int &feature_index, float &projection, float threshold) {
    int m = max_index_abs(dir);
    int face = get(dir, m) < 0 ? m * 2 + 1 : m * 2;                           // support_face_index, :244-252
    float proj[4]; int vidx[4]; int idx[4];
    projection = -SCALAR_MAX;
    int count = 1, max_i = 0;
    idx[0] = 0;
    for (int i = 0; i < 4; ++i) {
        int vi = c_box_face[face * 4 + i];
        vidx[i] = vi;
        float p = dot(box_vertex(he, vi), dir);
        proj[i] = p;
        if (p > projection) { projection = p; idx[0] = i; max_i = i; }
    }
    for (int i = 0; i < 4; ++i) if (i != max_i && proj[i] > projection - threshold) idx[count++] = i;
    if (count == 1) { feature = BF_VERTEX; feature_index = vidx[idx[0]]; }
    else if (count == 2) { feature = BF_EDGE; feature_index = box_edge_index(vidx[idx[0]], vidx[idx[1]]); }
    else if (count == 3) {
        feature = BF_EDGE;
        float p0 = proj[idx[0]], p1 = proj[idx[1]], p2 = proj[idx[2]];
        if (p0 <= p1 && p0 <= p2) feature_index = box_edge_index(vidx[idx[1]], vidx[idx[2]]);
        else if (p1 <= p0 && p1 <= p2) feature_index = box_edge_index(vidx[idx[0]], vidx[idx[2]]);
        else feature_index = box_edge_index(vidx[idx[0]], vidx[idx[1]]);
    } else { feature = BF_FACE; feature_index = face; }
}
B2D_D void box_support_feature_w(v3 he, v3 pos, q4 orn, v3 axis_pos, v3 axis_dir, int &f, int &idx, float &proj, float tol) {   // :98-105
    v3 ld = rotate(conjugate(orn), axis_dir);
    box_support_feature(he, ld, f, idx, proj, tol);
    proj += dot(pos - axis_pos, axis_dir);
}
B2D_D void box_face_world(v3 he, int f, v3 pos, q4 orn, v3 *out) {            // :143-161
    #pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = to_world(box_vertex(he, c_box_face[f * 4 + i]), pos, orn);
}
B2D_D void box_edge_world(v3 he, int e, v3 pos, q4 orn, v3 *out) {            // :130-141
    out[0] = to_world(box_vertex(he, c_box_edge[e * 2]), pos, orn);
    out[1] = to_world(box_vertex(he, c_box_edge[e * 2 + 1]), pos, orn);
}
B2D_D v3 box_face_center(v3 he, int f, v3 pos, q4 orn) { v3 n = rotate(orn, face_normal(f)); return pos + n * get(he, f / 2); }   // :194-198
B2D_D m3 box_face_basis(int f, q4 orn) {                                       // :200-205
    v3 y = face_normal(f), x = face_tangent(f), z = cross(x, y);
    return m3_columns(rotate(orn, x), rotate(orn, y), rotate(orn, z));
}
B2D_D v2 box_face_half_extents(v3 he, int f) {                                 // :207-217
    v2 r;
    if (f == 0 || f == 1) { r.x = he.z; r.y = he.y; }
    else if (f == 2 || f == 3) { r.x = he.x; r.y = he.z; }
    else { r.x = he.y; r.y = he.x; }
    return r;
}

// ---------------------------------------------------------------- src/edyn/util/aabb_util.cpp

B2D_D v3 axis_vec(int a) { return mk3(a == 0 ? 1.0f : 0.0f, a == 1 ? 1.0f : 0.0f, a == 2 ? 1.0f : 0.0f); }

B2D_D box3 shape_aabb(int kind, float4 sp, v3 pos, q4 orn) {
    box3 bb;
    if (kind == SH_SPHERE) {                           // aabb_util.cpp:65-70
        float r = sp.x;
        bb.mn = mk3(pos.x - r, pos.y - r, pos.z - r); bb.mx = mk3(pos.x + r, pos.y + r, pos.z + r);
    } else if (kind == SH_CAPSULE) {                   // aabb_util.cpp:81-88
        v3 dir = rotate(orn, axis_vec((int)sp.z));
        v3 v = dir * sp.y;
        v3 p0 = pos - v, p1 = pos + v;
        v3 off = mk3(sp.x, sp.x, sp.x);
        bb.mn = vmin(p0, p1) - off; bb.mx = vmax(p0, p1) + off;
    } else if (kind == SH_BOX) {                       // aabb_util.cpp:42-63
        bb.mn = pos; bb.mx = pos;
        m3 basis = to_m3(orn);
        v3 he = mk3(sp);
        #pragma unroll
        for (int i = 0; i < 3; ++i) {
            v3 row = i == 0 ? basis.r0 : (i == 1 ? basis.r1 : basis.r2);
            float mn = get(bb.mn, i), mx = get(bb.mx, i);
            #pragma unroll
            for (int j = 0; j < 3; ++j) {
                float e = get(row, j) * -get(he, j);
                float f = -e;
                if (e < f) { mn += e; mx += f; } else { mn += f; mx += e; }
            }
            set(bb.mn, i, mn); set(bb.mx, i, mx);
        }
    } else if (kind == SH_PLANE) {                     // aabb_util.cpp:9-40
        const float H = 99999.0f;
        v3 n = mk3(sp);
        v3 umin = mk3(-1, -1, -1), umax = mk3(1, 1, 1);
        if (n.x == 1 && n.y == 0 && n.z == 0) umax.x = 0;
        else if (n.x == -1 && n.y == 0 && n.z == 0) umin.x = 0;
        else if (n.x == 0 && n.y == 1 && n.z == 0) umax.y = 0;
        else if (n.x == 0 && n.y == -1 && n.z == 0) umin.y = 0;
        else if (n.x == 0 && n.y == 0 && n.z == 1) umax.z = 0;
        else if (n.x == 0 && n.y == 0 && n.z == -1) umin.z = 0;
        v3 pw = n * sp.w;
        bb.mn = umin * H + pw; bb.mx = umax * H + pw;
    } else {
        bb.mn = pos; bb.mx = pos;
    }
    return bb;
}

// ---------------------------------------------------------------- collision/collide/*.cpp

B2D_D void capsule_vertices(float4 c, v3 pos, q4 orn, v3 *out) {              // shapes/capsule_shape.hpp:21-27
    v3 dir = rotate(orn, axis_vec((int)c.z));
    out[0] = pos + dir * c.y;
    out[1] = pos - dir * c.y;
}
B2D_D float capsule_support_projection(const v3 *v, float radius, v3 dir) { return fmaxf(dot(v[0], dir), dot(v[1], dir)) + radius; }   // util/shape_util.cpp:297-300

B2D_D CPoint mkpt(v3 a, v3 b, v3 n, float d, unsigned att) { CPoint p; p.pivotA = a; p.pivotB = b; p.normal = n; p.distance = d; p.att = att; return p; }

// collide_sphere_sphere.cpp:5-27
B2D_D void collide_sphere_sphere(float4 A, float4 B, const CCtx &c, CResult &r) {
    v3 d = c.posA - c.posB;
    float dist_sqr = length_sqr(d);
    float rr = A.x + B.x + c.threshold;
    if (dist_sqr > rr * rr) return;
    float dist = sqrtf(dist_sqr);
    v3 dn = dist > EPS ? d / dist : mk3(1, 0, 0);
    v3 rA = -dn * A.x; rA = rotate(conjugate(c.ornA), rA);
    v3 rB = dn * B.x; rB = rotate(conjugate(c.ornB), rB);
    add_point(r, mkpt(rA, rB, dn, dist - A.x - B.x, ATT_NONE));
}
// collide_sphere_plane.cpp:5-20 (no collision_threshold on this pair, as in the reference)
B2D_D void collide_sphere_plane(float4 S, float4 P, const CCtx &c, CResult &r) {
    v3 normal = mk3(P);
    v3 center = normal * P.w;
    v3 d = c.posA - center;
    float l = dot(normal, d);
    if (l > S.x) return;
    v3 pivotA = rotate(conjugate(c.ornA), -normal * S.x);
    v3 pivotB = rotate(conjugate(c.ornB), d - normal * l - center);
    add_point(r, mkpt(pivotA, pivotB, normal, l - S.x, ATT_B));
}
// collide_box_plane.cpp:7-56
B2D_D void collide_box_plane(float4 Bx, float4 P, const CCtx &c, CResult &r) {
    v3 he = mk3(Bx), n = mk3(P);
    v3 center = n * P.w;
    int fA, fiA; float projA;
    box_support_feature_w(he, c.posA, c.ornA, center, -n, fA, fiA, projA, FEATURE_TOL);
    float distance = -projA;
    if (distance > c.threshold) return;
    int nv = fA == BF_VERTEX ? 1 : (fA == BF_EDGE ? 2 : 4);
    for (int i = 0; i < nv; ++i) {
        int vi = fA == BF_VERTEX ? fiA : (fA == BF_EDGE ? c_box_edge[fiA * 2 + i] : c_box_face[fiA * 4 + i]);
        v3 pivotA = box_vertex(he, vi);
        v3 pAw = to_world(pivotA, c.posA, c.ornA);
        v3 pBw = project_plane(pAw, center, n);
        add_point(r, mkpt(pivotA, to_object(pBw, c.posB, c.ornB), n, dot(pAw - pBw, n), ATT_B));
    }
}
// collide_capsule_plane.cpp:6-38 (pivotB left in world space, as written there at :35-36)
B2D_D void collide_capsule_plane(float4 C, float4 P, const CCtx &c, CResult &r) {
    v3 n = mk3(P);
    v3 center = n * P.w;
    v3 cv[2]; capsule_vertices(C, c.posA, c.ornA, cv);
    float proj[2] = {dot(cv[0] - center, n), dot(cv[1] - center, n)};
    #pragma unroll
    for (int i = 0; i < 2; ++i) {
        float distance = proj[i] - C.x;
        if (distance > c.threshold) continue;
        v3 vertex = cv[i];
        v3 pAw = vertex - n * C.x;
        add_point(r, mkpt(to_object(pAw, c.posA, c.ornA), project_plane(vertex, center, n), n, distance, ATT_B));
    }
}
// collide_sphere_box.cpp:7-55
B2D_D void collide_sphere_box(float4 S, float4 Bx, const CCtx &c, CResult &r) {
    v3 he = mk3(Bx);
    const q4 ornB_conj = conjugate(c.ornB);
    const v3 posA_in_B = rotate(ornB_conj, c.posA - c.posB);
    const q4 ornA_in_B = ornB_conj * c.ornA;
    v3 closest = closest_point_box_outside(he, posA_in_B);
    v3 normalB = posA_in_B - closest;
    float d_sqr = length_sqr(normalB);
    float min_dist = S.x + c.threshold;
    if (d_sqr > min_dist * min_dist) return;
    float center_distance;
    unsigned att = ATT_NONE;
    if (d_sqr <= EPS) {
        center_distance = -closest_point_box_inside(he, posA_in_B, closest, normalB);
        att = ATT_B;
    } else {
        center_distance = sqrtf(d_sqr);
        normalB /= center_distance;
        if (fabsf(normalB.x) > 1.0f - EPS || fabsf(normalB.y) > 1.0f - EPS || fabsf(normalB.z) > 1.0f - EPS) att = ATT_B;
    }
    v3 pivotA_in_B = posA_in_B - normalB * S.x;
    v3 pivotA = to_object(pivotA_in_B, posA_in_B, ornA_in_B);
    add_point(r, mkpt(pivotA, closest, rotate(c.ornB, normalB), center_distance - S.x, att));
}
// collide_capsule_capsule.cpp:7-81
B2D_D void collide_capsule_capsule(float4 A, float4 B, const CCtx &c, CResult &r) {
    v3 vA[2], vB[2];
    capsule_vertices(A, c.posA, c.ornA, vA);
    capsule_vertices(B, c.posB, c.ornB, vB);
    float s0, t0, s1 = 0, t1 = 0; v3 cA[2], cB[2]; int np = 0;
    float dist_sqr = closest_point_segment_segment(vA[0], vA[1], vB[0], vB[1], s0, t0, cA[0], cB[0], true, np, s1, t1, cA[1], cB[1]);
    float min_dist = A.x + B.x + c.threshold;
    if (dist_sqr > min_dist * min_dist) return;
    v3 normal; float distance;
    if (dist_sqr > EPS) {
        float dist = sqrtf(dist_sqr);
        normal = (cA[0] - cB[0]) / dist;
        distance = dist - A.x - B.x;
    } else {
        v3 axA = vA[1] - vA[0], axB = vB[1] - vB[0];
        normal = cross(axA, axB);
        if (dot(c.posA - c.posB, normal) < 0) normal *= -1.0f;
        if (!try_normalize(normal)) normal = mk3(0, 1, 0);
        distance = -(A.x + B.x);
    }
    for (int i = 0; i < np; ++i) {
        v3 pAw = cA[i] - normal * A.x;
        v3 pBw = cB[i] + normal * B.x;
        add_point(r, mkpt(to_object(pAw, c.posA, c.ornA), to_object(pBw, c.posB, c.ornB), normal, distance, ATT_NONE));
    }
}
// collide_capsule_sphere.cpp:10-52
B2D_D void collide_capsule_sphere(float4 C, float4 S, const CCtx &c, CResult &r) {
    v3 cv[2]; capsule_vertices(C, c.posA, c.ornA, cv);
    v3 closest; float t;
    float dist_sqr = closest_point_segment(cv[0], cv[1], c.posB, t, closest);
    float min_dist = C.x + S.x + c.threshold;
    if (dist_sqr > min_dist * min_dist) return;
    v3 normal = closest - c.posB;
    float nls = length_sqr(normal);
    float distance;
    if (nls > EPS) {
        float nl = sqrtf(nls);
        normal /= nl;
        distance = nl - C.x - S.x;
    } else {
        normal = quat_z(c.ornA);
        distance = -(C.x + S.x);
    }
    v3 normalB = rotate(conjugate(c.ornB), normal);
    v3 pAw = closest - normal * C.x;
    add_point(r, mkpt(to_object(pAw, c.posA, c.ornA), normalB * S.x, normal, distance, ATT_NONE));
}

// collide_capsule_box.cpp:14-213
__device__ __noinline__ void collide_capsule_box(float4 C, float4 Bx, const CCtx &c, CResult &r) {
    v3 he = mk3(Bx);
    const v3 posA = mk3(0, 0, 0);
    const q4 ornA = c.ornA;
    const v3 posB = c.posB - c.posA;
    const q4 ornB = c.ornB;
    v3 cv[2]; capsule_vertices(C, posA, ornA, cv);
    float distance = -SCALAR_MAX, projection_box = -SCALAR_MAX;
    v3 sep = mk3(0, 0, 0);
    for (int i = 0; i < 3; ++i) {
        v3 dir = rotate(ornB, axis_vec(i));
        if (dot(posA - posB, dir) < 0) dir = -dir;
        float projA = -capsule_support_projection(cv, C.x, -dir);
        float projB = dot(posB, dir) + get(he, i);
        float dist = projA - projB;
        if (dist > distance) { distance = dist; projection_box = projB; sep = dir; }
    }
    for (int i = 0; i < 12; ++i) {
        v3 ev[2]; box_edge_world(he, i, posB, ornB, ev);
        float s, t, sp, tp; v3 cA, cB, d0, d1; int np;
        closest_point_segment_segment(ev[0], ev[1], cv[0], cv[1], s, t, cA, cB, false, np, sp, tp, d0, d1);
        v3 dir = cA - cB;
        if (!try_normalize(dir)) continue;
        if (dot(posA - posB, dir) < 0) dir *= -1.0f;
        float projA = -capsule_support_projection(cv, C.x, -dir);
        float projB = box_support_projection(he, posB, ornB, dir);
        float dist = projA - projB;
        if (dist > distance) { distance = dist; projection_box = projB; sep = dir; }
    }
    if (distance > c.threshold) return;
    float pcv[2] = {dot(cv[0], sep), dot(cv[1], sep)};
    bool is_edge = fabsf(pcv[0] - pcv[1]) < FEATURE_TOL;
    v3 origin_box = sep * projection_box;
    float fdistB; int fB, fiB;
    box_support_feature_w(he, posB, ornB, origin_box, sep, fB, fiB, fdistB, FEATURE_TOL);
    CPoint pt; pt.normal = sep; pt.distance = distance; pt.att = ATT_NONE;
    if (fB == BF_FACE) {
        v3 fv[4]; box_face_world(he, fiB, posB, ornB, fv);
        pt.att = ATT_B;
        if (is_edge) {
            for (int k = 0; k < 2; ++k) {
                v3 pA = cv[k];
                if (point_in_quad_prism(fv, sep, pA)) {
                    pt.pivotA = to_object(pA - sep * C.x, posA, ornA);
                    v3 pBw = project_plane(pA, origin_box, sep);
                    pt.pivotB = to_object(pBw, posB, ornB);
                    add_point(r, pt);
                }
            }
            if (r.num == 2) return;
            v3 fc = box_face_center(he, fiB, posB, ornB);
            m3 fb = box_face_basis(fiB, ornB);
            v2 hx = box_face_half_extents(he, fiB);
            v3 o0 = to_object(cv[0], fc, fb), o1 = to_object(cv[1], fc, fb);
            v2 p0, p1; p0.x = o0.x; p0.y = o0.z; p1.x = o1.x; p1.y = o1.z;
            float s[2];
            int np = intersect_line_aabb(p0, p1, neg(hx), hx, s[0], s[1]);
            for (int i = 0; i < np; ++i) {
                if (s[i] < 0 || s[i] > 1) continue;
                v3 ep = lerp(cv[0], cv[1], s[i]);
                v3 fp = project_plane(ep, fc, sep);
                pt.pivotA = to_object(ep - sep * C.x, posA, ornA);
                pt.pivotB = to_object(fp, posB, ornB);
                add_point(r, pt);
            }
        } else {
            v3 ccv = pcv[0] < pcv[1] ? cv[0] : cv[1];
            v3 pAw = ccv - sep * C.x;
            v3 pBw = project_plane(pAw, origin_box, sep);
            pt.pivotA = to_object(pAw, posA, ornA);
            pt.pivotB = to_object(pBw, posB, ornB);
            add_point(r, pt);
        }
    } else if (fB == BF_EDGE) {
        v3 ev[2]; box_edge_world(he, fiB, posB, ornB, ev);
        pt.att = ATT_NONE;
        if (is_edge) {
            float s0, t0, s1 = 0, t1 = 0; v3 cA[2], cB[2]; int np = 0;
            closest_point_segment_segment(cv[0], cv[1], ev[0], ev[1], s0, t0, cA[0], cB[0], true, np, s1, t1, cA[1], cB[1]);
            for (int i = 0; i < np; ++i) {
                pt.pivotA = to_object(cA[i] - sep * C.x, posA, ornA);
                pt.pivotB = to_object(cB[i], posB, ornB);
                add_point(r, pt);
            }
        } else {
            v3 ccv = pcv[0] < pcv[1] ? cv[0] : cv[1];
            v3 edir = ev[1] - ev[0];
            v3 pBw; float t;
            closest_point_line(ev[0], edir, ccv, t, pBw);
            pt.pivotB = to_object(pBw, posB, ornB);
            pt.pivotA = to_object(ccv - sep * C.x, posA, ornA);
            add_point(r, pt);
        }
    } else {
        pt.pivotB = box_vertex(he, fiB);
        v3 pBw = to_world(pt.pivotB, posB, ornB);
        v3 pAw = pBw + sep * distance;
        pt.pivotA = to_object(pAw, posA, ornA);
        pt.att = ATT_NONE;
        add_point(r, pt);
    }
}

// collide_box_box.cpp:14-266 -- 15-axis SAT, support-feature classification, face/edge clipping.
__device__ __noinline__ void collide_box_box(float4 A, float4 B, const CCtx &c, CResult &r) {
    v3 heA = mk3(A), heB = mk3(B);
    const v3 posA = c.posA, posB = c.posB;
    const q4 ornA = c.ornA, ornB = c.ornB;
    v3 axA[3] = {quat_x(ornA), quat_y(ornA), quat_z(ornA)};
    v3 axB[3] = {quat_x(ornB), quat_y(ornB), quat_z(ornB)};
    float distance = -SCALAR_MAX;
    v3 sep = mk3(0, 0, 0);
    for (int i = 0; i < 3; ++i) {
        v3 dir = axA[i];
        if (dot(posA - posB, dir) < 0) dir = -dir;
        float projA = dot(posA, dir) - get(heA, i);
        float projB = box_support_projection(heB, posB, ornB, dir);
        float dist = projA - projB;
        if (dist > distance) { distance = dist; sep = dir; }
    }
    for (int i = 0; i < 3; ++i) {
        v3 dir = axB[i];
        if (dot(posA - posB, dir) < 0) dir = -dir;
        float projA = -box_support_projection(heA, posA, ornA, -dir);
        float projB = dot(posB, dir) + get(heB, i);
        float dist = projA - projB;
        if (dist > distance) { distance = dist; sep = dir; }
    }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
        v3 dir = cross(axA[i], axB[j]);
        float dls = length_sqr(dir);
        if (!(dls > EPS)) continue;
        dir /= sqrtf(dls);
        if (dot(posA - posB, dir) < 0) dir *= -1.0f;
        float projA = -box_support_projection(heA, posA, ornA, -dir);
        float projB = box_support_projection(heB, posB, ornB, dir);
        float dist = projA - projB;
        if (dist > distance) { distance = dist; sep = dir; }
    }
    if (distance > c.threshold) return;

    int fA, fB, fiA, fiB; float prA, prB;
    box_support_feature_w(heA, posA, ornA, mk3(0, 0, 0), -sep, fA, fiA, prA, FEATURE_TOL);
    box_support_feature_w(heB, posB, ornB, mk3(0, 0, 0), sep, fB, fiB, prB, FEATURE_TOL);

    CPoint pt; pt.normal = sep; pt.distance = distance; pt.att = ATT_NONE;
    pt.pivotA = pt.pivotB = mk3(0, 0, 0);

    if (fA == BF_FACE && fB == BF_FACE) {
        v3 fvA[4], fvB[4];
        box_face_world(heA, fiA, posA, ornA, fvA);
        v3 fnA = rotate(ornA, face_normal(fiA));
        box_face_world(heB, fiB, posB, ornB, fvB);
        v3 fnB = rotate(ornB, face_normal(fiB));
        pt.att = ATT_B;
        for (int i = 0; i < 4; ++i) {
            if (point_in_quad_prism(fvA, fnA, fvB[i])) {
                v3 pf = project_plane(fvB[i], fvA[0], fnA);
                pt.pivotA = to_object(pf, posA, ornA);
                pt.pivotB = to_object(fvB[i], posB, ornB);
                maybe_add_point(r, pt);
            }
        }
        for (int i = 0; i < 4; ++i) {
            if (point_in_quad_prism(fvB, fnB, fvA[i])) {
                v3 pf = project_plane(fvA[i], fvB[0], fnB);
                pt.pivotA = to_object(fvA[i], posA, ornA);
                pt.pivotB = to_object(pf, posB, ornB);
                maybe_add_point(r, pt);
            }
        }
        if (r.num < 4) {
            v3 fc = box_face_center(heA, fiA, posA, ornA);
            m3 fb = box_face_basis(fiA, ornA);
            v2 hx = box_face_half_extents(heA, fiA);
            for (int j = 0; j < 4; ++j) {
                v3 b0w = fvB[j], b1w = fvB[(j + 1) & 3];
                v3 b0 = to_object(b0w, fc, fb), b1 = to_object(b1w, fc, fb);
                v2 p0, p1; p0.x = b0.x; p0.y = b0.z; p1.x = b1.x; p1.y = b1.z;
                float s[2];
                int np = intersect_line_aabb(p0, p1, neg(hx), hx, s[0], s[1]);
                for (int k = 0; k < np; ++k) {
                    if (s[k] < 0 || s[k] > 1) continue;
                    v3 q1 = lerp(b0w, b1w, s[k]);
                    v3 q0 = project_plane(q1, fc, fnA);
                    pt.pivotA = to_object(q0, posA, ornA);
                    pt.pivotB = to_object(q1, posB, ornB);
                    maybe_add_point(r, pt);
                }
            }
        }
    } else if ((fA == BF_FACE && fB == BF_EDGE) || (fB == BF_FACE && fA == BF_EDGE)) {
        const bool faceA = fA == BF_FACE;
        v3 fn = faceA ? rotate(ornA, face_normal(fiA)) : rotate(ornB, face_normal(fiB));
        v3 fv[4], ev[2];
        if (faceA) { box_face_world(heA, fiA, posA, ornA, fv); box_edge_world(heB, fiB, posB, ornB, ev); }
        else { box_face_world(heB, fiB, posB, ornB, fv); box_edge_world(heA, fiA, posA, ornA, ev); }
        pt.att = faceA ? ATT_A : ATT_B;
        for (int i = 0; i < 2; ++i) {
            if (point_in_quad_prism(fv, fn, ev[i])) {
                v3 pf = project_plane(ev[i], fv[0], fn);
                pt.pivotA = faceA ? to_object(pf, posA, ornA) : to_object(ev[i], posA, ornA);
                pt.pivotB = faceA ? to_object(ev[i], posB, ornB) : to_object(pf, posB, ornB);
                add_point(r, pt);
            }
        }
        if (r.num < 2) {
            v3 fc = faceA ? box_face_center(heA, fiA, posA, ornA) : box_face_center(heB, fiB, posB, ornB);
            m3 fb = faceA ? box_face_basis(fiA, ornA) : box_face_basis(fiB, ornB);
            v2 hx = faceA ? box_face_half_extents(heA, fiA) : box_face_half_extents(heB, fiB);
            v3 e0 = to_object(ev[0], fc, fb), e1 = to_object(ev[1], fc, fb);
            v2 p0, p1; p0.x = e0.x; p0.y = e0.z; p1.x = e1.x; p1.y = e1.z;
            float s[2];
            int np = intersect_line_aabb(p0, p1, neg(hx), hx, s[0], s[1]);
            for (int i = 0; i < np; ++i) {
                if (s[i] < 0 || s[i] > 1) continue;
                v3 ep = lerp(ev[0], ev[1], s[i]);
                v3 fp = project_plane(ep, fc, sep);
                pt.pivotA = to_object(faceA ? fp : ep, posA, ornA);
                pt.pivotB = to_object(faceA ? ep : fp, posB, ornB);
                add_point(r, pt);
            }
        }
    } else if (fA == BF_EDGE && fB == BF_EDGE) {
        float s0, t0, s1 = 0, t1 = 0; v3 p0[2], p1[2]; int np = 0;
        v3 eA[2], eB[2];
        box_edge_world(heA, fiA, posA, ornA, eA);
        box_edge_world(heB, fiB, posB, ornB, eB);
        closest_point_segment_segment(eA[0], eA[1], eB[0], eB[1], s0, t0, p0[0], p1[0], true, np, s1, t1, p0[1], p1[1]);
        pt.att = ATT_NONE;
        for (int i = 0; i < np; ++i) {
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

// ---------------------------------------------------------------- dispatch (collision_util.cpp:440-475, collide.hpp:369-374)

B2D_D void swap_result(CResult &r) {                    // collision_result.hpp:23-46
    for (int i = 0; i < r.num; ++i) {
        CPoint &p = r.pt[i];
        v3 t = p.pivotA; p.pivotA = p.pivotB; p.pivotB = t;
        p.normal *= -1.0f;
        if (p.att == ATT_A) p.att = ATT_B; else if (p.att == ATT_B) p.att = ATT_A;
    }
}

// Ordered pair kernel id; 0 means "no collide() overload in scope".
B2D_D int pair_fn(int a, int b) {
    if (a == SH_SPHERE && b == SH_SPHERE) return 1;
    if (a == SH_SPHERE && b == SH_PLANE) return 2;
    if (a == SH_SPHERE && b == SH_BOX) return 3;
    if (a == SH_BOX && b == SH_PLANE) return 4;
    if (a == SH_BOX && b == SH_BOX) return 5;
    if (a == SH_CAPSULE && b == SH_PLANE) return 6;
    if (a == SH_CAPSULE && b == SH_CAPSULE) return 7;
    if (a == SH_CAPSULE && b == SH_SPHERE) return 8;
    if (a == SH_CAPSULE && b == SH_BOX) return 9;
    return 0;
}
// the seven light overloads; box-box (5) and capsule-box (9) are not called from here
B2D_D void run_light_pair(int fn, float4 A, float4 B, const CCtx &c, CResult &r) {
    switch (fn) {
    case 1: collide_sphere_sphere(A, B, c, r); break;
    case 2: collide_sphere_plane(A, B, c, r); break;
    case 3: collide_sphere_box(A, B, c, r); break;
    case 4: collide_box_plane(A, B, c, r); break;
    case 6: collide_capsule_plane(A, B, c, r); break;
    case 7: collide_capsule_capsule(A, B, c, r); break;
    case 8: collide_capsule_sphere(A, B, c, r); break;
    default: break;
    }
}
B2D_D void run_pair(int fn, float4 A, float4 B, const CCtx &c, CResult &r) {
    switch (fn) {
    case 5: collide_box_box(A, B, c, r); break;
    case 9: collide_capsule_box(A, B, c, r); break;
    default: run_light_pair(fn, A, B, c, r); break;
    }
}
B2D_D void collide(int kindA, float4 A, int kindB, float4 B, const CCtx &c, CResult &r) {
    int fn = pair_fn(kindA, kindB);
    if (fn) { run_pair(fn, A, B, c, r); return; }
    fn = pair_fn(kindB, kindA);
    if (fn) {                                           // swap_collide
        CCtx s; s.posA = c.posB; s.ornA = c.ornB; s.posB = c.posA; s.ornB = c.ornA; s.threshold = c.threshold;
        run_pair(fn, B, A, s, r);
        swap_result(r);
    }
}

// ---------------------------------------------------------------- src/edyn/collision/raycast.cpp
// shape_raycast for the four shapes.  fraction / normal / feature are the reference's bits (no clamping to [0, 1]: the
// world query filters), except the capsule hemisphere normal, which is taken at the hit point from the hemisphere centre.

constexpr uint32_t RAY_FEATURE_NONE = 0xFFFFFFFFu;      // B2D_RAY_FEATURE_NONE
constexpr uint32_t RAY_CAPSULE_SIDE = 2u;               // B2D_RAY_CAPSULE_SIDE
struct RayHit { bool hit; float fraction; v3 normal; uint32_t feature; };

B2D_D bool intersect_ray_sphere(v3 p0, v3 p1, v3 pos, float radius, float &t) {   // geom.cpp:1276-1305
    v3 d = p1 - p0, m = p0 - pos;
    float a = dot(d, d), b = dot(m, d), c = dot(m, m) - radius * radius;
    if (c > 0 && b > 0) return false;
    float discr = b * b - a * c;
    if (discr < 0) return false;
    t = (-b - sqrtf(discr)) / a;
    t = 0.0f < t ? t : 0.0f;                                // std::max(scalar(0), t): NaN gives 0
    return true;
}
B2D_D bool closest_point_line_line(v3 p1, v3 q1, v3 p2, v3 q2, float &s, float &t) {   // geom.cpp:46-70
    v3 d1 = q1 - p1, d2 = q2 - p2, r = p1 - p2;
    float a = dot(d1, d1), b = dot(d1, d2), c = dot(d1, r), e = dot(d2, d2), f = dot(d2, r);
    float d = a * e - b * b;
    if (!(d > EPS)) return false;
    float d_inv = 1.0f / d;
    s = (b * f - c * e) * d_inv;
    t = (a * f - b * c) * d_inv;
    return true;
}
enum { RCYL_INTERSECTS = 0, RCYL_FAR = 1, RCYL_PARALLEL = 2 };
// geom.cpp:1225-1274.  Returns the kind; normal / dist_sqr are set when it intersects.
B2D_D int intersect_ray_cylinder(v3 p0, v3 p1, v3 pos, q4 orn, float radius, float half_length, int axis,
                                 float &fraction_in, float &dist_sqr, v3 &normal) {
    v3 dir = rotate(orn, axis_vec(axis));
    v3 v0 = pos + dir * half_length, v1 = pos - dir * half_length;
    float s, t;
    if (!closest_point_line_line(v0, v1, p0, p1, s, t)) return RCYL_PARALLEL;
    float radius_sqr = square(radius);
    normal = lerp(p0, p1, t) - lerp(v0, v1, s);
    dist_sqr = length_sqr(normal);
    if (dist_sqr > radius_sqr) return RCYL_FAR;
    v3 d = p1 - p0, e = v1 - v0;
    float dd = dot(d, d), ee = dot(e, e), de = dot(d, e);
    float delta_sqr = (radius_sqr - dist_sqr) * ee / (dd * ee - de * de);
    fraction_in = t - sqrtf(delta_sqr);
    return RCYL_INTERSECTS;
}
B2D_D v3 normalize(v3 v) { return v / length(v); }                              // vector3.hpp:231-235

B2D_D RayHit ray_miss() { RayHit r; r.hit = false; r.fraction = SCALAR_MAX; r.normal = mk3(0, 0, 0); r.feature = RAY_FEATURE_NONE; return r; }

B2D_D RayHit raycast_sphere(float4 sp, v3 pos, v3 p0, v3 p1) {                  // raycast.cpp:182-195
    RayHit r = ray_miss();
    float t;
    if (!intersect_ray_sphere(p0, p1, pos, sp.x, t)) return r;
    r.hit = true; r.fraction = t; r.normal = normalize(lerp(p0, p1, t) - pos);
    return r;
}
B2D_D RayHit raycast_box(float4 sp, v3 pos, q4 orn, v3 p0w, v3 p1w) {           // raycast.cpp:58-109
    RayHit r = ray_miss();
    v3 p0 = to_object(p0w, pos, orn), p1 = to_object(p1w, pos, orn), dir = p1 - p0, he = mk3(sp);
    float t_min = -SCALAR_MAX, t_max = SCALAR_MAX;
    int face = -1;
    #pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float di = get(dir, i), pi = get(p0, i), hi = get(he, i);
        if (fabsf(di) < EPS) {
            if (fabsf(pi) > hi) return r;
        } else {
            float d_inv = 1.0f / di;
            float t1 = (-hi - pi) * d_inv, t2 = (hi - pi) * d_inv;
            if (t1 > t2) { float x = t1; t1 = t2; t2 = x; }
            if (t1 > t_min) face = i * 2 + (pi > 0 ? 0 : 1);
            t_min = t_min < t1 ? t1 : t_min;                   // std::max
            t_max = t2 < t_max ? t2 : t_max;                   // std::min
            if (t_min > t_max) return r;
        }
    }
    if (face < 0) return r;                                    // the reference reads get_face_normal(SIZE_MAX) here
    r.hit = true; r.fraction = t_min; r.normal = rotate(orn, face_normal(face)); r.feature = (uint32_t)face;
    return r;
}
B2D_D RayHit raycast_capsule(float4 sp, v3 pos, q4 orn, v3 p0, v3 p1) {         // raycast.cpp:197-257
    RayHit r = ray_miss();
    float u_in = 0, dist_sqr = 0; v3 n = mk3(0, 0, 0);
    const int kind = intersect_ray_cylinder(p0, p1, pos, orn, sp.x, sp.y, (int)sp.z, u_in, dist_sqr, n);
    if (kind == RCYL_FAR) return r;
    v3 v[2]; capsule_vertices(sp, pos, orn, v);
    v3 cap_dir = v[1] - v[0];
    int hemi;
    if (kind == RCYL_PARALLEL) {
        hemi = dot(p0 - pos, cap_dir) < 0 ? 0 : 1;
    } else {
        v3 x = lerp(p0, p1, u_in);
        float pr0 = dot(x - v[0], cap_dir), pr1 = dot(x - v[1], cap_dir);
        if (pr0 > 0 && pr1 < 0) {
            r.hit = true; r.fraction = u_in; r.normal = n / sqrtf(dist_sqr); r.feature = RAY_CAPSULE_SIDE;
            return r;
        }
        hemi = pr0 < 0 ? 0 : 1;
    }
    float f;
    if (!intersect_ray_sphere(p0, p1, v[hemi], sp.x, f)) return r;
    // the reference takes lerp(p0, p1, u_in) - pos here (raycast.cpp:217-218): the wrong point from the wrong centre
    r.hit = true; r.fraction = f; r.normal = normalize(lerp(p0, p1, f) - v[hemi]); r.feature = (uint32_t)hemi;
    return r;
}
B2D_D RayHit raycast_plane(float4 sp, v3 p0, v3 p1) {                          // raycast.cpp:356-378
    RayHit r = ray_miss();
    v3 n = mk3(sp);
    v3 c = n * sp.w;
    float d = dot(p1 - p0, n), e = dot(c - p0, n);
    if (fabsf(d) < EPS) {
        if (!(fabsf(e) < EPS)) return r;
        r.fraction = 0.0f;
    } else {
        r.fraction = e / d;
    }
    r.hit = true; r.normal = n;
    return r;
}
B2D_D RayHit shape_raycast(int kind, float4 sp, v3 pos, q4 orn, v3 p0, v3 p1) {
    switch (kind) {
    case SH_SPHERE: return raycast_sphere(sp, pos, p0, p1);
    case SH_BOX: return raycast_box(sp, pos, orn, p0, p1);
    case SH_CAPSULE: return raycast_capsule(sp, pos, orn, p0, p1);
    case SH_PLANE: return raycast_plane(sp, p0, p1);
    default: return ray_miss();
    }
}

} // namespace b2d
