// TEST INFRASTRUCTURE -- CPU oracle (see ora_math.hpp header).  extern "C" surface used by
// oracle/oracle.py (ctypes).  Array layouts mirror include/b2d.h so tests feed both sides identically.
#include "ora_world.hpp"
#include <cstring>

using namespace ora;

namespace {
vec3 v3(const float *p) { return {p[0], p[1], p[2]}; }
quat q4(const float *p) { return {p[0], p[1], p[2], p[3]}; }
void put3(float *p, vec3 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
void put4(float *p, quat q) { p[0] = q.x; p[1] = q.y; p[2] = q.z; p[3] = q.w; }
mat3 m9(const float *p) { return {{{p[0], p[1], p[2]}, {p[3], p[4], p[5]}, {p[6], p[7], p[8]}}}; }
void put9(float *p, const mat3 &m) { for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) p[i * 3 + j] = m.row[i][j]; }
shape mk_shape(uint32_t kind, const float *p) { shape s; s.kind = kind; for (int i = 0; i < 4; ++i) s.p[i] = p[i]; return s; }
}

extern "C" {

void *ora_create(float dt, int vel_iters, int pos_iters, int threads) {
    World *w = new World();
    w->dt = dt; w->vel_iters = vel_iters; w->pos_iters = pos_iters; w->threads = threads < 1 ? 1 : threads;
    return w;
}
void ora_destroy(void *h) { delete static_cast<World *>(h); }

// kind: 0 dynamic, 1 kinematic, 2 static.  inv_inertia: row-major 3x3 body-space inverse inertia.
int ora_add_bodies(void *h, uint32_t n, const float *pos, const float *orn, const float *linvel, const float *angvel,
                   const float *inv_mass, const float *inv_inertia, const float *gravity, const uint32_t *kind,
                   const uint32_t *shape_kind, const float *shape_params, const float *friction,
                   const float *restitution, const uint64_t *group, const uint64_t *mask) {
    World &w = *static_cast<World *>(h);
    int first = int(w.bodies.size());
    w.bodies.reserve(w.bodies.size() + n);
    for (uint32_t i = 0; i < n; ++i) {
        Body b{};
        b.pos = v3(pos + 3 * i); b.orn = q4(orn + 4 * i);
        b.linvel = v3(linvel + 3 * i); b.angvel = v3(angvel + 3 * i);
        b.kind = kind[i];
        b.inv_m = b.kind == BK_DYNAMIC ? inv_mass[i] : 0;
        b.inv_I = b.kind == BK_DYNAMIC ? m9(inv_inertia + 9 * i) : mat3_zero();
        b.gravity = v3(gravity + 3 * i);
        b.sh = mk_shape(shape_kind[i], shape_params + 4 * i);
        b.friction = friction[i]; b.restitution = restitution[i];
        b.rolling = b.kind == BK_DYNAMIC && (b.sh.kind == SH_SPHERE || b.sh.kind == SH_CAPSULE);
        b.has_filter = group && mask && !(group[i] == ~uint64_t(0) && mask[i] == ~uint64_t(0));
        b.group = group ? group[i] : ~uint64_t(0); b.mask = mask ? mask[i] : ~uint64_t(0);
        if (b.kind == BK_STATIC) b.linvel = b.angvel = vec3{0, 0, 0};
        w.add_body(b);
    }
    return first;
}

// hinge_constraint::set_axes, hinge_constraint.cpp:11-17
int ora_add_hinges(void *h, uint32_t n, const uint32_t *a, const uint32_t *b, const float *pivotA,
                   const float *pivotB, const float *axisA, const float *axisB) {
    World &w = *static_cast<World *>(h);
    int first = int(w.hinges.size());
    for (uint32_t i = 0; i < n; ++i) {
        Hinge hc{};
        hc.a = a[i]; hc.b = b[i];
        hc.pivot[0] = v3(pivotA + 3 * i); hc.pivot[1] = v3(pivotB + 3 * i);
        vec3 p, q;
        vec3 ax = v3(axisA + 3 * i); plane_space(ax, p, q); hc.frame[0] = mat3_columns(ax, p, q);
        ax = v3(axisB + 3 * i); plane_space(ax, p, q); hc.frame[1] = mat3_columns(ax, p, q);
        w.hinges.push_back(hc);
    }
    return first;
}

void ora_remove_bodies(void *h, uint32_t n, const uint32_t *ids) {
    World &w = *static_cast<World *>(h);
    for (uint32_t i = 0; i < n; ++i) if (ids[i] < w.bodies.size()) w.remove_body(ids[i]);
}

void ora_set_sleeping(void *h, int enabled) { static_cast<World *>(h)->sleeping_enabled = enabled != 0; }
// wake_up_entity (util/island_util.cpp): the island follows at the next island update
void ora_wake_bodies(void *h, uint32_t n, const uint32_t *ids) {
    World &w = *static_cast<World *>(h);
    for (uint32_t i = 0; i < n; ++i) if (ids[i] < w.bodies.size()) w.wake_body(ids[i]);
}
void ora_get_sleeping(void *h, uint32_t *asleep) {
    World &w = *static_cast<World *>(h);
    for (size_t i = 0; i < w.bodies.size(); ++i) asleep[i] = w.bodies[i].asleep ? 1u : 0u;
}

void ora_add_exclusions(void *h, uint32_t n, const uint32_t *a, const uint32_t *b) {
    World &w = *static_cast<World *>(h);
    for (uint32_t i = 0; i < n; ++i) w.exclusions.insert(World::key(a[i], b[i]));
}

void ora_remove_exclusions(void *h, uint32_t n, const uint32_t *a, const uint32_t *b) {      // remove_collision_exclusion
    World &w = *static_cast<World *>(h);
    for (uint32_t i = 0; i < n; ++i) w.exclusions.erase(World::key(a[i], b[i]));
}

void ora_step(void *h, int n) { World &w = *static_cast<World *>(h); for (int i = 0; i < n; ++i) w.step(); }

// mask bits: 1 broadphase, 2 narrowphase, 4 islands, 8 solver
void ora_run_phases(void *h, uint32_t mask) {
    World &w = *static_cast<World *>(h);
    if (mask & 1) w.broadphase();
    if (mask & 2) w.narrowphase();
    if (mask & 4) w.islands();
    if (mask & 8) w.solve();
}

uint32_t ora_num_bodies(void *h) { return uint32_t(static_cast<World *>(h)->bodies.size()); }

void ora_get_state(void *h, float *pos, float *orn, float *linvel, float *angvel, float *aabb6, float *inv_IW9) {
    World &w = *static_cast<World *>(h);
    for (size_t i = 0; i < w.bodies.size(); ++i) {
        const Body &b = w.bodies[i];
        if (pos) put3(pos + 3 * i, b.pos);
        if (orn) put4(orn + 4 * i, b.orn);
        if (linvel) put3(linvel + 3 * i, b.linvel);
        if (angvel) put3(angvel + 3 * i, b.angvel);
        if (aabb6) { put3(aabb6 + 6 * i, b.bb.min); put3(aabb6 + 6 * i + 3, b.bb.max); }
        if (inv_IW9) put9(inv_IW9 + 9 * i, b.inv_IW);
    }
}

// Overwrite the transform/velocity of every body (lock-step tests), refreshing AABB and inv_IW like
// the post-step passes do (solver.cpp:453-465).
void ora_set_state(void *h, const float *pos, const float *orn, const float *linvel, const float *angvel) {
    World &w = *static_cast<World *>(h);
    for (size_t i = 0; i < w.bodies.size(); ++i) {
        Body &b = w.bodies[i];
        b.pos = v3(pos + 3 * i); b.orn = q4(orn + 4 * i);
        if (b.kind != BK_STATIC) { b.linvel = v3(linvel + 3 * i); b.angvel = v3(angvel + 3 * i); }
        w.refresh_body(uint32_t(i));
    }
}

uint32_t ora_num_manifolds(void *h) { return uint32_t(static_cast<World *>(h)->manifolds.size()); }

// pairs: 2 uint32 per manifold (body[0], body[1]) in creation order.
void ora_get_pairs(void *h, uint32_t *pairs) {
    World &w = *static_cast<World *>(h);
    for (size_t i = 0; i < w.manifolds.size(); ++i) { pairs[2 * i] = w.manifolds[i].a; pairs[2 * i + 1] = w.manifolds[i].b; }
}

// Per manifold: num points; per point slot (4 per manifold): pivotA(3) pivotB(3) normal(3) local_normal(3)
// distance friction restitution imp_n imp_t0 imp_t1 -> 18 floats; att + lifetime -> 2 uint32.
void ora_get_contacts(void *h, uint32_t *num, float *pt18, uint32_t *pt_u2) {
    World &w = *static_cast<World *>(h);
    for (size_t i = 0; i < w.manifolds.size(); ++i) {
        const Manifold &m = w.manifolds[i];
        num[i] = m.num;
        for (uint32_t k = 0; k < 4; ++k) {
            float *f = pt18 + (i * 4 + k) * 18;
            uint32_t *u = pt_u2 + (i * 4 + k) * 2;
            if (k >= m.num) { std::memset(f, 0, 18 * sizeof(float)); u[0] = u[1] = 0; continue; }
            const Point &p = m.pt[k];
            put3(f, p.pivotA); put3(f + 3, p.pivotB); put3(f + 6, p.normal); put3(f + 9, p.local_normal);
            f[12] = p.distance; f[13] = p.friction; f[14] = p.restitution; f[15] = p.imp_n; f[16] = p.imp_t[0]; f[17] = p.imp_t[1];
            u[0] = p.att; u[1] = p.lifetime;
        }
    }
}

// Merge trace (ora_world.hpp, merge_branch): on = record it in every following narrowphase; get: one word per manifold
// from the last one (zeros where it was off).  Returns the number of words, or MB_COUNT when out is null.
void ora_set_merge_trace(void *h, int on) { static_cast<World *>(h)->trace_merge = on != 0; }
uint32_t ora_get_merge_trace(void *h, uint64_t *out) {
    World &w = *static_cast<World *>(h);
    if (!out) return MB_COUNT;
    for (size_t i = 0; i < w.manifolds.size(); ++i) out[i] = i < w.merge_trace.size() ? w.merge_trace[i] : 0;
    return uint32_t(w.manifolds.size());
}

// Replace all manifolds (solver-only / narrowphase-only tests).  Same layout as ora_get_contacts.
void ora_set_contacts(void *h, uint32_t n, const uint32_t *pairs, const uint32_t *num, const float *pt18, const uint32_t *pt_u2) {
    World &w = *static_cast<World *>(h);
    w.manifolds.clear(); w.manifold_map.clear();
    for (uint32_t i = 0; i < n; ++i) {
        Manifold m{}; m.a = pairs[2 * i]; m.b = pairs[2 * i + 1]; m.num = num[i];
        for (uint32_t k = 0; k < m.num; ++k) {
            const float *f = pt18 + (size_t(i) * 4 + k) * 18;
            const uint32_t *u = pt_u2 + (size_t(i) * 4 + k) * 2;
            Point &p = m.pt[k];
            p.pivotA = v3(f); p.pivotB = v3(f + 3); p.normal = v3(f + 6); p.local_normal = v3(f + 9);
            p.distance = f[12]; p.friction = f[13]; p.restitution = f[14]; p.imp_n = f[15]; p.imp_t[0] = f[16]; p.imp_t[1] = f[17];
            p.att = u[0]; p.lifetime = u[1];
        }
        w.manifold_map[World::key(m.a, m.b)] = uint32_t(w.manifolds.size());
        w.manifolds.push_back(m);
    }
}

// Replaces the partition the next PH_SOLVE groups its rows by (the per-island position-iteration early-out is the one
// place where it matters).  Tests use it to follow the reference's island BOOKKEEPING, which can lag the connected
// components: a split pending on an island is lost when that island is merged into a bigger one the same step
// (island_manager.cpp:352-357 after :297-350).
void ora_set_islands(void *h, const uint32_t *label) {
    World &w = *static_cast<World *>(h);
    w.island.assign(label, label + w.bodies.size());
}
void ora_get_islands(void *h, uint32_t *label) {
    World &w = *static_cast<World *>(h);
    if (w.island.size() != w.bodies.size()) w.islands();
    std::memcpy(label, w.island.data(), w.island.size() * sizeof(uint32_t));
}

void ora_get_hinge_impulses(void *h, float *imp5) {
    World &w = *static_cast<World *>(h);
    for (size_t i = 0; i < w.hinges.size(); ++i) {
        for (int k = 0; k < 3; ++k) imp5[i * 5 + k] = w.hinges[i].imp_lin[k];
        for (int k = 0; k < 2; ++k) imp5[i * 5 + 3 + k] = w.hinges[i].imp_hinge[k];
    }
}

// Warm-start impulses of the joints (store_applied_impulses, hinge_constraint.cpp:215-259), e.g. taken from the device.
void ora_set_hinge_impulses(void *h, const float *imp5) {
    World &w = *static_cast<World *>(h);
    for (size_t i = 0; i < w.hinges.size(); ++i) {
        for (int k = 0; k < 3; ++k) w.hinges[i].imp_lin[k] = imp5[i * 5 + k];
        for (int k = 0; k < 2; ++k) w.hinges[i].imp_hinge[k] = imp5[i * 5 + 3 + k];
    }
}

// Inject the Gauss-Seidel order the device used: hinge indices, then manifold body pairs.
void ora_set_order(void *h, uint32_t nh, const uint32_t *hinge_idx, uint32_t nm, const uint32_t *pairs) {
    World &w = *static_cast<World *>(h);
    w.use_order = true;
    w.hinge_order.assign(hinge_idx, hinge_idx + nh);
    w.manifold_order.resize(nm); w.point_order.clear();
    for (uint32_t i = 0; i < nm; ++i) w.manifold_order[i] = World::key(pairs[2 * i], pairs[2 * i + 1]);
}
// The same with one entry per contact ROW: (body pair, index of the point in the manifold's list) -- the granularity at
// which the reference orders rows (every contact point is a constraint entity of its own, island_solver.cpp:113-160).
void ora_set_point_order(void *h, uint32_t nh, const uint32_t *hinge_idx, uint32_t nc, const uint32_t *contact3) {
    World &w = *static_cast<World *>(h);
    w.use_order = true;
    w.hinge_order.assign(hinge_idx, hinge_idx + nh);
    w.manifold_order.resize(nc); w.point_order.resize(nc);
    for (uint32_t i = 0; i < nc; ++i) { w.manifold_order[i] = World::key(contact3[3 * i], contact3[3 * i + 1]); w.point_order[i] = contact3[3 * i + 2]; }
}
void ora_set_position_type_order(void *h, int contacts_first) { static_cast<World *>(h)->position_contacts_first = contacts_first != 0; }
void ora_set_position_renormalize_all(int on) { position_renormalize_all = on != 0; }
// Restitution solver: iterations (0 = off) and, per step, the entity graph's orders it depends on (see ora_world.hpp)
void ora_set_restitution_iterations(void *h, int iters, int individual) {
    World &w = *static_cast<World *>(h);
    w.restitution_iters = iters; w.individual_restitution_iters = individual;
}
void ora_set_graph_order(void *h, const uint32_t *adj_off, const uint32_t *adj_nbr, uint32_t n_tagged, const uint32_t *tagged_pairs) {
    World &w = *static_cast<World *>(h);
    const uint32_t nb = uint32_t(w.bodies.size());
    w.adj_off.assign(adj_off, adj_off + nb + 1);
    w.adj_nbr.assign(adj_nbr, adj_nbr + adj_off[nb]);
    w.rest_edge_order.resize(n_tagged);
    for (uint32_t i = 0; i < n_tagged; ++i) w.rest_edge_order[i] = World::key(tagged_pairs[2 * i], tagged_pairs[2 * i + 1]);
    w.graph_order_set = true;
}
void ora_set_pool_order(void *h, int on) { static_cast<World *>(h)->emulate_pool_order = on != 0; }
void ora_clear_order(void *h) { static_cast<World *>(h)->use_order = false; static_cast<World *>(h)->point_order.clear(); }

int ora_should_collide(void *h, uint32_t a, uint32_t b) { return static_cast<World *>(h)->should_collide(a, b) ? 1 : 0; }

// ------------------------------------------------------------------ pure functions (pinned against oracle/_ref)

// The five Jacobians hinge_constraint::prepare builds (hinge_constraint.cpp:26-69), same layout as ref_hinge_rows.
int ora_hinge_rows(const float *pivotA, const float *pivotB, const float *axisA, const float *axisB,
                   const float *posA, const float *ornA, const float *posB, const float *ornB, float *J60) {
    vec3 p, q;
    plane_space(v3(axisA), p, q);
    mat3 frameA = mat3_columns(v3(axisA), p, q);
    vec3 pA = v3(posA), pB = v3(posB); quat qA = q4(ornA), qB = q4(ornB);
    vec3 pivA = to_world(v3(pivotA), pA, qA), pivB = to_world(v3(pivotB), pB, qB);
    vec3 rA = pivA - pA, rB = pivB - pB;
    mat3 sA = {{{0, -rA.z, rA.y}, {rA.z, 0, -rA.x}, {-rA.y, rA.x, 0}}};
    mat3 sB = {{{0, -rB.z, rB.y}, {rB.z, 0, -rB.x}, {-rB.y, rB.x, 0}}};
    const vec3 I[3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int i = 0; i < 3; ++i) { put3(J60 + i * 12, I[i]); put3(J60 + i * 12 + 3, -sA.row[i]); put3(J60 + i * 12 + 6, -I[i]); put3(J60 + i * 12 + 9, sB.row[i]); }
    vec3 pq[2] = {rotate(qA, frameA.column(1)), rotate(qA, frameA.column(2))};
    for (int i = 0; i < 2; ++i) { put3(J60 + (3 + i) * 12, vec3{0, 0, 0}); put3(J60 + (3 + i) * 12 + 3, pq[i]); put3(J60 + (3 + i) * 12 + 6, vec3{0, 0, 0}); put3(J60 + (3 + i) * 12 + 9, -pq[i]); }
    (void)axisB;
    return 5;
}


// out: per point 10 floats (pivotA, pivotB, normal, distance) + att.  Returns the number of points.
int ora_collide(uint32_t kindA, const float *pA, uint32_t kindB, const float *pB, const float *posA, const float *ornA,
                const float *posB, const float *ornB, float *out10, uint32_t *att) {
    shape a = mk_shape(kindA, pA), b = mk_shape(kindB, pB);
    aabb bbA = shape_aabb(a, v3(posA), q4(ornA)), bbB = shape_aabb(b, v3(posB), q4(ornB));
    cctx ctx{v3(posA), q4(ornA), bbA, v3(posB), q4(ornB), bbB, COLLISION_THRESHOLD};
    cresult r;
    collide(a, b, ctx, r);
    for (size_t i = 0; i < r.num; ++i) {
        put3(out10 + 10 * i, r.pt[i].pivotA); put3(out10 + 10 * i + 3, r.pt[i].pivotB); put3(out10 + 10 * i + 6, r.pt[i].normal);
        out10[10 * i + 9] = r.pt[i].distance; att[i] = r.pt[i].att;
    }
    return int(r.num);
}
void ora_shape_aabb(uint32_t kind, const float *p, const float *pos, const float *orn, float *out6) {
    aabb bb = shape_aabb(mk_shape(kind, p), v3(pos), q4(orn));
    put3(out6, bb.min); put3(out6 + 3, bb.max);
}
void ora_integrate(const float *q, const float *w, float dt, float *out4) { put4(out4, integrate(q4(q), v3(w), dt)); }
void ora_plane_space(const float *n, float *p, float *q) { vec3 a, b; plane_space(v3(n), a, b); put3(p, a); put3(q, b); }
int ora_intersect_line_aabb(const float *p0, const float *p1, const float *mn, const float *mx, float *s) {
    return int(intersect_line_aabb({p0[0], p0[1]}, {p1[0], p1[1]}, {mn[0], mn[1]}, {mx[0], mx[1]}, s[0], s[1]));
}
// out: s,t, c1(3), c2(3), sp,tp, c1p(3), c2p(3) -> 16 floats; returns num_points; *dist = squared distance
int ora_closest_segment_segment(const float *p1, const float *q1, const float *p2, const float *q2, float *out16, float *dist) {
    scalar s, t, sp = 0, tp = 0; vec3 c1, c2, c1p{0, 0, 0}, c2p{0, 0, 0}; size_t np = 0;
    *dist = closest_point_segment_segment(v3(p1), v3(q1), v3(p2), v3(q2), s, t, c1, c2, &np, &sp, &tp, &c1p, &c2p);
    out16[0] = s; out16[1] = t; put3(out16 + 2, c1); put3(out16 + 5, c2);
    out16[8] = sp; out16[9] = tp; put3(out16 + 10, c1p); put3(out16 + 13, c2p);
    return int(np);
}
// Sequentially feeds `n` points through maybe_add_point (collision_result.cpp:12-33); returns count, writes pivotA's.
int ora_maybe_add_points(uint32_t n, const float *pivotA, const float *pivotB, float *outA, float *outB) {
    cresult r;
    for (uint32_t i = 0; i < n; ++i) {
        cpoint p{}; p.pivotA = v3(pivotA + 3 * i); p.pivotB = v3(pivotB + 3 * i); p.normal = {0, 1, 0};
        maybe_add_point(r, p);
    }
    for (size_t i = 0; i < r.num; ++i) { put3(outA + 3 * i, r.pt[i].pivotA); put3(outB + 3 * i, r.pt[i].pivotB); }
    return int(r.num);
}
void ora_moment_of_inertia(uint32_t kind, const float *p, float mass, float *out9) { put9(out9, moment_of_inertia(mk_shape(kind, p), mass)); }
void ora_inverse_symmetric(const float *m, float *out9) { put9(out9, inverse_symmetric(m9(m))); }
void ora_world_inertia(const float *orn, const float *inv_I, float *out9) {
    mat3 basis = to_mat3(q4(orn)); put9(out9, basis * m9(inv_I) * transpose(basis));
}
// J: 12 floats; in: inv_mA, inv_IA(9), inv_mB, inv_IB(9), error, erp, restitution, vA wA vB wB (12) -> eff_mass, rhs
void ora_prepare_row(const float *J, float inv_mA, const float *inv_IA, float inv_mB, const float *inv_IB, float error,
                     float erp, float restitution, const float *vels12, float *out2) {
    Row r{}; for (int i = 0; i < 4; ++i) r.J[i] = v3(J + 3 * i);
    prepare_row(r, inv_mA, m9(inv_IA), inv_mB, m9(inv_IB), error, erp, restitution, v3(vels12), v3(vels12 + 3), v3(vels12 + 6), v3(vels12 + 9));
    out2[0] = r.eff_mass; out2[1] = r.rhs;
}
// row5: eff_mass rhs lo hi impulse; returns delta impulse, writes the new impulse into row5[4]
float ora_solve_row(const float *J, float *row5, const float *dv12) {
    Row r{}; for (int i = 0; i < 4; ++i) r.J[i] = v3(J + 3 * i);
    r.eff_mass = row5[0]; r.rhs = row5[1]; r.lo = row5[2]; r.hi = row5[3]; r.impulse = row5[4];
    float d = solve_row(r, v3(dv12), v3(dv12 + 3), v3(dv12 + 6), v3(dv12 + 9));
    row5[4] = r.impulse;
    return d;
}

// constraint_row_friction: J24 = row[0].J[0..3], row[1].J[0..3]; fr6 = eff_mass[2] rhs[2] impulse[2] (impulse updated);
// masses20 = inv_mA, inv_IA(9), inv_mB, inv_IB(9); dv12 = dvA dwA dvB dwB (updated).  warm != 0: warm_start only.
void ora_solve_friction(const float *J24, float *fr6, float mu, float normal_impulse, const float *masses20, float *dv12, int warm) {
    FrictionPair f{};
    for (int i = 0; i < 2; ++i) for (int k = 0; k < 4; ++k) f.J[i][k] = v3(J24 + 12 * i + 3 * k);
    for (int i = 0; i < 2; ++i) { f.eff_mass[i] = fr6[i]; f.rhs[i] = fr6[2 + i]; f.impulse[i] = fr6[4 + i]; }
    f.mu = mu;
    vec3 dvA = v3(dv12), dwA = v3(dv12 + 3), dvB = v3(dv12 + 6), dwB = v3(dv12 + 9);
    const mat3 IA = m9(masses20 + 1), IB = m9(masses20 + 11);
    if (warm) warm_start_friction(f, masses20[0], IA, masses20[10], IB, dvA, dwA, dvB, dwB);
    else solve_friction(f, normal_impulse, masses20[0], IA, masses20[10], IB, dvA, dwA, dvB, dwB);
    fr6[4] = f.impulse[0]; fr6[5] = f.impulse[1];
    put3(dv12, dvA); put3(dv12 + 3, dwA); put3(dv12 + 6, dvB); put3(dv12 + 9, dwB);
}

// contact_constraint::prepare; argument layout of ref_contact_prepare (oracle/ref_glue.cpp)
void ora_contact_prepare(const float *cp14, float dt, const float *a23, const float *b23,
                         float *nJ12, float *n5, float *fJ24, float *fr6, float *mu) {
    Point cp{};
    cp.pivotA = v3(cp14); cp.pivotB = v3(cp14 + 3); cp.normal = v3(cp14 + 6); cp.distance = cp14[9];
    cp.friction = cp14[10]; cp.restitution = cp14[11]; cp.imp_n = cp14[12]; cp.imp_t[0] = cp14[13]; cp.imp_t[1] = cp14[14];
    Row nr{}; FrictionPair f{}; scalar error = 0;
    prepare_contact(cp, dt, v3(a23), q4(a23 + 3), v3(b23), q4(b23 + 3), v3(a23 + 7), v3(a23 + 10), a23[13], m9(a23 + 14),
                    v3(b23 + 7), v3(b23 + 10), b23[13], m9(b23 + 14), nr, error, f);
    for (int k = 0; k < 4; ++k) put3(nJ12 + 3 * k, nr.J[k]);
    n5[0] = nr.lo; n5[1] = nr.hi; n5[2] = nr.impulse; n5[3] = error; n5[4] = cp.restitution;
    for (int i = 0; i < 2; ++i) {
        for (int k = 0; k < 4; ++k) put3(fJ24 + 12 * i + 3 * k, f.J[i][k]);
        fr6[i] = f.eff_mass[i]; fr6[2 + i] = f.rhs[i]; fr6[4 + i] = f.impulse[i];
    }
    *mu = f.mu;
}

// contact_constraint::solve_position + position_solver::solve; argument layout of ref_contact_solve_position.
// A body with inv_m == 0 is non-procedural here (the restatement leaves it untouched, see position_solve).
int ora_contact_solve_position(const float *cp13, float *a26, float *b26, float *out5) {
    Point cp{};
    cp.pivotA = v3(cp13); cp.pivotB = v3(cp13 + 3); cp.normal = v3(cp13 + 6); cp.local_normal = v3(cp13 + 9);
    cp.att = uint32_t(cp13[12]);
    auto load = [](const float *p) {
        Body b{};
        b.pos = v3(p); b.orn = q4(p + 3); b.inv_m = p[7]; b.inv_IW = m9(p + 8); b.inv_I = m9(p + 17);
        b.kind = p[7] != 0 ? BK_DYNAMIC : BK_STATIC;
        return b;
    };
    Body A = load(a26), B = load(b26);
    scalar max_error = 0;
    const bool solved = contact_solve_position(cp, A, B, max_error);
    auto store = [](float *p, const Body &b) { put3(p, b.pos); p[3] = b.orn.x; p[4] = b.orn.y; p[5] = b.orn.z; p[6] = b.orn.w; put9(p + 8, b.inv_IW); };
    store(a26, A); store(b26, B);
    put3(out5, cp.normal); out5[3] = cp.distance; out5[4] = max_error;
    return solved ? 1 : 0;
}

// find_nearest_contact / find_nearest_contact_rolling / should_remove_point; argument layouts of the ref_* twins
uint32_t ora_find_nearest_contact(const float *cpA, const float *cpB, uint32_t n, const float *resA, const float *resB) {
    Point cp{}; cp.pivotA = v3(cpA); cp.pivotB = v3(cpB);
    cresult res{}; res.num = n;
    for (uint32_t i = 0; i < n; ++i) { res.pt[i].pivotA = v3(resA + 3 * i); res.pt[i].pivotB = v3(resB + 3 * i); }
    return uint32_t(find_nearest_contact(cp, res));
}
uint32_t ora_find_nearest_contact_rolling(uint32_t n, const float *resA, const float *cp_pivot, const float *origin, const float *orn,
                                          const float *angvel, float dt) {
    cresult res{}; res.num = n;
    for (uint32_t i = 0; i < n; ++i) res.pt[i].pivotA = v3(resA + 3 * i);
    return uint32_t(find_nearest_contact_rolling(res, v3(cp_pivot), v3(origin), q4(orn), v3(angvel), dt));
}
int ora_should_remove_point(const float *pivotA, const float *pivotB, const float *normal, const float *posA, const float *ornA,
                            const float *posB, const float *ornB) {
    Point cp{}; cp.pivotA = v3(pivotA); cp.pivotB = v3(pivotB); cp.normal = v3(normal);
    return should_remove_point(cp, v3(posA), q4(ornA), v3(posB), q4(ornB)) ? 1 : 0;
}

// hinge_constraint::solve_position through position_solver::solve; hinge12 = pivotA pivotB axisA axisB (set_axes);
// body26 as in ora_contact_solve_position; returns the max error.
float ora_hinge_solve_position(const float *hinge12, float *a26, float *b26) {
    Hinge hc{};
    hc.pivot[0] = v3(hinge12); hc.pivot[1] = v3(hinge12 + 3);
    vec3 p, q;
    vec3 ax = v3(hinge12 + 6); plane_space(ax, p, q); hc.frame[0] = mat3_columns(ax, p, q);
    ax = v3(hinge12 + 9); plane_space(ax, p, q); hc.frame[1] = mat3_columns(ax, p, q);
    auto load = [](const float *pb) {
        Body b{};
        b.pos = v3(pb); b.orn = q4(pb + 3); b.inv_m = pb[7]; b.inv_IW = m9(pb + 8); b.inv_I = m9(pb + 17);
        b.kind = pb[7] != 0 ? BK_DYNAMIC : BK_STATIC;
        return b;
    };
    Body A = load(a26), B = load(b26);
    scalar max_error = 0;
    hinge_solve_position(hc, A, B, max_error);
    auto store = [](float *pb, const Body &b) { put3(pb, b.pos); pb[3] = b.orn.x; pb[4] = b.orn.y; pb[5] = b.orn.z; pb[6] = b.orn.w; put9(pb + 8, b.inv_IW); };
    store(a26, A); store(b26, B);
    return max_error;
}

// material mixing (dynamics/material_mixing.hpp:12-34) and the closed-interval AABB test (math/geom.cpp:762-770)
void ora_material_mix(float frictionA, float frictionB, float restitutionA, float restitutionB, float *out2) {
    out2[0] = material_mix_friction(frictionA, frictionB); out2[1] = material_mix_restitution(restitutionA, restitutionB);
}
int ora_intersect_aabb(const float *a6, const float *b6) {
    aabb a{v3(a6), v3(a6 + 3)}, b{v3(b6), v3(b6 + 3)};
    return intersect(a, b) ? 1 : 0;
}

} // extern "C"
