// TEST INFRASTRUCTURE -- CPU oracle (see ora_math.hpp / ora_world.hpp headers).
#include "ora_world.hpp"
#include <atomic>
#include <cstring>
#include <numeric>
#include <thread>

namespace ora {

// ------------------------------------------------------------------ helpers

template<typename F>
static void parallel_for(int threads, size_t n, F f) {
    if (threads <= 1 || n < 64) { for (size_t i = 0; i < n; ++i) f(i); return; }
    std::atomic<size_t> next{0};
    const size_t chunk = std::max<size_t>(16, n / (size_t(threads) * 8));
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t) pool.emplace_back([&] {
        for (;;) {
            size_t s = next.fetch_add(chunk);
            if (s >= n) break;
            size_t e = std::min(n, s + chunk);
            for (size_t i = s; i < e; ++i) f(i);
        }
    });
    for (auto &th : pool) th.join();
}

// src/edyn/dynamics/moment_of_inertia.cpp:11-91,159-181
mat3 moment_of_inertia(const shape &sh, scalar mass) {
    auto diag = [](vec3 v) { return mat3{{{v.x, 0, 0}, {0, v.y, 0}, {0, 0, v.z}}}; };
    switch (sh.kind) {
    case SH_SPHERE: {
        scalar i = scalar(0.4) * mass * sh.p[0] * sh.p[0];
        return mat3{{{1 * i, 0 * i, 0 * i}, {0 * i, 1 * i, 0 * i}, {0 * i, 0 * i, 1 * i}}};
    }
    case SH_BOX: {
        vec3 ext = vec3{sh.p[0], sh.p[1], sh.p[2]} * scalar(2);
        vec3 v = scalar(1) / scalar(12) * mass * vec3{ext.y * ext.y + ext.z * ext.z,
                                                       ext.z * ext.z + ext.x * ext.x,
                                                       ext.x * ext.x + ext.y * ext.y};
        return diag(v);
    }
    case SH_CAPSULE: {
        scalar radius = sh.p[0], len = sh.p[1] * 2;
        size_t axis = (size_t)sh.p[2];
        scalar cyl_vol = PI * radius * radius * len;                                  // math/shape_volume.cpp:10
        scalar sph_vol = PI * radius * radius * radius * scalar(4) / scalar(3);       // :14
        scalar total = cyl_vol + sph_vol;
        scalar cyl_mass = mass * cyl_vol / total;
        scalar sph_mass = mass * sph_vol / total;
        scalar cxx = scalar(0.5) * cyl_mass * radius * radius;
        scalar cyz = scalar(1) / scalar(12) * cyl_mass * (scalar(3) * radius * radius + len * len);
        // moment_of_inertia_solid_cylinder already permutes by axis (:27-44); the capsule code then reads .x/.y of
        // that permuted vector (:76-77), which is kept as is for axis != x.
        vec3 cyl{cyz, cyz, cyz}; cyl[axis] = cxx;
        scalar sph_i = scalar(0.4) * sph_mass * radius * radius;
        scalar xx = sph_i + cyl.x;
        scalar yy_zz = sph_i + sph_mass * square(scalar(4) * len + scalar(3) * radius) / scalar(64) + cyl.y;
        vec3 v{yy_zz, yy_zz, yy_zz}; v[axis] = xx;
        return diag(v);
    }
    default:
        return diag(vec3{SCALAR_MAX, SCALAR_MAX, SCALAR_MAX});
    }
}

// src/edyn/constraints/constraint_row.cpp:6-22
void prepare_row(Row &row, scalar inv_mA, const mat3 &inv_IA, scalar inv_mB, const mat3 &inv_IB,
                 scalar error, scalar erp, scalar restitution, vec3 vA, vec3 wA, vec3 vB, vec3 wB) {
    scalar J_invM_JT = dot(row.J[0], row.J[0]) * inv_mA + dot(inv_IA * row.J[1], row.J[1]) +
                       dot(row.J[2], row.J[2]) * inv_mB + dot(inv_IB * row.J[3], row.J[3]);
    row.eff_mass = 1 / J_invM_JT;
    scalar relvel = dot(row.J[0], vA) + dot(row.J[1], wA) + dot(row.J[2], vB) + dot(row.J[3], wB);
    row.rhs = -(error * erp + relvel * (1 + restitution));
}

// src/edyn/constraints/constraint_row.cpp:38-57
scalar solve_row(Row &row, vec3 dvA, vec3 dwA, vec3 dvB, vec3 dwB) {
    scalar delta_relvel = dot(row.J[0], dvA) + dot(row.J[1], dwA) + dot(row.J[2], dvB) + dot(row.J[3], dwB);
    scalar delta_impulse = (row.rhs - delta_relvel) * row.eff_mass;
    scalar impulse = row.impulse + delta_impulse;
    if (impulse < row.lo) { delta_impulse = row.lo - row.impulse; row.impulse = row.lo; }
    else if (impulse > row.hi) { delta_impulse = row.hi - row.impulse; row.impulse = row.hi; }
    else row.impulse = impulse;
    return delta_impulse;
}

static scalar effective_mass(const vec3 J[4], scalar inv_mA, const mat3 &inv_IA, scalar inv_mB, const mat3 &inv_IB) {
    // src/edyn/util/constraint_util.cpp:137-146
    scalar s = dot(J[0], J[0]) * inv_mA + dot(inv_IA * J[1], J[1]) + dot(J[2], J[2]) * inv_mB + dot(inv_IB * J[3], J[3]);
    return scalar(1) / s;
}
static scalar relative_speed(const vec3 J[4], vec3 vA, vec3 wA, vec3 vB, vec3 wB) {   // constraint_util.cpp:148-158
    return dot(J[0], vA) + dot(J[1], wA) + dot(J[2], vB) + dot(J[3], wB);
}

// ------------------------------------------------------------------ bodies

uint32_t World::add_body(const Body &b) {
    bodies.push_back(b);
    uint32_t i = uint32_t(bodies.size() - 1);
    bodies[i].dv = bodies[i].dw = vec3{0, 0, 0};
    refresh_body(i);
    if (bodies[i].kind == BK_DYNAMIC) proc_pool.push_back(i);
    return i;
}

void World::refresh_body(uint32_t i) {
    Body &b = bodies[i];
    if (b.kind == BK_DYNAMIC) {                       // util/rigidbody.cpp:75-77, sys/update_inertias.cpp:12-16
        mat3 basis = to_mat3(b.orn);
        b.inv_IW = basis * b.inv_I * transpose(basis);
    } else {
        b.inv_IW = mat3_zero();
    }
    if (b.sh.kind != SH_NONE) b.bb = shape_aabb(b.sh, b.pos, b.orn);
}

bool World::should_collide(uint32_t a, uint32_t b) const {   // collision/should_collide.cpp:23-57
    if (a == b) return false;
    const Body &A = bodies[a], &B = bodies[b];
    if (A.has_filter && B.has_filter) {
        if ((A.group & B.mask) == 0 || (B.group & A.mask) == 0) return false;
    } else if (A.has_filter || B.has_filter) {
        const Body &F = A.has_filter ? A : B;
        const uint64_t all = ~uint64_t(0);
        if ((F.group & all) == 0 || (F.mask & all) == 0) return false;
    }
    if (exclusions.count(key(a, b))) return false;
    return true;
}

// ------------------------------------------------------------------ broadphase

static inline uint64_t cell_key(int64_t x, int64_t y, int64_t z) {
    return (uint64_t(x & 0x1FFFFF) << 42) | (uint64_t(y & 0x1FFFFF) << 21) | uint64_t(z & 0x1FFFFF);
}

// registry.destroy(entity) of a rigid body: its tree node goes (broadphase.cpp:54-68) and island_manager's
// on_destroy<graph_node> destroys every edge entity attached to the node -- contact manifolds and constraints
// (island_manager.cpp:47-66).  Indices stay stable here: the slot becomes a static body without a shape, a joint that
// loses a body is parked on the dead slot (neither end procedural: it is never prepared or solved again).
void World::remove_body(uint32_t i) {
    Body &b = bodies[i];
    if (auto it = std::find(proc_pool.begin(), proc_pool.end(), i); it != proc_pool.end()) { *it = proc_pool.back(); proc_pool.pop_back(); }   // swap and pop
    b.kind = BK_STATIC; b.sh.kind = SH_NONE;
    b.linvel = b.angvel = b.dv = b.dw = vec3{0, 0, 0};
    b.inv_m = 0; b.inv_I = b.inv_IW = mat3_zero();
    size_t w = 0;
    for (size_t k = 0; k < manifolds.size(); ++k) {
        if (manifolds[k].a == i || manifolds[k].b == i) continue;
        if (w != k) manifolds[w] = manifolds[k];
        ++w;
    }
    if (w != manifolds.size()) {
        manifolds.resize(w);
        manifold_map.clear();
        for (uint32_t k = 0; k < manifolds.size(); ++k) manifold_map[key(manifolds[k].a, manifolds[k].b)] = k;
    }
    for (Hinge &h : hinges) if (h.a == i || h.b == i) { h.a = h.b = i; }
    if (i < island.size()) island[i] = ~0u;
    for (Body &o : bodies) o.asleep = false;       // on_destroy<island_resident> queues the island for wake-up (:74-97); restated coarsely
}

void World::broadphase() {
    // destroy_separated_manifolds, broadphase.cpp:119-134; threshold broadphase.hpp:18
    const scalar sep_thr = BREAKING_THRESHOLD * scalar(1.3);
    const vec3 sep_off = vec3{1, 1, 1} * -sep_thr;
    {
        size_t w = 0;
        for (size_t i = 0; i < manifolds.size(); ++i) {
            const Manifold &m = manifolds[i];
            // view<contact_manifold>(exclude_sleeping_disabled), broadphase.cpp:121: a sleeping manifold is left alone
            const bool sleeping = !bodies[m.a].awake() && !bodies[m.b].awake();
            if (!sleeping && !intersect(inset(bodies[m.a].bb, sep_off), bodies[m.b].bb)) continue;
            if (w != i) manifolds[w] = manifolds[i];
            ++w;
        }
        if (w != manifolds.size()) {
            manifolds.resize(w);
            manifold_map.clear();
            for (uint32_t i = 0; i < manifolds.size(); ++i) manifold_map[key(manifolds[i].a, manifolds[i].b)] = i;
        }
    }

    // Candidate search structure.  The reference walks two dynamic AABB trees (broadphase.cpp:183-194);
    // the tree's fat margin does not influence the result because of the exact re-test at :150, so any
    // exact spatial index yields the same pair set.  Uniform grid over "regular" bodies + a brute-force
    // list for bodies larger than a cell (planes).
    const uint32_t n = uint32_t(bodies.size());
    const scalar margin = BREAKING_THRESHOLD;
    scalar sum = 0; uint32_t cnt = 0;
    std::vector<scalar> ext(n, 0);
    for (uint32_t i = 0; i < n; ++i) {
        const Body &b = bodies[i];
        if (b.sh.kind == SH_NONE) continue;
        vec3 e = b.bb.max - b.bb.min;
        ext[i] = std::max(e.x, std::max(e.y, e.z));
        if (b.procedural()) { sum += ext[i]; ++cnt; }
    }
    const scalar big = cnt ? 4 * (sum / cnt) : SCALAR_MAX;
    scalar cell = 0;
    std::vector<uint32_t> large;
    std::vector<uint8_t> is_large(n, 0);
    for (uint32_t i = 0; i < n; ++i) {
        if (bodies[i].sh.kind == SH_NONE) continue;
        if (bodies[i].sh.kind == SH_PLANE || ext[i] > big) { large.push_back(i); is_large[i] = 1; }
        else cell = std::max(cell, ext[i]);
    }
    cell = cell + 2 * margin + scalar(1e-3);
    const scalar inv_cell = 1 / cell;
    std::unordered_map<uint64_t, std::vector<uint32_t>> grid;
    grid.reserve(n);
    std::vector<int64_t> cx(n), cy(n), cz(n);
    for (uint32_t i = 0; i < n; ++i) {
        const Body &b = bodies[i];
        if (b.sh.kind == SH_NONE || is_large[i]) continue;
        vec3 c = (b.bb.min + b.bb.max) * scalar(0.5);
        cx[i] = (int64_t)std::floor(c.x * inv_cell); cy[i] = (int64_t)std::floor(c.y * inv_cell); cz[i] = (int64_t)std::floor(c.z * inv_cell);
        grid[cell_key(cx[i], cy[i], cz[i])].push_back(i);
    }

    const vec3 off = vec3{1, 1, 1} * -BREAKING_THRESHOLD;      // m_aabb_offset, broadphase.hpp:15
    // Awake procedural bodies issue the queries (broadphase.cpp:183) in the order of view<AABB, procedural_tag>: newest
    // first = descending index (confirmed against the real stepper, tests/test_ref_stepper.py; after removals see
    // emulate_pool_order).  This fixes which body becomes body[0].
    // The queries themselves are independent and run on all threads (collide_tree_async, broadphase.cpp:157-175, stores the
    // hits per entity); the manifolds are then created serially in view order (finish_async_update, :197-214), because
    // a pair found by an earlier query must not be created again by its partner's.
    std::vector<std::vector<uint32_t>> hits(n);
    parallel_for(threads, n, [&](size_t idx) {
        const uint32_t ii = uint32_t(idx);
        const Body &A = bodies[ii];
        if (!A.awake() || A.sh.kind == SH_NONE) return;          // view<AABB, procedural_tag>(exclude_sleeping_disabled)
        const aabb q = inset(A.bb, off);
        std::vector<uint32_t> &cand = hits[ii];
        auto test = [&](uint32_t j) {
            if (j == ii) return;
            if (!should_collide(ii, j)) return;
            if (manifold_map.count(key(ii, j))) return;
            if (intersect(q, bodies[j].bb)) cand.push_back(j);
        };
        if (!is_large[ii]) {
            for (int64_t dx = -1; dx <= 1; ++dx) for (int64_t dy = -1; dy <= 1; ++dy) for (int64_t dz = -1; dz <= 1; ++dz) {
                auto it = grid.find(cell_key(cx[ii] + dx, cy[ii] + dy, cz[ii] + dz));
                if (it == grid.end()) continue;
                for (uint32_t j : it->second)
                    if (cx[j] == cx[ii] + dx && cy[j] == cy[ii] + dy && cz[j] == cz[ii] + dz) test(j);
            }
        } else {
            for (uint32_t j = 0; j < n; ++j) if (!is_large[j] && bodies[j].sh.kind != SH_NONE) test(j);
        }
        for (uint32_t j : large) test(j);
        // procedural tree first, then the non-procedural tree (broadphase.cpp:189-192); ascending id inside each.
        std::sort(cand.begin(), cand.end(), [&](uint32_t x, uint32_t y) {
            bool px = bodies[x].procedural(), py = bodies[y].procedural();
            if (px != py) return px;
            return x < y;
        });
    });
    auto create_for = [&](uint32_t ii) {
        for (uint32_t j : hits[ii]) {                   // make_contact_manifold, util/constraint_util.cpp:67-102
            if (manifold_map.count(key(ii, j))) continue;        // made a moment ago by the partner's (earlier) query
            Manifold m{}; m.a = ii; m.b = j; m.num = 0;
            manifold_map[key(ii, j)] = uint32_t(manifolds.size());
            manifolds.push_back(m);
        }
    };
    if (emulate_pool_order) { for (size_t k = proc_pool.size(); k-- > 0;) create_for(proc_pool[k]); }
    else for (uint32_t ii = n; ii-- > 0;) create_for(ii);
}

// ------------------------------------------------------------------ narrowphase

// src/edyn/util/collision_util.cpp:233-255; *via_B (merge trace): the nearest point won through pivot B
size_t find_nearest_contact(const Point &cp, const cresult &res, bool *via_B) {
    scalar shortest = square(CACHING_THRESHOLD);
    size_t nearest = res.num;
    for (size_t i = 0; i < res.num; ++i) {
        scalar dA = length_sqr(res.pt[i].pivotA - cp.pivotA);
        scalar dB = length_sqr(res.pt[i].pivotB - cp.pivotB);
        if (dA < shortest) { shortest = dA; nearest = i; if (via_B) *via_B = false; }
        if (dB < shortest) { shortest = dB; nearest = i; if (via_B) *via_B = true; }
    }
    return nearest;
}
// src/edyn/util/collision_util.cpp:257-280 (uses result.pivotA for either body, as the reference does)
size_t find_nearest_contact_rolling(const cresult &res, vec3 cp_pivot, vec3 origin, quat orn, vec3 angvel, scalar dt) {
    size_t nearest = res.num;
    quat prev_orn = integrate(orn, angvel, -dt);
    vec3 prev_pivot = to_world(cp_pivot, origin, prev_orn);
    scalar shortest = square(CACHING_THRESHOLD);
    for (size_t i = 0; i < res.num; ++i) {
        vec3 pA = to_world(res.pt[i].pivotA, origin, orn);
        scalar d = distance_sqr(pA, prev_pivot);
        if (d < shortest) { shortest = d; nearest = i; }
    }
    return nearest;
}
// src/edyn/util/collision_util.cpp:397-413
bool should_remove_point(const Point &cp, vec3 posA, quat ornA, vec3 posB, quat ornB) {
    const scalar thr = BREAKING_THRESHOLD;
    const scalar thr_sqr = thr * thr;
    vec3 pA = to_world(cp.pivotA, posA, ornA);
    vec3 pB = to_world(cp.pivotB, posB, ornB);
    vec3 n = cp.normal;
    vec3 d = pA - pB;
    scalar nd = dot(d, n);
    vec3 td = d - nd * n;
    return nd > thr || length_sqr(td) > thr_sqr;
}
// src/edyn/util/collision_util.cpp:205-231
static void merge_point(const cpoint &rp, Point &cp, quat ornA, quat ornB) {
    cp.pivotA = rp.pivotA; cp.pivotB = rp.pivotB; cp.normal = rp.normal;
    cp.distance = rp.distance; cp.att = rp.att;
    if (rp.att != ATT_NONE) cp.local_normal = rotate(conjugate(rp.att == ATT_A ? ornA : ornB), rp.normal);
    else cp.local_normal = vec3{0, 0, 0};
}
// src/edyn/util/collision_util.cpp:319-395 + :282-317 (material mix; dynamics/material_mixing.hpp:12-18)
static Point create_point(const cpoint &rp, const Body &A, const Body &B) {
    Point cp{};
    cp.pivotA = rp.pivotA; cp.pivotB = rp.pivotB; cp.normal = rp.normal;
    cp.att = rp.att; cp.distance = rp.distance;
    if (rp.att != ATT_NONE) cp.local_normal = rotate(conjugate(rp.att == ATT_A ? A.orn : B.orn), rp.normal);
    else cp.local_normal = vec3{0, 0, 0};
    cp.friction = material_mix_friction(A.friction, B.friction);
    cp.restitution = material_mix_restitution(A.restitution, B.restitution);
    cp.lifetime = 0; cp.imp_n = 0; cp.imp_t[0] = cp.imp_t[1] = 0;
    return cp;
}

// include/edyn/util/collision_util.hpp:105-276, sequential flavour (narrowphase.hpp:62-84): points are
// destroyed/created immediately; new points are pushed at the head of the manifold's list.  tr (may be null): the
// merge_branch bits this call took.
static void process_collision(Manifold &m, const cresult &res, const Body &A, const Body &B, scalar dt, uint64_t *tr) {
    uint64_t t = 0;
    auto hit = [&](uint32_t b) { t |= uint64_t(1) << b; };
    bool merged[4] = {false, false, false, false};
    const size_t num0 = m.num;
    uint32_t slot[4] = {0, 1, 2, 3};                 // the slot each point of the list sat in when the step started
    unsigned removed = 0;                            // by slot
    size_t i = 0;
    while (i < m.num) {
        Point &cp = m.pt[i];
        ++cp.lifetime;
        bool via_B = false;
        size_t nearest = find_nearest_contact(cp, res, &via_B);
        uint32_t how = via_B ? MB_NEAREST_B : MB_NEAREST_A;
        if (nearest == res.num && A.rolling) { nearest = find_nearest_contact_rolling(res, cp.pivotA, A.pos, A.orn, A.angvel, dt); how = MB_ROLL_A; }
        if (nearest == res.num && B.rolling) {
            if (A.rolling) hit(MB_ROLL_BOTH);
            nearest = find_nearest_contact_rolling(res, cp.pivotB, B.pos, B.orn, B.angvel, dt); how = MB_ROLL_B;
        }
        if (nearest < res.num && !merged[nearest]) {
            hit(how);
            merge_point(res.pt[nearest], cp, A.orn, B.orn);
            merged[nearest] = true;
            ++i;
            continue;
        }
        if (nearest < res.num) hit(MB_TAKEN);
        if (should_remove_point(cp, A.pos, A.orn, B.pos, B.orn)) {
            const vec3 d = to_world(cp.pivotA, A.pos, A.orn) - to_world(cp.pivotB, B.pos, B.orn);
            hit(dot(d, cp.normal) > BREAKING_THRESHOLD ? MB_REMOVE_NORMAL : MB_REMOVE_TANGENT);
            removed |= 1u << slot[i];
            for (size_t k = i + 1; k < m.num; ++k) { m.pt[k - 1] = m.pt[k]; slot[k - 1] = slot[k]; }
            --m.num;
        } else {
            hit(MB_KEPT);
            ++i;
        }
    }
    if (num0 == 0 && res.num == 0) hit(MB_EARLY_RETURN);
    if (res.num == 0 && m.num > 0) hit(MB_EMPTY_KEEP);
    if (res.num == 0 && removed) hit(MB_EMPTY_REMOVE);
    if (removed && num0 >= 2) {
        if (removed & 1u) hit(MB_REMOVE_FIRST);
        if (removed >> (num0 - 1) & 1u) hit(MB_REMOVE_LAST);
        if (removed & ((1u << (num0 - 1)) - 1u) & ~1u) hit(MB_REMOVE_MIDDLE);
        for (size_t k = 1; k + 1 < num0; ++k)
            if (!(removed >> k & 1u) && (removed & ((1u << k) - 1u)) && (removed >> (k + 1))) hit(MB_REMOVE_GAP);
        if (num0 == 4 && removed == 15u) hit(MB_REMOVE_ALL4);
    }
    bool all = true;
    for (size_t k = 0; k < res.num; ++k) all = all && merged[k];
    if (all) {
        if (num0 > 0 && res.num > 0 && !removed) hit(MB_SETTLED);
        if (tr) *tr = t;
        return;
    }

    struct Local { cpoint p; int ent; insert_type type; };
    Local L[4];
    for (auto &l : L) { l.ent = -1; l.type = INS_NONE; }
    size_t num_points = m.num;
    if (num_points > 0) {
        for (size_t k = 0; k < m.num; ++k) {
            L[k].p = cpoint{m.pt[k].pivotA, m.pt[k].pivotB, m.pt[k].normal, m.pt[k].distance, ATT_NONE};
            L[k].ent = int(k);
        }
    } else {
        ++num_points;
        L[0].p = res.pt[0];
        L[0].type = INS_APPEND;
        merged[0] = true;
    }
    // insertion_point_index with the branch it took recorded
    auto insert = [&](const vec3 *pivots, vec3 p) {
        const size_t n = num_points;
        int col = -1;
        const insert_res ir = insertion_point_index(pivots, 4, num_points, p, &col);
        static const uint32_t b1[4] = {MB_COUNT, MB_INS1_SIMILAR, MB_COUNT, MB_INS1_APPEND};
        static const uint32_t b3[4] = {MB_INS3_COL1, MB_INS3_COL0, MB_INS3_COL2, MB_INS3_SHORTEST};
        if (n == 1) hit(b1[ir.type]);
        else if (n == 2) hit(ir.type == INS_APPEND ? MB_INS2_APPEND : ir.type == INS_SIMILAR ? MB_INS2_SIMILAR
                             : ir.type == INS_REPLACE ? MB_INS2_REPLACE0 + uint32_t(ir.index) : MB_INS2_NONE);
        else if (n == 3) hit(ir.type == INS_NONE ? MB_INS3_NONE : ir.type == INS_APPEND ? MB_INS3_APPEND : b3[col]);
        else if (n == 4) hit(ir.type == INS_SIMILAR ? MB_INS4_SIMILAR : ir.type == INS_REPLACE ? MB_INS4_REPLACE0 + uint32_t(ir.index) : MB_INS4_NONE);
        return ir;
    };
    for (size_t k = 0; k < res.num; ++k) {
        if (merged[k]) continue;
        const cpoint &rp = res.pt[k];
        vec3 pivots[4];
        for (size_t j = 0; j < num_points; ++j) pivots[j] = L[j].p.pivotA;
        insert_res ir = insert(pivots, rp.pivotA);
        if (ir.type == INS_NONE) {
            for (size_t j = 0; j < num_points; ++j) pivots[j] = L[j].p.pivotB;
            ir = insert(pivots, rp.pivotB);
            if (ir.type != INS_NONE) hit(MB_PIVOT_B);
        }
        if (ir.type != INS_NONE) {
            if (L[ir.index].type == INS_REPLACE && ir.type == INS_SIMILAR) hit(MB_REPLACE_THEN_SIMILAR);
            if (L[ir.index].type == INS_SIMILAR && ir.type == INS_REPLACE) hit(MB_SIMILAR_THEN_REPLACE);
            L[ir.index].p = rp; L[ir.index].type = ir.type;
        }
    }
    Point existing[4]; bool alive[4] = {false, false, false, false}, similar[4] = {false, false, false, false};
    const size_t n_exist = m.num;
    for (size_t k = 0; k < n_exist; ++k) { existing[k] = m.pt[k]; alive[k] = true; }
    Point created[4]; size_t n_created = 0;
    for (size_t k = 0; k < num_points; ++k) {
        Local &l = L[k];
        switch (l.type) {
        case INS_NONE: break;
        case INS_APPEND: created[n_created++] = create_point(l.p, A, B); break;
        case INS_SIMILAR:
            if (l.ent < 0) { hit(MB_SIMILAR_CREATED); created[n_created++] = create_point(l.p, A, B); }
            else { similar[l.ent] = true; merge_point(l.p, existing[l.ent], A.orn, B.orn); }
            break;
        case INS_REPLACE:
            if (l.ent >= 0) {
                hit(MB_REPLACE_PERSISTED);
                if (slot[l.ent] != uint32_t(l.ent)) hit(MB_REPLACE_AFTER_GAP);
                alive[l.ent] = false;
            }
            created[n_created++] = create_point(l.p, A, B);
            break;
        }
    }
    size_t w = 0;
    for (size_t k = n_created; k-- > 0;) m.pt[w++] = created[k];      // last created = list head
    for (size_t k = 0; k < n_exist; ++k) {
        if (!alive[k]) continue;
        if (w > slot[k]) hit(MB_MOVE_UP);
        if (w < slot[k]) hit(MB_MOVE_DOWN);
        if (similar[k]) hit(w == slot[k] ? MB_SIMILAR_INPLACE : MB_SIMILAR_MOVED);
        m.pt[w++] = existing[k];
    }
    m.num = uint32_t(w);
    if (w == 4) hit(MB_FULL4);
    if ((t >> MB_MOVE_UP & 1u) && (t >> MB_MOVE_DOWN & 1u)) hit(MB_MOVE_BOTH);
    if (tr) *tr = t;
}

void World::narrowphase() {
    if (trace_merge) merge_trace.assign(manifolds.size(), 0);
    parallel_for(threads, manifolds.size(), [&](size_t mi) {
        Manifold &m = manifolds[mi];
        const Body &A = bodies[m.a], &B = bodies[m.b];
        if (!A.awake() && !B.awake()) return;                     // narrowphase.cpp:31 excludes sleeping manifolds
        // update_contact_distances, collision_util.cpp:28-45
        for (size_t k = 0; k < m.num; ++k) {
            Point &cp = m.pt[k];
            vec3 pAw = to_world(cp.pivotA, A.pos, A.orn);
            vec3 pBw = to_world(cp.pivotB, B.pos, B.orn);
            cp.distance = dot(cp.normal, pAw - pBw);
        }
        cresult res;
        detect_collision(A.sh, B.sh, A.pos, A.orn, A.bb, B.pos, B.orn, B.bb, res);
        process_collision(m, res, A, B, dt, trace_merge ? &merge_trace[mi] : nullptr);
    });
}

// ------------------------------------------------------------------ islands

// Connected components over procedural (dynamic) nodes; static/kinematic nodes do not connect
// (core/entity_graph.hpp:303-307, simulation/island_manager.cpp:117-247).  Edges: every manifold
// (make_contact_manifold adds a null_constraint edge even with zero points) and every joint.
void World::islands() {
    const uint32_t n = uint32_t(bodies.size());
    std::vector<uint32_t> parent(n);
    std::iota(parent.begin(), parent.end(), 0u);
    auto find = [&](uint32_t x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
    auto unite = [&](uint32_t a, uint32_t b) {
        if (!bodies[a].procedural() || !bodies[b].procedural()) return;
        uint32_t ra = find(a), rb = find(b);
        if (ra == rb) return;
        if (ra < rb) parent[rb] = ra; else parent[ra] = rb;
    };
    for (const Manifold &m : manifolds) unite(m.a, m.b);
    for (const Hinge &h : hinges) unite(h.a, h.b);
    island.assign(n, ~0u);
    for (uint32_t i = 0; i < n; ++i) if (bodies[i].procedural()) island[i] = find(i);
    update_sleep();
}

// wake_up_islands + put_islands_to_sleep (island_manager.cpp:524-539, :568-623) over labels that are recomputed every
// step instead of incrementally maintained island entities:
//  * an island with an awake and a sleeping member has just been joined by a new edge -> insert_to_island ->
//    wake_up_island (:257-295): everybody wakes;
//  * island::sleep_timestamp follows the island entity.  merge_islands keeps the biggest constituent (:303-316),
//    split_islands keeps the original entity for the biggest part (:431-447); restated on labels: a new island takes
//    the timestamp of its biggest previous constituent O (procedural-body count, ties to the smaller label) iff it is
//    also O's biggest heir, otherwise it starts without one;
//  * could_go_to_sleep (:575-603): no member faster than 0.005 m/s or pi/48 rad/s; put_islands_to_sleep (:605-623)
//    with m_last_time = time of the PREVIOUS update (set at :538), time of update j = j * fixed_dt, attach time 0.
void World::update_sleep() {
    const uint32_t n = uint32_t(bodies.size());
    const uint64_t j = updates++;
    if (!sleeping_enabled) return;
    prev_island.resize(n, ~0u); isl_size.resize(n, 0); isl_sleep_ts.resize(n, -1.0);
    const double last_time = j ? double(j - 1) * double(dt) : 0.0;
    std::vector<uint32_t> size_new(n, 0);
    std::vector<uint8_t> any_awake(n, 0), any_fast(n, 0);
    std::vector<uint64_t> contributor(n, 0), heir(n, 0);
    const scalar lin2 = scalar(0.005) * scalar(0.005), ang2 = (PI / scalar(48)) * (PI / scalar(48));
    for (uint32_t i = 0; i < n; ++i) {
        const Body &b = bodies[i];
        if (!b.procedural()) continue;
        const uint32_t r = island[i];
        ++size_new[r];
        if (!b.asleep) any_awake[r] = 1;
        if (length_sqr(b.linvel) > lin2 || length_sqr(b.angvel) > ang2) any_fast[r] = 1;
        const uint32_t o = prev_island[i];
        if (o != ~0u) contributor[r] = std::max(contributor[r], (uint64_t(isl_size[o]) << 32) | uint64_t(~o));
    }
    for (uint32_t i = 0; i < n; ++i) {
        if (!bodies[i].procedural()) continue;
        const uint32_t o = prev_island[i], r = island[i];
        if (o != ~0u) heir[o] = std::max(heir[o], (uint64_t(size_new[r]) << 32) | uint64_t(~r));
    }
    std::vector<double> ts_new(n, -1.0);
    std::vector<uint8_t> sleep_now(n, 0);
    for (uint32_t r = 0; r < n; ++r) {
        if (!size_new[r] || !any_awake[r]) continue;              // sleeping islands are not visited (exclude_sleeping_disabled)
        double ts = -1.0;
        if (contributor[r]) {
            const uint32_t o = ~uint32_t(contributor[r] & 0xFFFFFFFFu);
            if (~uint32_t(heir[o] & 0xFFFFFFFFu) == r) ts = isl_sleep_ts[o];
        }
        if (!any_fast[r]) {
            if (ts < 0) ts = last_time;
            else if (last_time - ts > 2.0) { sleep_now[r] = 1; ts = -1.0; }
        } else ts = -1.0;
        ts_new[r] = ts;
    }
    for (uint32_t i = 0; i < n; ++i) {
        Body &b = bodies[i];
        if (!b.procedural()) { prev_island[i] = ~0u; continue; }
        const uint32_t r = island[i];
        if (any_awake[r]) b.asleep = false;
        if (sleep_now[r]) { b.asleep = true; b.linvel = b.angvel = vec3{0, 0, 0}; }       // put_to_sleep, :541-566
        prev_island[i] = r;
    }
    isl_size = size_new;
    isl_sleep_ts = ts_new;
}

// ------------------------------------------------------------------ solver

namespace {
struct SBody {                 // constraint_body + row masses, solver.cpp:101-147
    vec3 v, w; scalar inv_m; mat3 inv_I; bool proc;
};
struct SRow { Row r; uint32_t a, b; };
struct SFric : FrictionPair { uint32_t normal_row; };
struct IslandWork {
    std::vector<uint32_t> hinges;                 // indices into World::hinges
    std::vector<std::pair<uint32_t, uint32_t>> pts;   // (manifold, point)
    std::vector<uint32_t> bodies;
};
}

// solve_friction, constraint_row_friction.cpp:11-54
void solve_friction(FrictionPair &f, scalar normal_impulse, scalar inv_mA, const mat3 &inv_IA, scalar inv_mB, const mat3 &inv_IB,
                    vec3 &dvA, vec3 &dwA, vec3 &dvB, vec3 &dwB) {
    scalar delta[2], imp[2];
    for (int i = 0; i < 2; ++i) {
        scalar drs = relative_speed(f.J[i], dvA, dwA, dvB, dwB);
        delta[i] = (f.rhs[i] - drs) * f.eff_mass[i];
        imp[i] = f.impulse[i] + delta[i];
    }
    scalar len_sqr = imp[0] * imp[0] + imp[1] * imp[1];
    scalar max_len = f.mu * normal_impulse;
    if (len_sqr > square(max_len)) {
        scalar len = std::sqrt(len_sqr);
        if (len > EPS) { imp[0] = imp[0] / len * max_len; imp[1] = imp[1] / len * max_len; }
        else { imp[0] = imp[1] = 0; }
        for (int i = 0; i < 2; ++i) delta[i] = imp[i] - f.impulse[i];
    }
    for (int i = 0; i < 2; ++i) {
        f.impulse[i] = imp[i];
        dvA += inv_mA * f.J[i][0] * delta[i];
        dwA += inv_IA * f.J[i][1] * delta[i];
        dvB += inv_mB * f.J[i][2] * delta[i];
        dwB += inv_IB * f.J[i][3] * delta[i];
    }
}
// warm_start(constraint_row_friction&), constraint_row_friction.cpp:56-66
void warm_start_friction(const FrictionPair &f, scalar inv_mA, const mat3 &inv_IA, scalar inv_mB, const mat3 &inv_IB,
                         vec3 &dvA, vec3 &dwA, vec3 &dvB, vec3 &dwB) {
    for (int i = 0; i < 2; ++i) {
        dvA += inv_mA * f.J[i][0] * f.impulse[i];
        dwA += inv_IA * f.J[i][1] * f.impulse[i];
        dvB += inv_mB * f.J[i][2] * f.impulse[i];
        dwB += inv_IB * f.J[i][3] * f.impulse[i];
    }
}

// contact_constraint::prepare, contact_constraint.cpp:15-56 (origin == position: no centre-of-mass offset is staged)
void prepare_contact(const Point &cp, scalar dt, vec3 posA, quat ornA, vec3 posB, quat ornB,
                     vec3 vA, vec3 wA, scalar inv_mA, const mat3 &inv_IA, vec3 vB, vec3 wB, scalar inv_mB, const mat3 &inv_IB,
                     Row &nr, scalar &error, FrictionPair &f) {
    vec3 pAw = to_world(cp.pivotA, posA, ornA);
    vec3 pBw = to_world(cp.pivotB, posB, ornB);
    vec3 rA = pAw - posA, rB = pBw - posB;
    nr.J[0] = cp.normal; nr.J[1] = cross(rA, cp.normal); nr.J[2] = -cp.normal; nr.J[3] = -cross(rB, cp.normal);
    nr.impulse = cp.imp_n; nr.lo = 0; nr.hi = LARGE;
    error = 0;
    if (cp.distance > 0) error = cp.distance / dt;
    f.mu = cp.friction;
    vec3 t[2]; plane_space(cp.normal, t[0], t[1]);
    for (int i = 0; i < 2; ++i) {
        f.J[i][0] = t[i]; f.J[i][1] = cross(rA, t[i]); f.J[i][2] = -t[i]; f.J[i][3] = -cross(rB, t[i]);
        f.impulse[i] = cp.imp_t[i];
        f.eff_mass[i] = effective_mass(f.J[i], inv_mA, inv_IA, inv_mB, inv_IB);
        f.rhs[i] = -relative_speed(f.J[i], vA, wA, vB, wB);
    }
}

// contact_constraint::solve_position, contact_constraint.cpp:58-90
bool contact_solve_position(Point &cp, Body &A, Body &B, scalar &max_error) {
    vec3 pAw = to_world(cp.pivotA, A.pos, A.orn);
    vec3 pBw = to_world(cp.pivotB, B.pos, B.orn);
    if (cp.att == ATT_A) cp.normal = rotate(A.orn, cp.local_normal);
    else if (cp.att == ATT_B) cp.normal = rotate(B.orn, cp.local_normal);
    cp.distance = dot(pAw - pBw, cp.normal);
    vec3 rA = pAw - A.pos, rB = pBw - B.pos;
    if (cp.distance > -EPS) return false;
    scalar error = -cp.distance;
    vec3 J[4] = {cp.normal, cross(rA, cp.normal), -cp.normal, -cross(rB, cp.normal)};
    position_solve(A, B, J, error, max_error);
    return true;
}

// hinge_constraint::solve_position, hinge_constraint.cpp:180-213
void hinge_solve_position(const Hinge &hc, Body &A, Body &B, scalar &max_error) {
    vec3 axisA = rotate(A.orn, hc.frame[0].column(0));
    vec3 axisB = rotate(B.orn, hc.frame[1].column(0));
    vec3 p, q; plane_space(axisA, p, q);
    vec3 u = cross(axisA, axisB);
    const vec3 z{0, 0, 0};
    { scalar e = dot(u, p); if (std::abs(e) > EPS) { vec3 J[4] = {z, p, z, -p}; position_solve(A, B, J, e, max_error); } }
    { scalar e = dot(u, q); if (std::abs(e) > EPS) { vec3 J[4] = {z, q, z, -q}; position_solve(A, B, J, e, max_error); } }
    vec3 pivotA = to_world(hc.pivot[0], A.pos, A.orn);
    vec3 pivotB = to_world(hc.pivot[1], B.pos, B.orn);
    vec3 dir = pivotA - pivotB;
    scalar e = length(dir);
    if (e > EPS) {
        dir /= e;
        vec3 rA = pivotA - A.pos, rB = pivotB - B.pos;
        vec3 J[4] = {dir, cross(rA, dir), -dir, -cross(rB, dir)};
        position_solve(A, B, J, -e, max_error);
    }
}

static SBody solver_body(const Body &b) {
    SBody s;
    s.proc = b.awake();
    if (s.proc) { s.inv_m = b.inv_m; s.inv_I = b.inv_IW; } else { s.inv_m = 0; s.inv_I = mat3_zero(); }
    if (b.kind == BK_STATIC) { s.v = s.w = vec3{0, 0, 0}; } else { s.v = b.linvel; s.w = b.angvel; }
    return s;
}

bool position_renormalize_all = false;
// position_solver::solve, dynamics/position_solver.hpp:16-51
void position_solve(Body &A, Body &B, const vec3 J[4], scalar error, scalar &max_error) {
    const bool pA = A.awake(), pB = B.awake();
    const scalar inv_mA = pA ? A.inv_m : 0, inv_mB = pB ? B.inv_m : 0;
    mat3 zero = mat3_zero();
    const mat3 &inv_IA = pA ? A.inv_IW : zero;
    const mat3 &inv_IB = pB ? B.inv_IW : zero;
    scalar eff_mass = effective_mass(J, inv_mA, inv_IA, inv_mB, inv_IB);
    scalar correction = error * scalar(0.2) * eff_mass;
    // The reference also runs these updates for non-procedural bodies with zero mass/inertia, which only
    // re-normalises their (unit) orientation -- a no-op unless the quaternion is an ulp off unit length; skipped by
    // default (and on the device) so islands sharing a static body can run in parallel, reproduced on request
    // (position_renormalize_all) to match the reference to the last bit on arbitrarily oriented static bodies.
    if (pA) {
        A.pos += inv_mA * J[0] * correction;
        vec3 acA = inv_IA * J[1] * correction;
        A.orn = A.orn + quat_derivative(A.orn, acA);
        A.orn = normalize(A.orn);
    }
    if (pB) {
        B.pos += inv_mB * J[2] * correction;
        vec3 acB = inv_IB * J[3] * correction;
        B.orn = B.orn + quat_derivative(B.orn, acB);
        B.orn = normalize(B.orn);
    }
    if (position_renormalize_all) {
        if (!pA) A.orn = normalize(A.orn);
        if (!pB) B.orn = normalize(B.orn);
    }
    if (pA) { mat3 basis = to_mat3(A.orn); A.inv_IW = basis * A.inv_I * transpose(basis); }
    if (pB) { mat3 basis = to_mat3(B.orn); B.inv_IW = basis * B.inv_I * transpose(basis); }
    max_error = std::max(std::abs(error), max_error);
}

// ------------------------------------------------------------------ restitution solver
// get_manifold_min_relvel, restitution_solver.cpp:32-83
scalar World::manifold_min_relvel(const Manifold &m) const {
    const Body &A = bodies[m.a], &B = bodies[m.b];
    const vec3 z{0, 0, 0};
    const vec3 lvA = A.kind == BK_STATIC ? z : A.linvel, avA = A.kind == BK_STATIC ? z : A.angvel;
    const vec3 lvB = B.kind == BK_STATIC ? z : B.linvel, avB = B.kind == BK_STATIC ? z : B.angvel;
    scalar min_relvel = SCALAR_MAX;
    for (uint32_t p = 0; p < m.num; ++p) {
        const Point &cp = m.pt[p];
        vec3 pivotA = to_world(cp.pivotA, A.pos, A.orn), pivotB = to_world(cp.pivotB, B.pos, B.orn);
        vec3 rA = pivotA - A.pos, rB = pivotB - B.pos;
        vec3 vA = lvA + cross(avA, rA), vB = lvB + cross(avB, rB);
        vec3 relvel = vA - vB;
        min_relvel = std::min(dot(relvel, cp.normal), min_relvel);
    }
    return min_relvel;
}

// the solve_manifolds lambda, restitution_solver.cpp:146-310: rows of all points of the group from the CURRENT velocities,
// a few Gauss-Seidel sweeps (normal row, then its friction pair), then the delta velocities are applied at once
void World::solve_restitution_group(const std::vector<uint32_t> &group) {
    struct GRow { Row r; FrictionPair f; uint32_t a, b; scalar inv_mA, inv_mB; mat3 inv_IA, inv_IB; };
    std::vector<GRow> rows;
    for (uint32_t mi : group) {
        const Manifold &m = manifolds[mi];
        const Body &A = bodies[m.a], &B = bodies[m.b];
        SBody sA = solver_body(A), sB = solver_body(B);
        for (uint32_t p = 0; p < m.num; ++p) {
            Point cp = m.pt[p];
            cp.imp_n = 0; cp.imp_t[0] = cp.imp_t[1] = 0; cp.distance = 0;             // impulse 0, constraint_row_options{}.error == 0
            GRow g{}; g.a = m.a; g.b = m.b; g.inv_mA = sA.inv_m; g.inv_mB = sB.inv_m; g.inv_IA = sA.inv_I; g.inv_IB = sB.inv_I;
            scalar error;
            prepare_contact(cp, dt, A.pos, A.orn, B.pos, B.orn, sA.v, sA.w, sA.inv_m, sA.inv_I, sB.v, sB.w, sB.inv_m, sB.inv_I, g.r, error, g.f);
            prepare_row(g.r, sA.inv_m, sA.inv_I, sB.inv_m, sB.inv_I, 0, scalar(0.2), cp.restitution, sA.v, sA.w, sB.v, sB.w);
            rows.push_back(g);
        }
    }
    vec3 dummy_dv{0, 0, 0}, dummy_dw{0, 0, 0};                                          // non-procedural bodies (restitution_solver.cpp:85-86)
    auto DV = [&](uint32_t i) -> vec3 & { return bodies[i].awake() ? bodies[i].dv : dummy_dv; };
    auto DW = [&](uint32_t i) -> vec3 & { return bodies[i].awake() ? bodies[i].dw : dummy_dw; };
    for (int it = 0; it < individual_restitution_iters; ++it) {
        for (GRow &g : rows) {
            vec3 &dvA = DV(g.a), &dwA = DW(g.a), &dvB = DV(g.b), &dwB = DW(g.b);
            scalar delta = solve_row(g.r, dvA, dwA, dvB, dwB);
            dvA += g.inv_mA * g.r.J[0] * delta; dwA += g.inv_IA * g.r.J[1] * delta;     // apply_row_impulse, constraint_row.cpp:24-32
            dvB += g.inv_mB * g.r.J[2] * delta; dwB += g.inv_IB * g.r.J[3] * delta;
            solve_friction(g.f, g.r.impulse, g.inv_mA, g.inv_IA, g.inv_mB, g.inv_IB, dvA, dwA, dvB, dwB);
        }
    }
    for (uint32_t mi : group) {
        for (uint32_t i : {manifolds[mi].a, manifolds[mi].b}) {
            Body &b = bodies[i];
            if (b.kind == BK_STATIC) continue;
            b.linvel += b.dv; b.angvel += b.dw;
            b.dv = b.dw = vec3{0, 0, 0};
        }
    }
}

// solve_restitution_iteration, restitution_solver.cpp:88-384, for one island; `tagged` = its manifolds with
// contact_manifold_with_restitution in island.edges order
bool World::restitution_iteration(const std::vector<uint32_t> &tagged) {
    scalar min_relvel = SCALAR_MAX;
    int64_t fastest = -1;
    for (uint32_t mi : tagged) {
        scalar local = manifold_min_relvel(manifolds[mi]);
        if (local < min_relvel) { min_relvel = local; fastest = mi; }
    }
    if (fastest < 0) return true;
    const scalar relvel_threshold = scalar(-0.005);
    if (min_relvel > relvel_threshold) return true;
    const Manifold &fm = manifolds[size_t(fastest)];
    auto connecting = [&](uint32_t i) { return bodies[i].kind == BK_DYNAMIC; };
    scalar speedA = 0, speedB = 0;
    if (bodies[fm.a].kind != BK_STATIC) speedA = length_sqr(bodies[fm.a].linvel);
    if (bodies[fm.b].kind != BK_STATIC) speedB = length_sqr(bodies[fm.b].linvel);
    uint32_t start;
    if (speedA > speedB) start = connecting(fm.a) ? fm.a : fm.b;
    else start = connecting(fm.b) ? fm.b : fm.a;
    // entity_graph::traverse, core/entity_graph.hpp:357-426: breadth first over the adjacency lists
    const uint32_t nb = uint32_t(bodies.size());
    std::vector<uint8_t> visited(nb, 0);
    std::vector<uint32_t> to_visit{start}, group;
    while (!to_visit.empty()) {
        const uint32_t node = to_visit.back();
        to_visit.pop_back();
        visited[node] = 1;
        if (!connecting(node)) continue;
        const uint32_t a0 = adj_off[node], a1 = adj_off[node + 1];
        group.clear();
        for (uint32_t k = a0; k < a1; ++k) {                       // visit_edges: the manifolds of this node, fast enough
            if (!(adj_nbr[k] >> 31)) continue;
            auto it = manifold_map.find(key(node, adj_nbr[k] & 0x7FFFFFFFu));
            if (it == manifold_map.end()) continue;
            if (manifold_min_relvel(manifolds[it->second]) < relvel_threshold) group.push_back(it->second);
        }
        if (!group.empty()) solve_restitution_group(group);
        for (uint32_t k = a0; k < a1; ++k) {
            const uint32_t nbr = adj_nbr[k] & 0x7FFFFFFFu;
            if (!visited[nbr]) { to_visit.insert(to_visit.begin(), nbr); visited[nbr] = 1; }
        }
    }
    return false;
}

// solve_restitution, restitution_solver.cpp:386-408; called first thing in solver::update, before gravity (solver.cpp:397)
void World::solve_restitution() {
    const uint32_t nb = uint32_t(bodies.size());
    if (!graph_order_set) {                                        // no graph supplied: ascending neighbour ids, pair-key order (= the device's conventions)
        std::vector<std::vector<uint32_t>> nbrs(nb);
        for (const Manifold &m : manifolds) { nbrs[m.a].push_back(m.b | 0x80000000u); nbrs[m.b].push_back(m.a | 0x80000000u); }
        for (const Hinge &h : hinges) if (h.a != h.b) { nbrs[h.a].push_back(h.b); nbrs[h.b].push_back(h.a); }
        adj_off.assign(nb + 1, 0); adj_nbr.clear();
        for (uint32_t i = 0; i < nb; ++i) {
            auto &v = nbrs[i];
            std::sort(v.begin(), v.end(), [](uint32_t x, uint32_t y) { return (x & 0x7FFFFFFFu) < (y & 0x7FFFFFFFu) || ((x & 0x7FFFFFFFu) == (y & 0x7FFFFFFFu) && x > y); });
            v.erase(std::unique(v.begin(), v.end(), [](uint32_t x, uint32_t y) { return (x & 0x7FFFFFFFu) == (y & 0x7FFFFFFFu); }), v.end());
            adj_nbr.insert(adj_nbr.end(), v.begin(), v.end());
            adj_off[i + 1] = uint32_t(adj_nbr.size());
        }
        rest_edge_order.clear();
        for (const Manifold &m : manifolds) rest_edge_order.push_back(key(m.a, m.b));
        std::sort(rest_edge_order.begin(), rest_edge_order.end());    // ties of the fastest manifold go to the smaller pair key (the device's rule)
    }
    // the tagged manifolds per island (make_contact_manifold, constraint_util.cpp:86-101: mixed restitution > EPSILON)
    std::unordered_map<uint32_t, std::vector<uint32_t>> per_island;
    std::vector<uint32_t> labels;
    for (uint64_t k : rest_edge_order) {
        auto it = manifold_map.find(k);
        if (it == manifold_map.end()) continue;
        const Manifold &m = manifolds[it->second];
        if (!(material_mix_restitution(bodies[m.a].restitution, bodies[m.b].restitution) > EPS)) continue;
        if (!bodies[m.a].awake() && !bodies[m.b].awake()) continue;             // island_view(exclude_sleeping_disabled)
        const uint32_t lab = bodies[m.a].awake() ? island[m.a] : island[m.b];
        auto &v = per_island[lab];
        if (v.empty()) labels.push_back(lab);
        v.push_back(it->second);
    }
    for (int i = 0; i < restitution_iters; ++i) {
        bool all_solved = true;
        for (uint32_t lab : labels) all_solved &= restitution_iteration(per_island[lab]);
        if (all_solved) break;
    }
    graph_order_set = false;                                       // the order belongs to one step
}

void World::solve() {
    const uint32_t nb = uint32_t(bodies.size());
    if (island.size() != bodies.size()) islands();
    if (restitution_iters > 0) solve_restitution();               // solver.cpp:397
    // apply_gravity, sys/apply_gravity.hpp:12-17
    for (Body &b : bodies) if (b.awake()) b.linvel += b.gravity * dt;

    // Group constraints per island in Gauss-Seidel order.
    std::unordered_map<uint32_t, uint32_t> isl_index;
    std::vector<IslandWork> work;
    auto island_of = [&](uint32_t a, uint32_t b) -> IslandWork & {
        uint32_t lab = bodies[a].awake() ? island[a] : island[b];
        auto it = isl_index.find(lab);
        if (it == isl_index.end()) { it = isl_index.emplace(lab, uint32_t(work.size())).first; work.emplace_back(); }
        return work[it->second];
    };
    for (uint32_t i = 0; i < nb; ++i) if (bodies[i].awake()) island_of(i, i).bodies.push_back(i);
    if (use_order) {
        for (uint32_t h : hinge_order)
            if (bodies[hinges[h].a].awake() || bodies[hinges[h].b].awake()) island_of(hinges[h].a, hinges[h].b).hinges.push_back(h);
        std::vector<char> seen(manifolds.size(), 0);
        for (size_t oi = 0; oi < manifold_order.size(); ++oi) {
            const uint64_t k = manifold_order[oi];
            auto it = manifold_map.find(k);
            if (it == manifold_map.end()) continue;
            seen[it->second] = 1;
            const Manifold &m = manifolds[it->second];
            if (!bodies[m.a].awake() && !bodies[m.b].awake()) continue;
            IslandWork &w = island_of(m.a, m.b);
            const uint32_t one = oi < point_order.size() ? point_order[oi] : 0xFFFFFFFFu;       // rows point by point (the reference's own order)
            if (one != 0xFFFFFFFFu) { if (one < m.num) w.pts.emplace_back(it->second, one); }
            else for (uint32_t p = 0; p < m.num; ++p) w.pts.emplace_back(it->second, p);
        }
        // manifolds the injected order does not name (the two sides drifted apart in a free run): natural order, at the end
        for (uint32_t mi = uint32_t(manifolds.size()); mi-- > 0;) {
            const Manifold &m = manifolds[mi];
            if (seen[mi] || m.num == 0 || (!bodies[m.a].awake() && !bodies[m.b].awake())) continue;
            IslandWork &w = island_of(m.a, m.b);
            for (uint32_t p = 0; p < m.num; ++p) w.pts.emplace_back(mi, p);
        }
    } else {
        // Natural order: constraint-type major (hinge before contact, constraints/constraint.hpp:23-34),
        // newest-first inside a type, list order inside a manifold (the reference's actual order is island.edges order, which
        // tests replay through set_point_order).
        for (uint32_t h = uint32_t(hinges.size()); h-- > 0;)
            if (bodies[hinges[h].a].awake() || bodies[hinges[h].b].awake()) island_of(hinges[h].a, hinges[h].b).hinges.push_back(h);
        for (uint32_t mi = uint32_t(manifolds.size()); mi-- > 0;) {
            const Manifold &m = manifolds[mi];
            if (m.num == 0) continue;
            if (!bodies[m.a].awake() && !bodies[m.b].awake()) continue;
            IslandWork &w = island_of(m.a, m.b);
            for (uint32_t p = 0; p < m.num; ++p) w.pts.emplace_back(mi, p);
        }
    }

    const int vi = vel_iters, pi = pos_iters;
    parallel_for(threads, work.size(), [&](size_t wi) {
        IslandWork &W = work[wi];
        std::vector<SRow> rows; std::vector<SFric> fric;
        rows.reserve(W.hinges.size() * 5 + W.pts.size());
        fric.reserve(W.pts.size());

        // ---- prepare_constraints (solver.cpp:177-215)
        for (uint32_t h : W.hinges) {                        // hinge_constraint::prepare, hinge_constraint.cpp:26-69
            Hinge &hc = hinges[h];
            const Body &A = bodies[hc.a], &B = bodies[hc.b];
            SBody sA = solver_body(A), sB = solver_body(B);
            vec3 pivotA = to_world(hc.pivot[0], A.pos, A.orn);
            vec3 pivotB = to_world(hc.pivot[1], B.pos, B.orn);
            vec3 rA = pivotA - A.pos, rB = pivotB - B.pos;
            mat3 sA_ = {{{0, -rA.z, rA.y}, {rA.z, 0, -rA.x}, {-rA.y, rA.x, 0}}};   // skew_matrix, matrix3x3.hpp:243-249
            mat3 sB_ = {{{0, -rB.z, rB.y}, {rB.z, 0, -rB.x}, {-rB.y, rB.x, 0}}};
            const vec3 I[3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
            for (int i = 0; i < 3; ++i) {
                SRow sr{}; sr.a = hc.a; sr.b = hc.b;
                sr.r.J[0] = I[i]; sr.r.J[1] = -sA_.row[i]; sr.r.J[2] = -I[i]; sr.r.J[3] = sB_.row[i];
                sr.r.lo = -SCALAR_MAX; sr.r.hi = SCALAR_MAX; sr.r.impulse = hc.imp_lin[i];
                prepare_row(sr.r, sA.inv_m, sA.inv_I, sB.inv_m, sB.inv_I, 0, scalar(0.2), 0, sA.v, sA.w, sB.v, sB.w);
                rows.push_back(sr);
            }
            vec3 p = rotate(A.orn, hc.frame[0].column(1));
            vec3 q = rotate(A.orn, hc.frame[0].column(2));
            const vec3 pq[2] = {p, q};
            for (int i = 0; i < 2; ++i) {
                SRow sr{}; sr.a = hc.a; sr.b = hc.b;
                sr.r.J[0] = vec3{0, 0, 0}; sr.r.J[1] = pq[i]; sr.r.J[2] = vec3{0, 0, 0}; sr.r.J[3] = -pq[i];
                sr.r.lo = -SCALAR_MAX; sr.r.hi = SCALAR_MAX; sr.r.impulse = hc.imp_hinge[i];
                prepare_row(sr.r, sA.inv_m, sA.inv_I, sB.inv_m, sB.inv_I, 0, scalar(0.2), 0, sA.v, sA.w, sB.v, sB.w);
                rows.push_back(sr);
            }
        }
        const size_t first_contact_row = rows.size();
        for (auto [mi, p] : W.pts) {                         // contact_constraint::prepare, contact_constraint.cpp:15-56
            Manifold &m = manifolds[mi];
            Point &cp = m.pt[p];
            const Body &A = bodies[m.a], &B = bodies[m.b];
            SBody sA = solver_body(A), sB = solver_body(B);
            SRow sr{}; sr.a = m.a; sr.b = m.b;
            SFric f{}; f.normal_row = uint32_t(rows.size());
            scalar error;
            prepare_contact(cp, dt, A.pos, A.orn, B.pos, B.orn, sA.v, sA.w, sA.inv_m, sA.inv_I, sB.v, sB.w, sB.inv_m, sB.inv_I, sr.r, error, f);
            // solver.cpp:217-236: the rows carry no restitution when the restitution solver runs
            prepare_row(sr.r, sA.inv_m, sA.inv_I, sB.inv_m, sB.inv_I, error, scalar(0.2), restitution_iters > 0 ? scalar(0) : cp.restitution, sA.v, sA.w, sB.v, sB.w);
            rows.push_back(sr); fric.push_back(f);
        }
        (void)first_contact_row;

        vec3 dummy_dv{0, 0, 0}, dummy_dw{0, 0, 0};
        auto DV = [&](uint32_t i) -> vec3 & { return bodies[i].awake() ? bodies[i].dv : dummy_dv; };
        auto DW = [&](uint32_t i) -> vec3 & { return bodies[i].awake() ? bodies[i].dw : dummy_dw; };
        auto MA = [&](uint32_t i) { return bodies[i].awake() ? bodies[i].inv_m : scalar(0); };
        mat3 zero = mat3_zero();
        auto IA = [&](uint32_t i) -> const mat3 & { return bodies[i].awake() ? bodies[i].inv_IW : zero; };

        auto apply = [&](const SRow &sr, scalar imp) {       // apply_row_impulse, constraint_row.cpp:24-32
            DV(sr.a) += MA(sr.a) * sr.r.J[0] * imp;
            DV(sr.b) += MA(sr.b) * sr.r.J[2] * imp;
            DW(sr.a) += IA(sr.a) * sr.r.J[1] * imp;
            DW(sr.b) += IA(sr.b) * sr.r.J[3] * imp;
            dummy_dv = dummy_dw = vec3{0, 0, 0};
        };
        // ---- warm start (island_solver.cpp:76-92)
        for (SRow &sr : rows) apply(sr, sr.r.impulse);
        for (SFric &f : fric) {
            const SRow &nr = rows[f.normal_row];
            warm_start_friction(f, MA(nr.a), IA(nr.a), MA(nr.b), IA(nr.b), DV(nr.a), DW(nr.a), DV(nr.b), DW(nr.b));
            dummy_dv = dummy_dw = vec3{0, 0, 0};
        }
        // ---- velocity iterations (island_solver.cpp:94-111)
        for (int it = 0; it < vi; ++it) {
            for (SRow &sr : rows) {
                scalar d = solve_row(sr.r, DV(sr.a), DW(sr.a), DV(sr.b), DW(sr.b));
                apply(sr, d);
            }
            for (SFric &f : fric) {
                const SRow &nr = rows[f.normal_row];
                solve_friction(f, nr.r.impulse, MA(nr.a), IA(nr.a), MA(nr.b), IA(nr.b), DV(nr.a), DW(nr.a), DV(nr.b), DW(nr.b));
                dummy_dv = dummy_dw = vec3{0, 0, 0};
            }
        }
        // ---- integrate_velocities (island_solver.cpp:358-376)
        for (uint32_t bi : W.bodies) {
            Body &b = bodies[bi];
            b.linvel += b.dv; b.angvel += b.dw;
            b.pos += b.linvel * dt;
            b.orn = integrate(b.orn, b.angvel, dt);
            b.dv = b.dw = vec3{0, 0, 0};
        }
        // ---- assign_applied_impulses (island_solver.cpp:232-248)
        {
            size_t ri = 0, fi = 0;
            for (uint32_t h : W.hinges) {
                Hinge &hc = hinges[h];
                for (int i = 0; i < 3; ++i) hc.imp_lin[i] = rows[ri++].r.impulse;
                for (int i = 0; i < 2; ++i) hc.imp_hinge[i] = rows[ri++].r.impulse;
            }
            for (auto [mi, p] : W.pts) {
                Point &cp = manifolds[mi].pt[p];
                cp.imp_n = rows[ri++].r.impulse;
                cp.imp_t[0] = fric[fi].impulse[0]; cp.imp_t[1] = fric[fi].impulse[1]; ++fi;
            }
        }
        // ---- position iterations (island_solver.cpp:263-353, :538-543)
        for (int it = 0; it < pi; ++it) {
            scalar max_error = 0;
            auto joints = [&] {
                scalar type_err = 0;
                for (uint32_t h : W.hinges) {                // hinge_constraint::solve_position, hinge_constraint.cpp:180-213
                    Hinge &hc = hinges[h];
                    hinge_solve_position(hc, bodies[hc.a], bodies[hc.b], type_err);
                }
                max_error = std::max(max_error, type_err);
            };
            auto contacts = [&] {
                scalar type_err = 0;
                for (auto [mi, p] : W.pts) {                 // contact_constraint::solve_position, contact_constraint.cpp:58-90
                    Manifold &m = manifolds[mi];
                    Point &cp = m.pt[p];
                    Body &A = bodies[m.a], &B = bodies[m.b];
                    contact_solve_position(cp, A, B, type_err);
                }
                max_error = std::max(max_error, type_err);
            };
            // island_solver.cpp:340 expands the constraint types as ARGUMENTS of max_variadic(...): the order in which
            // the types are swept is the compiler's argument evaluation order -- tuple order (hinge before contact) with
            // clang / MSVC, reversed with GCC.  Default: tuple order (what the device does); the GCC order is selectable
            // so that a GCC-built reference can be matched bit for bit.
            if (position_contacts_first) { contacts(); joints(); } else { joints(); contacts(); }
            if (max_error < scalar(0.005)) break;            // island_solver.cpp:350-353
        }
    });

    // update_aabbs (dynamic + kinematic) and update_inertias (dynamic): solver.cpp:453-465
    parallel_for(threads, bodies.size(), [&](size_t i) {
        Body &b = bodies[i];
        if (b.kind == BK_STATIC) return;
        if (b.sh.kind != SH_NONE) b.bb = shape_aabb(b.sh, b.pos, b.orn);
        if (b.kind == BK_DYNAMIC) { mat3 basis = to_mat3(b.orn); b.inv_IW = basis * b.inv_I * transpose(basis); }
    });
}

} // namespace ora
