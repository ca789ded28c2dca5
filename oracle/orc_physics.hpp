// ORACLE (test infrastructure, NOT product code): collision queries + kinematic character controller.
//
// The controller state machine is restated line by line from
//   src/libs/env/src/kinematic_character_controller.cpp:156-221 (recoverFromPenetration), :223-304 (stepUp),
//   :313-329 (updateTargetPositionBasedOnCollision), :337-393 (stepForwardAndStrafe), :400-442 (stepDown),
//   :509-517 (warp), :519-526 (preStep), :528-602 (playerStep), :625-644 (jump), :679-682 (onGround),
//   :753-792 (setAcceleration); constants kinematic_character_controller.hpp:155-177, agent.cpp:52-59.
//
// PINNED: the state machine below against the reference's own kinematic_character_controller.cpp, compiled in place on the Bullet
// stand-in of ref_shim/mini_bullet and run beside this file tick by tick (tests/test_ref_shim.py).
// The collision arithmetic underneath (btGhostObject::convexSweepTest, contact manifolds) lives in
// Bullet 2.89, which is NOT vendored under /root/reference and not installed: PARITY UNPINNED for that part.
// It is replaced by an exact analytic definition with the same contract:
//   * sweep(upright capsule, from->to) vs a box = first t in [0,1] at which the capsule PENETRATES the
//     box by `allowedCcdPenetration` (Bullet world default 0.04) -- i.e. a ray against the box grown by the
//     capsule's segment and rounded by (radius - 0.04).  This is the fixed point Bullet's conservative
//     advancement (btContinuousConvexCollision, stop when distance+allowedPenetration <= 0.001) converges to.
//   * an already-penetrating start reports fraction 0 only when moving into the surface, else no hit.
//   * recoverFromPenetration uses the exact signed capsule/box distance; first collider (in list order)
//     deeper than maxPenetrationDepth (0.041) pushes the capsule out by its full depth.
//   * every collider of the env is a candidate (Bullet restricts to broadphase-overlapping pairs).
#pragma once
#include <vector>

#include "orc_math.hpp"

namespace orc {

constexpr float kCapsuleRadius = 0.33f;          // agent.cpp:53
constexpr float kCapsuleHalfHeight = 1.05f / 2;  // agent.cpp:52 (btCapsuleShape height = cylinder length)
constexpr float kAllowedCcdPenetration = 0.04f;  // btDispatcherInfo default (upstream)
constexpr float kSimdEpsilon = 1.1920929e-07f;   // SIMD_EPSILON == FLT_EPSILON

struct Collider {
    int kind = 0;  // 0 = axis-aligned box, 1 = upright capsule (another agent)
    Vec3 c;        // centre
    Vec3 h;        // box half extents (kind 0)
    bool enabled = true;  // !CF_NO_CONTACT_RESPONSE
    // boxes rotated about Y (the hexagonal mazes' walls): the box's local x axis in world space is (ax, 0, az), its local z
    // axis (-az, 0, ax).  The agent capsule is upright, hence symmetric about Y: queries run in the box's frame.
    bool rotated = false;
    float ax = 1.0f, az = 0.0f;
    Vec3 toLocal(Vec3 p) const { return rotated ? Vec3{p.x * ax + p.z * az, p.y, p.x * -az + p.z * ax} : p; }
    Vec3 toWorld(Vec3 n) const { return rotated ? Vec3{n.x * ax + n.z * -az, n.y, n.x * az + n.z * ax} : n; }
};

struct SweepHit {
    bool hit = false;
    float fraction = 1.0f;
    Vec3 normal;
    int index = -1;
    int feature = -1;  // of the winner: the box feature numbered as the device numbers it (0..2 faces, 3..14 edges, 15..22 corners), 0 for a capsule
};

// signed distance helper: point o (relative to box centre) vs box half H.  Returns distance (>=0 outside,
// negative = -(min face distance) inside) and the outward unit normal.
inline float pointBoxDistance(Vec3 o, Vec3 H, Vec3 &n) {
    Vec3 q{fabsf(o.x) - H.x, fabsf(o.y) - H.y, fabsf(o.z) - H.z};
    if (q.x <= 0.0f && q.y <= 0.0f && q.z <= 0.0f) {
        // inside: least-penetration axis (ties: x, then y, then z)
        int ax = 0;
        float best = q.x;
        if (q.y > best) { best = q.y; ax = 1; }
        if (q.z > best) { best = q.z; ax = 2; }
        n = {0, 0, 0};
        n[ax] = o[ax] < 0.0f ? -1.0f : 1.0f;
        return best;
    }
    Vec3 e{q.x > 0.0f ? q.x : 0.0f, q.y > 0.0f ? q.y : 0.0f, q.z > 0.0f ? q.z : 0.0f};
    float d = sqrtf(e.x * e.x + e.y * e.y + e.z * e.z);
    n = {o.x < 0.0f ? -e.x : e.x, o.y < 0.0f ? -e.y : e.y, o.z < 0.0f ? -e.z : e.z};
    n = n * (1.0f / d);
    return d;
}

// Ray o + t d, t in [0,1], against the rounded box {p : dist(p, box(H)) <= rho}.  Returns true and the first
// entry (t, outward normal, and the feature that gave it, 0 for a start inside).  Start inside => t = 0 iff moving into the surface.
inline bool rayRoundedBox(Vec3 o, Vec3 d, Vec3 H, float rho, float &tOut, Vec3 &nOut, int *fOut = nullptr) {
    Vec3 n0;
    const float d0 = pointBoxDistance(o, H, n0);
    if (d0 - rho <= 0.0f) {
        if (dot(d, n0) < -kSimdEpsilon) { tOut = 0.0f; nOut = n0; if (fOut) *fOut = 0; return true; }
        return false;
    }
    float best = 2.0f;
    Vec3 bestN;
    int bestF = -1;
    // 6 faces
    for (int i = 0; i < 3; ++i) {
        if (d[i] == 0.0f) continue;
        const float s = d[i] < 0.0f ? 1.0f : -1.0f;  // face whose outward normal opposes the motion
        const float t = (s * (H[i] + rho) - o[i]) / d[i];
        if (t < 0.0f || t > 1.0f || t >= best) continue;
        const int j = (i + 1) % 3, k = (i + 2) % 3;
        const float qj = o[j] + t * d[j], qk = o[k] + t * d[k];
        if (fabsf(qj) <= H[j] && fabsf(qk) <= H[k]) { best = t; bestN = {0, 0, 0}; bestN[i] = s; bestF = i; }
    }
    // 12 edges: axis k free, signs on i and j
    for (int k = 0; k < 3; ++k) {
        const int i = (k + 1) % 3, j = (k + 2) % 3;
        const float a = d[i] * d[i] + d[j] * d[j];
        if (a == 0.0f) continue;
        for (int si = -1; si <= 1; si += 2)
            for (int sj = -1; sj <= 1; sj += 2) {
                const float oi = o[i] - si * H[i], oj = o[j] - sj * H[j];
                const float b = oi * d[i] + oj * d[j];
                const float c = oi * oi + oj * oj - rho * rho;
                const float disc = b * b - a * c;
                if (disc < 0.0f) continue;
                const float t = (-b - sqrtf(disc)) / a;
                if (t < 0.0f || t > 1.0f || t >= best) continue;
                const float qi = oi + t * d[i], qj = oj + t * d[j], qk = o[k] + t * d[k];
                if (si * qi >= 0.0f && sj * qj >= 0.0f && fabsf(qk) <= H[k]) {
                    best = t;
                    bestN = {0, 0, 0};
                    bestN[i] = qi / rho;
                    bestN[j] = qj / rho;
                    bestF = 3 + 4 * k + (si > 0 ? 2 : 0) + (sj > 0 ? 1 : 0);
                }
            }
    }
    // 8 corners
    {
        const float a = dot(d, d);
        if (a != 0.0f)
            for (int sx = -1; sx <= 1; sx += 2)
                for (int sy = -1; sy <= 1; sy += 2)
                    for (int sz = -1; sz <= 1; sz += 2) {
                        const Vec3 oc{o.x - sx * H.x, o.y - sy * H.y, o.z - sz * H.z};
                        const float b = dot(oc, d);
                        const float c = dot(oc, oc) - rho * rho;
                        const float disc = b * b - a * c;
                        if (disc < 0.0f) continue;
                        const float t = (-b - sqrtf(disc)) / a;
                        if (t < 0.0f || t > 1.0f || t >= best) continue;
                        const Vec3 q = oc + d * t;
                        if (sx * q.x >= 0.0f && sy * q.y >= 0.0f && sz * q.z >= 0.0f) {
                            best = t; bestN = q * (1.0f / rho);
                            bestF = 15 + (sx > 0 ? 4 : 0) + (sy > 0 ? 2 : 0) + (sz > 0 ? 1 : 0);
                        }
                    }
    }
    if (best > 1.0f) return false;
    tOut = best;
    nOut = bestN;
    if (fOut) *fOut = bestF;
    return true;
}

// upright capsule (this agent) vs upright capsule (other agent): ray against a capsule of half-length 2*hh
// and radius R = 2r - pen.
inline float pointSegDistance(Vec3 o, float L, Vec3 &n) {
    float cy = o.y < -L ? -L : (o.y > L ? L : o.y);
    Vec3 e{o.x, o.y - cy, o.z};
    float d = length(e);
    if (d > 0.0f) n = e * (1.0f / d); else n = {1, 0, 0};
    return d;
}
inline bool rayCapsule(Vec3 o, Vec3 d, float L, float R, float &tOut, Vec3 &nOut) {
    Vec3 n0;
    const float d0 = pointSegDistance(o, L, n0);
    if (d0 - R <= 0.0f) {
        if (dot(d, n0) < -kSimdEpsilon) { tOut = 0.0f; nOut = n0; return true; }
        return false;
    }
    float best = 2.0f;
    Vec3 bestN;
    {
        const float a = d.x * d.x + d.z * d.z;
        if (a != 0.0f) {
            const float b = o.x * d.x + o.z * d.z, c = o.x * o.x + o.z * o.z - R * R;
            const float disc = b * b - a * c;
            if (disc >= 0.0f) {
                const float t = (-b - sqrtf(disc)) / a;
                if (t >= 0.0f && t <= 1.0f) {
                    const float qy = o.y + t * d.y;
                    if (fabsf(qy) <= L) { best = t; bestN = {(o.x + t * d.x) / R, 0.0f, (o.z + t * d.z) / R}; }
                }
            }
        }
    }
    const float a = dot(d, d);
    if (a != 0.0f)
        for (int s = -1; s <= 1; s += 2) {
            const Vec3 oc{o.x, o.y - s * L, o.z};
            const float b = dot(oc, d), c = dot(oc, oc) - R * R;
            const float disc = b * b - a * c;
            if (disc < 0.0f) continue;
            const float t = (-b - sqrtf(disc)) / a;
            if (t < 0.0f || t > 1.0f || t >= best) continue;
            const Vec3 q = oc + d * t;
            if (s * q.y >= 0.0f) { best = t; bestN = q * (1.0f / R); }
        }
    if (best > 1.0f) return false;
    tOut = best;
    nOut = bestN;
    return true;
}

// broadphase, the role btRayAabb plays in btGhostObject::convexSweepTest: skip colliders whose bounds grown by the capsule
// extents (full radius: 0.04 more than the narrow phase needs) miss the sweep segment's box
inline bool sweepBroadphaseMiss(const Collider &c, Vec3 from, Vec3 to) {
    Vec3 ext = c.kind == 0 ? Vec3{c.h.x + kCapsuleRadius, c.h.y + (kCapsuleHalfHeight + kCapsuleRadius), c.h.z + kCapsuleRadius}
                           : Vec3{2.0f * kCapsuleRadius, 2.0f * (kCapsuleHalfHeight + kCapsuleRadius), 2.0f * kCapsuleRadius};
    if (c.kind == 0 && c.rotated) {  // bounds of the rotated box
        ext.x = (fabsf(c.ax) * c.h.x + fabsf(c.az) * c.h.z) + kCapsuleRadius;
        ext.z = (fabsf(c.az) * c.h.x + fabsf(c.ax) * c.h.z) + kCapsuleRadius;
    }
    bool miss = false;
    for (int ax = 0; ax < 3; ++ax) {
        const float lo = from[ax] < to[ax] ? from[ax] : to[ax], hi = from[ax] < to[ax] ? to[ax] : from[ax];
        if (hi < c.c[ax] - ext[ax] || lo > c.c[ax] + ext[ax]) miss = true;
    }
    return miss;
}
// narrow phase of one sweep: the agent capsule from `from` along d against one collider (see the header comment)
inline bool sweepNarrow(const Collider &c, Vec3 from, Vec3 d, float &t, Vec3 &n, int *f = nullptr) {
    if (c.kind == 0) {
        const bool hit = rayRoundedBox(c.toLocal(from - c.c), c.toLocal(d), Vec3{c.h.x, c.h.y + kCapsuleHalfHeight, c.h.z}, kCapsuleRadius - kAllowedCcdPenetration, t, n, f);
        if (hit) n = c.toWorld(n);
        return hit;
    }
    if (f) *f = 0;
    return rayCapsule(from - c.c, d, 2.0f * kCapsuleHalfHeight, 2.0f * kCapsuleRadius - kAllowedCcdPenetration, t, n);
}

// KinematicClosestNotMeConvexResultCallback (kinematic_character_controller.cpp:53-96) over all colliders.
inline SweepHit convexSweep(const std::vector<Collider> &cols, int self, Vec3 from, Vec3 to, Vec3 filterDir, float minSlopeDot) {
    SweepHit res;
    const Vec3 d = to - from;
    for (int i = 0; i < int(cols.size()); ++i) {
        const Collider &c = cols[i];
        if (i == self || !c.enabled) continue;
        if (sweepBroadphaseMiss(c, from, to)) continue;
        float t;
        Vec3 n;
        int f;
        if (!sweepNarrow(c, from, d, t, n, &f)) continue;
        if (!(t < res.fraction)) continue;             // btCollisionWorld: castResult.m_fraction < m_closestHitFraction
        if (dot(filterDir, n) < minSlopeDot) continue;  // slope filter
        res.hit = true;
        res.fraction = t;
        res.normal = n;
        res.index = i;
        res.feature = f;
    }
    return res;
}

// signed capsule-vs-collider distance (negative = penetration depth) and outward normal
inline float capsuleDistance(const Collider &c, Vec3 p, Vec3 &n) {
    if (c.kind == 0) {
        const float d = pointBoxDistance(c.toLocal(p - c.c), Vec3{c.h.x, c.h.y + kCapsuleHalfHeight, c.h.z}, n) - kCapsuleRadius;
        n = c.toWorld(n);
        return d;
    }
    return pointSegDistance(p - c.c, 2.0f * kCapsuleHalfHeight, n) - 2.0f * kCapsuleRadius;
}

struct KCC {
    // ghost object
    Vec3 pos;                    // ghost origin
    Mat3 basis = mat3Identity();  // ghost basis (yaw)
    // controller state (ctor values, kinematic_character_controller.cpp:122-151)
    Vec3 horizontalVelocity;
    float verticalVelocity = 0, verticalOffset = 0;
    float fallSpeed = 55.0f, jumpSpeed = 10.0f;
    float stepHeight = 0.2f;
    float gravity = 1.4f * 9.8f;
    float maxSlopeCosine = crcos(45.0f * (3.14159265358979323846f / 180.0f));  // btCos(btRadians(45))
    float maxPenetrationDepth = 0.041f;
    float currentStepOffset = 0;
    bool wasOnGround = false, wasJumping = false;
    Vec3 jumpAxis{0, 1, 0};
    Vec3 currentPosition, targetPosition;
    float maxHorizontalSpeed = 4.5f, maxAirSpeed = 1.0f, normalDeceleration = 15.0f;
    float maxAcceleration = 35.0f + 15.0f, maxAirAcceleration = 3.0f, exceedingSpeedLimitDeceleration = (35.0f + 15.0f) * 2;

    bool onGround() const { return (fabsf(verticalVelocity) < kSimdEpsilon) && (fabsf(verticalOffset) < kSimdEpsilon); }

    void setAcceleration(Vec3 acc, float dt) {  // :753-792
        const bool isOnGround = onGround();
        const float accelerationMagnitude = length(acc);
        const float currMaxAcceleration = isOnGround ? maxAcceleration : maxAirAcceleration;
        // btVector3::fuzzyZero: length2() < SIMD_EPSILON*SIMD_EPSILON
        if (!(length2(acc) < kSimdEpsilon * kSimdEpsilon)) acc *= currMaxAcceleration / accelerationMagnitude;
        if (isOnGround) {
            horizontalVelocity += acc * dt;
            const float currHorizontalSpeed = length(horizontalVelocity);
            if (currHorizontalSpeed > maxHorizontalSpeed) {
                const float dv = exceedingSpeedLimitDeceleration * dt;
                if (currHorizontalSpeed - dv > maxHorizontalSpeed) horizontalVelocity *= (currHorizontalSpeed - dv) / currHorizontalSpeed;
                else horizontalVelocity *= maxHorizontalSpeed / currHorizontalSpeed;
            }
        } else {
            const float currHorizontalSpeed = length(horizontalVelocity);
            const Vec3 newHorizontalVelocity = horizontalVelocity + acc * dt;
            const float newHorizontalSpeed = length(newHorizontalVelocity);
            if (newHorizontalSpeed <= maxAirSpeed || newHorizontalSpeed < currHorizontalSpeed) horizontalVelocity = newHorizontalVelocity;
        }
    }

    void jump(Vec3 v) {  // :625-644 (v = (0,6.2,0), agent.cpp:160)
        jumpSpeed = length(v);
        verticalVelocity = jumpSpeed;
        wasJumping = true;
        jumpAxis = btNormalized(v);
    }

    void warp(Vec3 origin) {  // :509-517  (rotation reset to identity)
        basis = mat3Identity();
        pos = origin;
        horizontalVelocity = {0, 0, 0};
        verticalVelocity = 0;
    }

    bool recoverFromPenetration(const std::vector<Collider> &cols, int self, int *index = nullptr) {  // :156-221; index: the collider that pushed
        bool penetration = false;
        currentPosition = pos;
        for (int i = 0; i < int(cols.size()) && !penetration; ++i) {
            if (i == self || !cols[i].enabled) continue;
            Vec3 n;
            const float dist = capsuleDistance(cols[i], currentPosition, n);
            if (dist < -maxPenetrationDepth) {
                currentPosition += n * (-dist);
                penetration = true;
                if (index) *index = i;
            }
        }
        pos = currentPosition;
        return penetration;
    }

    void stepUp(const std::vector<Collider> &cols, int self) {  // :223-304
        float stepH = 0.0f;
        if (verticalVelocity < 0.0f) stepH = stepHeight;
        const Vec3 start = currentPosition;
        const Vec3 up{0, 1, 0};
        targetPosition = currentPosition + up * stepH + jumpAxis * (verticalOffset > 0.f ? verticalOffset : 0.f);
        currentPosition = targetPosition;
        SweepHit cb = convexSweep(cols, self, start, targetPosition, -up, maxSlopeCosine);
        if (cb.hit) {
            if (dot(cb.normal, up) > 0.0f) {
                currentStepOffset = stepH * cb.fraction;
                // setInterpolate3(cur, target, fraction) with cur == target
                const float s = 1.0f - cb.fraction;
                currentPosition = {s * currentPosition.x + cb.fraction * targetPosition.x, s * currentPosition.y + cb.fraction * targetPosition.y,
                                   s * currentPosition.z + cb.fraction * targetPosition.z};
            }
            pos = currentPosition;
            int numPenetrationLoops = 0;
            while (recoverFromPenetration(cols, self)) {
                numPenetrationLoops++;
                if (numPenetrationLoops > 4) break;
            }
            targetPosition = pos;
            currentPosition = targetPosition;
            if (verticalOffset > 0) {
                verticalOffset = 0.0f;
                verticalVelocity = 0.0f;
                currentStepOffset = stepHeight;
            }
        } else {
            currentStepOffset = stepH;
            currentPosition = targetPosition;
        }
    }

    void updateTargetPositionBasedOnCollision(Vec3 hitNormal, float fraction) {  // :313-329
        Vec3 movementDirection = targetPosition - currentPosition;
        const float movementLength = length(movementDirection);
        if (movementLength > kSimdEpsilon) {
            movementDirection = btNormalized(movementDirection);
            const Vec3 parallelDir = hitNormal * dot(movementDirection, hitNormal);
            const Vec3 perpindicularDir = movementDirection - parallelDir;
            targetPosition = currentPosition;
            targetPosition += perpindicularDir * movementLength;
            targetPosition += parallelDir * (movementLength * fraction);
        }
    }

    void stepForwardAndStrafe(const std::vector<Collider> &cols, int self, Vec3 hVel, float dt) {  // :337-393
        targetPosition = currentPosition + hVel * dt;
        int maxIter = 10;
        while (maxIter-- > 0) {
            const Vec3 sweepDirNegative = currentPosition - targetPosition;
            SweepHit cb;
            const bool same = currentPosition.x == targetPosition.x && currentPosition.y == targetPosition.y && currentPosition.z == targetPosition.z;
            if (!same) cb = convexSweep(cols, self, currentPosition, targetPosition, sweepDirNegative, 0.0f);
            if (cb.hit) {
                updateTargetPositionBasedOnCollision(cb.normal, cb.fraction);
                Vec3 currentDir = targetPosition - currentPosition;
                const float distance2 = length2(currentDir);
                if (distance2 > 0.0001f) {
                    currentDir = btNormalized(currentDir);
                    if (dot(currentDir, hVel) <= 0.0f) { targetPosition = currentPosition; break; }
                } else { targetPosition = currentPosition; break; }
            } else break;
        }
        currentPosition = targetPosition;
    }

    void stepDown(const std::vector<Collider> &cols, int self, float dt) {  // :400-442
        float downVelocity = (verticalVelocity < 0.f ? -verticalVelocity : 0.f);
        if (downVelocity > 0.0f && downVelocity > fallSpeed && (wasOnGround || !wasJumping)) downVelocity = fallSpeed;
        const Vec3 up{0, 1, 0};
        const Vec3 step_drop = up * (currentStepOffset + downVelocity * dt);
        targetPosition -= step_drop;
        SweepHit cb = convexSweep(cols, self, currentPosition, targetPosition, up, maxSlopeCosine);
        if (cb.hit) {
            const float s = 1.0f - cb.fraction;
            currentPosition = {s * currentPosition.x + cb.fraction * targetPosition.x, s * currentPosition.y + cb.fraction * targetPosition.y,
                               s * currentPosition.z + cb.fraction * targetPosition.z};
            verticalVelocity = 0.0f;
            verticalOffset = 0.0f;
            wasJumping = false;
        } else {
            currentPosition = targetPosition;
        }
    }

    void playerStep(const std::vector<Collider> &cols, int self, float dt) {  // preStep :519-526 + playerStep :528-602
        currentPosition = pos;
        targetPosition = currentPosition;
        const Vec3 originalPosition = currentPosition;
        wasOnGround = onGround();
        verticalVelocity -= gravity * dt;
        if (verticalVelocity > 0.0f && verticalVelocity > jumpSpeed) verticalVelocity = jumpSpeed;
        if (verticalVelocity < 0.0f && fabsf(verticalVelocity) > fabsf(fallSpeed)) verticalVelocity = -fabsf(fallSpeed);
        verticalOffset = verticalVelocity * dt;
        stepUp(cols, self);
        stepForwardAndStrafe(cols, self, horizontalVelocity, dt);
        stepDown(cols, self, dt);
        pos = currentPosition;
        horizontalVelocity = (currentPosition - originalPosition) * (1.0f / dt);  // btVector3 operator/(v, s) == v * (1/s)
        horizontalVelocity.y = 0;
        int numPenetrationLoops = 0;
        while (recoverFromPenetration(cols, self)) {
            numPenetrationLoops++;
            if (numPenetrationLoops > 4) break;
        }
        const float currHorizontalSpeed = length(horizontalVelocity);
        if (onGround()) {
            if (currHorizontalSpeed - normalDeceleration * dt < 0) horizontalVelocity = {0, 0, 0};
            else horizontalVelocity *= (currHorizontalSpeed - normalDeceleration * dt) / currHorizontalSpeed;
        }
    }
};

}  // namespace orc
