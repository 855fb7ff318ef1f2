// ufo_volume.cuh -- node cube vs bounding volume: intersects(AABB node, X) of the reference's
// geometry library (geometry/collision_checks.cpp:53-356) for the eight BoundingVar types
// (geometry/types.h: AABB, Frustum, LineSegment, OBB, Plane, Point, Ray, Sphere), on the host
// and on the device.  A volume is a union: a node passes if its cube intersects any shape; a
// volume of no shapes is the whole map.
//
// Bit-exactness rules (DESIGN.md section 7 lists them):
//   * FP64 through dop::, never contracted; sums evaluated left to right as the reference writes
//     them (dot = x + y + z, squaredNorm likewise, norm = sqrt(squaredNorm), normalisation divides
//     every component, the slab test takes 1.0 / d and multiplies).
//   * std::min / std::max are (b < a) ? b : a and (a < b) ? b : a, std::clamp is
//     (v < lo) ? lo : (hi < v) ? hi : v -- not fmin / fmax, so that a NaN (the direction of a
//     zero-length segment) travels exactly as it does in the reference.
//   * intersects(AABB, Plane) tests |n.c - distance|, the frustum's classify uses n.c + distance;
//     both are reproduced as they are.
#pragma once

#include "ufo_index.cuh"

namespace ufo_b200
{
// The C ABI's ufo_b200_volume: the members of one shape as the reference stores them.
enum : uint32_t {
	kVolAABB = 0,      // centre[3], half_size[3]
	kVolFrustum = 1,   // 6 x (normal[3], distance): top, bottom, left, right, near, far
	kVolSegment = 2,   // start[3], end[3]
	kVolOBB = 3,       // centre[3], half_size[3], rotation w x y z
	kVolPlane = 4,     // normal[3], distance
	kVolPoint = 5,     // xyz
	kVolRay = 6,       // origin[3], direction[3] (normalised by the Ray constructor)
	kVolSphere = 7,    // centre[3], radius
	kVolTypes = 8,
};

struct VolRec {
	uint32_t type;
	uint32_t reserved;
	double v[24];
};

// n == 0: the whole map.  lo / hi: getMin / getMax of the one AABB of a single-box volume, the
// form kernels test inline from their parameters (set_box)
struct Volume {
	const VolRec* rec;
	uint32_t n;
	double lo[3], hi[3];
};

namespace vol
{
UFO_HD double dmax(double a, double b) { return (a < b) ? b : a; }
UFO_HD double dmin(double a, double b) { return (b < a) ? b : a; }
UFO_HD double dclamp(double v, double lo, double hi) { return (v < lo) ? lo : ((hi < v) ? hi : v); }
UFO_HD double dot(const double a[3], const double b[3])
{
	return dop::add(dop::add(dop::mul(a[0], b[0]), dop::mul(a[1], b[1])), dop::mul(a[2], b[2]));
}

// intersectsLine (collision_checks.cpp:53-80)
UFO_HD bool line(const double mn[3], const double mx[3], const double o[3], const double d[3], double t_near, double t_far)
{
	for (int i = 0; i < 3; ++i) {
		if (0 != d[i]) {
			const double rd = dop::div(1.0, d[i]);
			const double t1 = dop::mul(dop::sub(mn[i], o[i]), rd);
			const double t2 = dop::mul(dop::sub(mx[i], o[i]), rd);
			if (t1 < t2) {
				t_near = dmax(t1, t_near);
				t_far = dmin(t2, t_far);
			} else {
				t_near = dmax(t2, t_near);
				t_far = dmin(t1, t_far);
			}
			if (t_near > t_far) return false;
		} else if (mn[i] > o[i] || mx[i] < o[i]) {
			return false;
		}
	}
	return true;
}

// Quaternion::toRotMatrix (math/quaternion.h:147-188); rows of the matrix
UFO_HD void rot_matrix(const double q[4], double R[3][3])
{
	using namespace dop;
	const double w = q[0], x = q[1], y = q[2], z = q[3];
	double n2 = mul(w, w);  // the reference sums from 0.0: 0 + w*w == w*w
	n2 = add(n2, mul(x, x));
	n2 = add(n2, mul(y, y));
	n2 = add(n2, mul(z, z));
	const double n = dop::sqrt(n2);
	const double s = n > 0 ? div(2.0, mul(n, n)) : 0.0;
	const double xs = mul(x, s), ys = mul(y, s), zs = mul(z, s);
	const double wx = mul(w, xs), wy = mul(w, ys), wz = mul(w, zs);
	const double xx = mul(x, xs), xy = mul(x, ys), xz = mul(x, zs);
	const double yy = mul(y, ys), yz = mul(y, zs), zz = mul(z, zs);
	R[0][0] = sub(1.0, add(yy, zz));
	R[1][1] = sub(1.0, add(xx, zz));
	R[2][2] = sub(1.0, add(xx, yy));
	R[1][0] = add(xy, wz);
	R[0][1] = sub(xy, wz);
	R[2][0] = sub(xz, wy);
	R[0][2] = add(xz, wy);
	R[2][1] = add(yz, wx);
	R[1][2] = sub(yz, wx);
}

// getInterval(AABB, axis) (collision_checks.cpp:176-196), vertices in the reference's order
UFO_HD void interval_aabb(const double lo[3], const double hi[3], const double ax[3], double& a, double& b)
{
	for (int k = 0; k < 8; ++k) {
		// (i.x,a.y,a.z) (i.x,a.y,i.z) (i.x,i.y,a.z) (i.x,i.y,i.z) (a.x,a.y,a.z) (a.x,a.y,i.z) ...
		const double v[3] = {(k & 4) ? hi[0] : lo[0], (k & 2) ? lo[1] : hi[1], (k & 1) ? lo[2] : hi[2]};
		const double p = dot(ax, v);
		if (k == 0) {
			a = b = p;
		} else {
			a = dmin(a, p);
			b = dmax(b, p);
		}
	}
}

// getInterval(OBB, axis) (collision_checks.cpp:198-234): vertex k = C (+/-) A0*E0 (+/-) A1*E1 (+/-) A2*E2,
// signs per vertex as the reference lists them, summed left to right
UFO_HD void interval_obb(const double C[3], const double E[3], const double R[3][3], const double ax[3], double& a, double& b)
{
	// bit j set: minus for axis j
	const unsigned signs[8] = {0u, 1u, 2u, 4u, 7u, 6u, 5u, 3u};
	for (int k = 0; k < 8; ++k) {
		double v[3];
		for (int c = 0; c < 3; ++c) {
			double t = C[c];
			for (int j = 0; j < 3; ++j) {
				const double u = dop::mul(R[j][c], E[j]);
				t = ((signs[k] >> j) & 1u) ? dop::sub(t, u) : dop::add(t, u);
			}
			v[c] = t;
		}
		const double p = dot(ax, v);
		if (k == 0) {
			a = b = p;
		} else {
			a = dmin(a, p);
			b = dmax(b, p);
		}
	}
}

// intersects(AABB, OBB) (collision_checks.cpp:292-320): separating axes, the cross-product ones
// included even when they are zero
UFO_HD bool obb(const double lo[3], const double hi[3], const double* s)
{
	double R[3][3];
	rot_matrix(s + 6, R);
	for (int i = 0; i < 15; ++i) {
		double ax[3];
		if (i < 3) {
			ax[0] = i == 0 ? 1.0 : 0.0;
			ax[1] = i == 1 ? 1.0 : 0.0;
			ax[2] = i == 2 ? 1.0 : 0.0;
		} else if (i < 6) {
			ax[0] = R[i - 3][0];
			ax[1] = R[i - 3][1];
			ax[2] = R[i - 3][2];
		} else {
			// cross(e_k, R_j) with k = (i - 6) / 3, j = (i - 6) % 3
			const int k = (i - 6) / 3, j = (i - 6) % 3;
			const double f[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
			const double* g = R[j];
			ax[0] = dop::sub(dop::mul(f[1], g[2]), dop::mul(f[2], g[1]));
			ax[1] = dop::sub(dop::mul(f[2], g[0]), dop::mul(f[0], g[2]));
			ax[2] = dop::sub(dop::mul(f[0], g[1]), dop::mul(f[1], g[0]));
		}
		double a0, a1, b0, b1;
		interval_aabb(lo, hi, ax, a0, a1);
		interval_obb(s, s + 3, R, ax, b0, b1);
		if (!((b0 <= a1) && (a0 <= b1))) return false;
	}
	return true;
}

// intersects(AABB, AABB) (collision_checks.cpp:256-264); the shape's min / max are getMin / getMax
UFO_HD bool aabb(const double lo[3], const double hi[3], const double* s)
{
	for (int k = 0; k < 3; ++k) {
		const double mn = dop::sub(s[k], s[3 + k]), mx = dop::add(s[k], s[3 + k]);
		if (!(lo[k] <= mx) || !(mn <= hi[k])) return false;
	}
	return true;
}

// classify(AABB, Plane) (collision_checks.cpp:145-157) < 0 for any plane: outside
UFO_HD bool frustum(const double c[3], const double hs[3], const double* s)
{
	for (int p = 0; p < 6; ++p) {
		const double* n = s + 4 * p;
		const double r = dop::add(dop::add(fabs(dop::mul(hs[0], n[0])), fabs(dop::mul(hs[1], n[1]))), fabs(dop::mul(hs[2], n[2])));
		const double d = dop::add(dot(n, c), n[3]);
		double side;
		if (fabs(d) < r) side = 0.0;
		else if (d < 0.0) side = dop::add(d, r);
		else side = dop::sub(d, r);
		if (side < 0) return false;
	}
	return true;
}
}  // namespace vol

// intersects(AABB(c, hs), shape); false for an unknown type (the C ABI rejects those up front)
UFO_HD bool shape_hits(const VolRec& r, const double c[3], const double hs[3])
{
	const double* s = r.v;
	const double lo[3] = {dop::sub(c[0], hs[0]), dop::sub(c[1], hs[1]), dop::sub(c[2], hs[2])};
	const double hi[3] = {dop::add(c[0], hs[0]), dop::add(c[1], hs[1]), dop::add(c[2], hs[2])};
	switch (r.type) {
		case kVolAABB:
			return vol::aabb(lo, hi, s);
		case kVolFrustum:
			return vol::frustum(c, hs, s);
		case kVolSegment: {
			double d[3] = {dop::sub(s[3], s[0]), dop::sub(s[4], s[1]), dop::sub(s[5], s[2])};
			const double len = dop::sqrt(vol::dot(d, d));
			d[0] = dop::div(d[0], len);
			d[1] = dop::div(d[1], len);
			d[2] = dop::div(d[2], len);
			return vol::line(lo, hi, s, d, 0.0, len);
		}
		case kVolOBB:
			return vol::obb(lo, hi, s);
		case kVolPlane: {
			const double p_len = dop::add(dop::add(dop::mul(hs[0], fabs(s[0])), dop::mul(hs[1], fabs(s[1]))), dop::mul(hs[2], fabs(s[2])));
			const double dist = dop::sub(vol::dot(s, c), s[3]);
			return fabs(dist) <= p_len;
		}
		case kVolPoint:
			return !(s[0] < lo[0] || s[1] < lo[1] || s[2] < lo[2] || s[0] > hi[0] || s[1] > hi[1] || s[2] > hi[2]);
		case kVolRay:
			return vol::line(lo, hi, s, s + 3, 0.0, INFINITY);
		case kVolSphere: {
			double q[3];
			for (int k = 0; k < 3; ++k) q[k] = dop::sub(s[k], vol::dclamp(s[k], lo[k], hi[k]));
			return vol::dot(q, q) < dop::mul(s[3], s[3]);
		}
		default:
			return false;
	}
}

#if defined(__CUDACC__)
__host__ __device__ __noinline__
#else
inline
#endif
bool volume_hits_any(const VolRec* rec, uint32_t n, const double c[3], const double hs[3])
{
	for (uint32_t i = 0; i < n; ++i)
		if (shape_hits(rec[i], c, hs)) return true;
	return false;
}

// The cube of centre c, half size hs is inside the filter of v (as one link of the chain from the
// root: the caller tests every cube on a node's path).  GENERAL = false: v is empty or one AABB whose
// min / max sit in v.lo / v.hi (the box entry points) and the test is inline on kernel parameters;
// the general form calls the out-of-line volume_hits_any, whose register needs (the OBB's separating
// axes) a kernel inherits.
template <bool GENERAL>
UFO_HD bool vol_hits_t(const Volume& v, const double c[3], double hs)
{
	if (v.n == 0) return true;
	if constexpr (GENERAL) {
		const double h[3] = {hs, hs, hs};
		return volume_hits_any(v.rec, v.n, c, h);
	} else {
		for (int k = 0; k < 3; ++k) {
			const double mn = dop::sub(c[k], hs), mx = dop::add(c[k], hs);
			if (!(mn <= v.hi[k]) || !(v.lo[k] <= mx)) return false;
		}
		return true;
	}
}

UFO_HD bool vol_hits(const Volume& v, const double c[3], double hs) { return vol_hits_t<true>(v, c, hs); }

// Host side: whether kernels need the general form of the test for v (host records); otherwise
// fills v.lo / v.hi for the inline one (the same doubles getMin / getMax give).
inline bool volume_is_general(Volume& v)
{
	if (v.n > 1 || (v.n == 1 && v.rec[0].type != kVolAABB)) return true;
	for (int k = 0; k < 3; ++k) {
		v.lo[k] = v.n ? v.rec[0].v[k] - v.rec[0].v[3 + k] : 0.0;
		v.hi[k] = v.n ? v.rec[0].v[k] + v.rec[0].v[3 + k] : 0.0;
	}
	return false;
}
}  // namespace ufo_b200
