// oracle/ref_volumes.cpp -- TEST INFRASTRUCTURE ONLY.
//
// The reference shim (ref_harness.cpp, included whole) plus the reference's bounding-volume forms
// of writeData / write / readData / setValueVolume / beginLeaves, its intersects(AABB, X) and the
// geometry constructors whose arithmetic decides a shape's doubles, built into
// oracle/_ref/libufo_ref_volumes.so by oracle/volumes.mk from the UNMODIFIED reference sources.
// Every ufo_ref_* entry point of libufo_ref.so is exported as well (tests/volumes_lib.py).  Shapes
// cross the boundary as the C ABI's ufo_b200_volume records: type in BoundingVar order, members in
// v as the reference stores them.  Nothing in the product path may link or load it.
#include "ref_harness.cpp"

#include <ufo/geometry/bounding_volume.h>

namespace
{
namespace geo = ufo::geometry;

struct VolumeRecord {
	uint32_t type;
	uint32_t reserved;
	double v[24];
};

geo::Point pt(const double* p) { return geo::Point(p[0], p[1], p[2]); }

// member by member, without the constructors that normalise or convert
geo::BoundingVar to_var(const VolumeRecord& r)
{
	const double* v = r.v;
	switch (r.type) {
		case 0: {
			geo::AABB a;
			a.center = pt(v);
			a.half_size = pt(v + 3);
			return a;
		}
		case 1: {
			geo::Frustum f;
			for (int i = 0; i < 6; ++i) f.planes[i] = geo::Plane(pt(v + 4 * i), v[4 * i + 3]);
			return f;
		}
		case 2:
			return geo::LineSegment(pt(v), pt(v + 3));
		case 3:
			return geo::OBB(pt(v), pt(v + 3), ufo::math::Quaternion(v[6], v[7], v[8], v[9]));
		case 4:
			return geo::Plane(pt(v), v[3]);
		case 5:
			return pt(v);
		case 6: {
			geo::Ray ray;
			ray.origin = pt(v);
			ray.direction = pt(v + 3);
			return ray;
		}
		default:
			return geo::Sphere(pt(v), v[3]);
	}
}

geo::BoundingVolume to_volume(const VolumeRecord* recs, size_t n)
{
	geo::BoundingVolume bv;
	for (size_t i = 0; i < n; ++i) bv.add(to_var(recs[i]));
	return bv;
}

size_t copy_out(const std::string& str, uint8_t* buf, size_t cap)
{
	if (buf && str.size() <= cap) std::memcpy(buf, str.data(), str.size());
	return str.size();
}

void put(const geo::Point& p, double* out)
{
	out[0] = p[0];
	out[1] = p[1];
	out[2] = p[2];
}
}  // namespace

extern "C" {

// BoundingVolume::intersects(AABB(centre, half_size)) (bounding_volume.cpp:46-56 ->
// intersects(AABB, X), collision_checks.cpp) for n cubes; an empty volume passes everything, as the
// recursions treat it.
void ufo_ref_vol_intersects(const VolumeRecord* recs, size_t n_recs, const double* centres, const double* half_sizes,
                            size_t n, uint8_t* out)
{
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	for (size_t i = 0; i < n; ++i) {
		geo::AABB a;
		a.center = pt(centres + 3 * i);
		a.half_size = pt(half_sizes + 3 * i);
		out[i] = (bv.empty() || bv.intersects(a)) ? 1 : 0;
	}
}

// Octree::writeData(stream, BoundingVolume, compress = false, min_depth) (octree.h:885-917)
size_t ufo_ref_write_data_bv(void* h, const VolumeRecord* recs, size_t n_recs, unsigned min_depth, uint8_t* buf,
                             size_t cap)
{
	RefMap* m = static_cast<RefMap*>(h);
	std::stringstream ss(std::ios_base::in | std::ios_base::out | std::ios_base::binary);
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	withMap(m, [&](auto& map) { return map.writeData(ss, bv, false, min_depth); });
	return copy_out(ss.str(), buf, cap);
}

// Octree::write(stream, BoundingVolume, compress, min_depth, acceleration, level) (octree.h:833-864):
// whatever it wrote (it reports false, header written, when no node intersects the volume)
size_t ufo_ref_write_bv(void* h, const VolumeRecord* recs, size_t n_recs, unsigned min_depth, int compress,
                        int acceleration, int level, uint8_t* buf, size_t cap)
{
	RefMap* m = static_cast<RefMap*>(h);
	std::stringstream ss(std::ios_base::in | std::ios_base::out | std::ios_base::binary);
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	withMap(m, [&](auto& map) { return map.write(ss, bv, compress != 0, min_depth, acceleration, level); });
	return copy_out(ss.str(), buf, cap);
}

// Octree::readData(stream, BoundingVolume, resolution, depth_levels) (octree.h:751-774)
int ufo_ref_read_data_bv(void* h, const VolumeRecord* recs, size_t n_recs, const uint8_t* buf, size_t size)
{
	RefMap* m = static_cast<RefMap*>(h);
	std::stringstream ss(std::string(reinterpret_cast<const char*>(buf), size),
	                     std::ios_base::in | std::ios_base::out | std::ios_base::binary);
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	return withMap(m, [&](auto& map) { return map.readData(ss, bv, map.getResolution(), map.getTreeDepthLevels()); })
	           ? 1
	           : 0;
}

// setValueVolume(BoundingVar, occupancy probability, min_depth) (occupancy_map_base.h:492-518)
void ufo_ref_set_value_volume_bv(void* h, const VolumeRecord* rec, double occupancy, unsigned min_depth)
{
	RefMap* m = static_cast<RefMap*>(h);
	const geo::BoundingVar var = to_var(*rec);
	withMap(m, [&](auto& map) { map.setValueVolume(var, occupancy, min_depth); });
}

// beginLeaves(BoundingVolume, occupied, free, unknown, contains = false, min_depth)
// (occupancy_map_base.h:155-163)
size_t ufo_ref_leaves_bv(void* h, int occupied, int free_space, int unknown, const VolumeRecord* recs, size_t n_recs,
                         unsigned min_depth, uint64_t* codes, uint32_t* depths, float* occ, size_t cap)
{
	RefMap* m = static_cast<RefMap*>(h);
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	return withMap(m, [&](auto& map) {
		size_t n = 0;
		for (auto it = map.beginLeaves(bv, occupied != 0, free_space != 0, unknown != 0, false, min_depth),
		          end = map.endLeaves();
		     it != end; ++it, ++n) {
			if (codes && n < cap) {
				codes[n] = it.getCode().getCode();
				depths[n] = it.getDepth();
				occ[n] = (float)it->occupancy;
			}
		}
		return n;
	});
}

// Frustum(pos, target, up, vertical_angle, horizontal_angle, near, far) (geometry/frustum.h):
// out = 6 x (normal xyz, distance)
void ufo_ref_frustum7(const double* pos, const double* target, const double* up, double vertical_angle,
                      double horizontal_angle, double near_distance, double far_distance, double* out)
{
	const geo::Frustum f(pt(pos), pt(target), pt(up), vertical_angle, horizontal_angle, near_distance, far_distance);
	for (int i = 0; i < 6; ++i) {
		put(f.planes[i].normal, out + 4 * i);
		out[4 * i + 3] = f.planes[i].distance;
	}
}

// OBB(centre, half_size, Point(roll, pitch, yaw)) (geometry/obb.h): out = rotation w x y z
void ufo_ref_quaternion_rpy(double roll, double pitch, double yaw, double* out)
{
	const geo::OBB o(geo::Point(0, 0, 0), geo::Point(1, 1, 1), geo::Point(roll, pitch, yaw));
	for (int i = 0; i < 4; ++i) out[i] = o.rotation[i];
}

// Ray(origin, direction) (geometry/ray.h): out = origin, normalised direction
void ufo_ref_ray(const double* origin, const double* direction, double* out)
{
	const geo::Ray r(pt(origin), pt(direction));
	put(r.origin, out);
	put(r.direction, out + 3);
}

// Plane(v1, v2, v3) (geometry/plane.h): out = normal xyz, distance
void ufo_ref_plane3(const double* v1, const double* v2, const double* v3, double* out)
{
	const geo::Plane p(pt(v1), pt(v2), pt(v3));
	put(p.normal, out);
	out[3] = p.distance;
}

}  // extern "C"
