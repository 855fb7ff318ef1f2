// ufomap.hpp -- source-compatible C++ facade of the UFOMap integration path over the
// C ABI in ufomap_b200.h.  A caller written against the reference's
//   #include <ufo/map/ufomap.h>        (ufomap/include/ufo/map/ufomap.h:45-48)
// and using OccupancyMap / OccupancyMapColor, insertPointCloud[Discrete],
// insertPointCloudDone/Wait, computeRay, toCode/toKey/toCoord, Code, Key, Point3,
// PointCloud compiles against this header unchanged (same namespaces, names, argument
// order and defaults); the work runs on the GPU behind libufomap_b200.so.
//
// Reference interfaces mirrored here (paths under /root/reference/ufomap/include/ufo/):
//   math/vector3.h:52-328          -> ufo::math::Vector3
//   math/quaternion.h, pose6.h     -> ufo::math::Quaternion, Pose6 (rotate + translate only)
//   map/types.h:54-102, color.h    -> KeyType, CodeType, DepthType, Point3, Point3Color, Color
//   map/point_cloud.h:64-278       -> PointCloudT, PointCloud, PointCloudColor
//   map/key.h:63-195               -> Key, KeyRay
//   map/code.h:69-371              -> Code, CodeRay
//   map/occupancy_map.h:49-82, occupancy_map_base.h:270-443,734-822, octree.h:299-496,
//   occupancy_map_color.h:49-400   -> OccupancyMap, OccupancyMapColor
//
// Differences, all documented in DESIGN.md: state getters use the INTENDED node semantics
// (the reference's getNode is off by one level, octree.h:974-985); early_stopping != 0 is
// rejected (order-dependent in the reference) unless setEarlyStoppingExact(true); errors of the void insert functions are
// kept in lastError().
#pragma once

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <fstream>
#include <istream>
#include <iterator>
#include <memory>
#include <optional>
#include <ostream>
#include <string>
#include <type_traits>
#include <variant>
#include <vector>

#include "../ufomap_b200.h"

namespace ufo::math
{
class Vector3
{
 public:
	Vector3() : v_{0.0, 0.0, 0.0} {}
	Vector3(double x, double y, double z) : v_{x, y, z} {}

	double& operator[](std::size_t i) { return v_[i]; }
	double const& operator[](std::size_t i) const { return v_[i]; }
	double& operator()(std::size_t i) { return v_[i]; }
	double const& operator()(std::size_t i) const { return v_[i]; }
	double& x() { return v_[0]; }
	double& y() { return v_[1]; }
	double& z() { return v_[2]; }
	double const& x() const { return v_[0]; }
	double const& y() const { return v_[1]; }
	double const& z() const { return v_[2]; }

	Vector3 operator-() const { return {-v_[0], -v_[1], -v_[2]}; }
	Vector3 operator+(Vector3 const& o) const { return {v_[0] + o.v_[0], v_[1] + o.v_[1], v_[2] + o.v_[2]}; }
	Vector3 operator-(Vector3 const& o) const { return {v_[0] - o.v_[0], v_[1] - o.v_[1], v_[2] - o.v_[2]}; }
	Vector3 operator*(double s) const { return {v_[0] * s, v_[1] * s, v_[2] * s}; }
	Vector3 operator/(double s) const { return {v_[0] / s, v_[1] / s, v_[2] / s}; }
	Vector3& operator+=(Vector3 const& o) { return *this = *this + o; }
	Vector3& operator-=(Vector3 const& o) { return *this = *this - o; }
	Vector3& operator*=(double s) { return *this = *this * s; }
	Vector3& operator/=(double s) { return *this = *this / s; }
	bool operator==(Vector3 const& o) const { return v_[0] == o.v_[0] && v_[1] == o.v_[1] && v_[2] == o.v_[2]; }
	bool operator!=(Vector3 const& o) const { return !(*this == o); }

	double dot(Vector3 const& o) const { return (v_[0] * o.v_[0]) + (v_[1] * o.v_[1]) + (v_[2] * o.v_[2]); }
	Vector3 cross(Vector3 const& o) const
	{
		return {v_[1] * o.v_[2] - v_[2] * o.v_[1], v_[2] * o.v_[0] - v_[0] * o.v_[2],
		        v_[0] * o.v_[1] - v_[1] * o.v_[0]};
	}
	double squaredNorm() const { return dot(*this); }
	double norm() const { return std::sqrt(squaredNorm()); }
	Vector3& normalize() { return *this /= norm(); }
	Vector3 normalized() const { return *this / norm(); }
	double distance(Vector3 const& o) const { return (*this - o).norm(); }
	double min() const { return std::min(std::min(v_[0], v_[1]), v_[2]); }
	double max() const { return std::max(std::max(v_[0], v_[1]), v_[2]); }
	std::size_t size() const { return 3; }
	double const* data() const { return v_; }

 private:
	double v_[3];
};

// Unit quaternion (w, x, y, z) -- only what the cloud transform needs.  The arithmetic lives in
// the library (ufo_b200_pose_from_rpy / ufo_b200_transform_points), which is compiled without
// FMA contraction and reproduces math/quaternion.h:69-93,253-286 bit for bit whatever flags the
// including translation unit is built with.
class Quaternion
{
 public:
	Quaternion() : w_(1), x_(0), y_(0), z_(0) {}
	Quaternion(double w, double x, double y, double z) : w_(w), x_(x), y_(y), z_(z) {}
	Quaternion(double roll, double pitch, double yaw)
	{
		double pose[7];
		ufo_b200_pose_from_rpy(0, 0, 0, roll, pitch, yaw, pose);
		w_ = pose[3];
		x_ = pose[4];
		y_ = pose[5];
		z_ = pose[6];
	}
	double w() const { return w_; }
	double x() const { return x_; }
	double y() const { return y_; }
	double z() const { return z_; }
	Quaternion inversed() const { return Quaternion(w_, -x_, -y_, -z_); }
	Vector3 rotate(Vector3 const& p) const
	{
		double pose[7] = {0, 0, 0, w_, x_, y_, z_};
		double r[3];
		ufo_b200_transform_points(pose, p.data(), 1, UFO_B200_XYZ_F64, r);
		// (goes through the zero-translation transform: identical except that a -0.0 component
		// comes back as +0.0, which no key computation can see)
		return Vector3(r[0], r[1], r[2]);
	}

 private:
	double w_, x_, y_, z_;
};

class Pose6
{
 public:
	Pose6() {}
	Pose6(Vector3 const& t, Quaternion const& r) : t_(t), r_(r) {}
	Pose6(double x, double y, double z, double roll, double pitch, double yaw)
	    : t_(x, y, z), r_(roll, pitch, yaw)
	{
	}
	Pose6(double t_x, double t_y, double t_z, double r_w, double r_x, double r_y, double r_z)
	    : t_(t_x, t_y, t_z), r_(r_w, r_x, r_y, r_z)
	{
	}
	Vector3 const& translation() const { return t_; }
	Vector3& translation() { return t_; }
	Quaternion const& rotation() const { return r_; }
	Quaternion& rotation() { return r_; }
	// math/pose6.h:115-125
	Vector3 transform(Vector3 const& p) const
	{
		double pose[7];
		pack(pose);
		double r[3];
		ufo_b200_transform_points(pose, p.data(), 1, UFO_B200_XYZ_F64, r);
		return Vector3(r[0], r[1], r[2]);
	}
	// tx ty tz qw qx qy qz, the C ABI's frame_pose
	void pack(double pose[7]) const
	{
		pose[0] = t_.x();
		pose[1] = t_.y();
		pose[2] = t_.z();
		pose[3] = r_.w();
		pose[4] = r_.x();
		pose[5] = r_.y();
		pose[6] = r_.z();
	}

 private:
	Vector3 t_;
	Quaternion r_;
};
}  // namespace ufo::math

namespace ufo::geometry
{
using Point = ufo::math::Vector3;
// geometry/aabb.h:49-70 -- the one bounding volume the mapping server exports with
struct AABB {
	Point center;
	Point half_size;
	AABB() {}
	AABB(Point const& c, double hs) : center(c), half_size(hs, hs, hs) {}
	AABB(Point const& min, Point const& max) : half_size((max - min) / 2.0) { center = min + half_size; }
	Point getMin() const { return center - half_size; }
	Point getMax() const { return center + half_size; }
};

// The other shapes of a bounding volume (geometry/*.h), with the reference's members and
// constructors.  The constructors whose arithmetic decides the doubles run in the library
// (ufo_b200_geometry_*, compiled without FMA contraction), so every caller gets the reference's
// values whatever flags it is built with.
struct Sphere {
	Point center;
	double radius;
	Sphere() : center(0.0, 0.0, 0.0), radius(0.0) {}
	Sphere(Point const& center, double radius) : center(center), radius(radius) {}
};

struct OBB {
	Point center;
	Point half_size;
	math::Quaternion rotation;
	OBB() {}
	OBB(Point const& center, Point const& half_size) : center(center), half_size(half_size) {}
	OBB(Point const& center, Point const& half_size, math::Quaternion const& rotation)
	    : center(center), half_size(half_size), rotation(rotation)
	{
	}
	// rotation = (roll, pitch, yaw)
	OBB(Point const& center, Point const& half_size, Point const& rotation)
	    : center(center), half_size(half_size), rotation(rotation[0], rotation[1], rotation[2])
	{
	}
};

struct Plane {
	Point normal;
	double distance;
	Plane() : normal(1.0, 0.0, 0.0), distance(0.0) {}
	Plane(Point const& normal, double distance) : normal(normal), distance(distance) {}
	Plane(Point const& v_1, Point const& v_2, Point const& v_3)
	{
		double p[4];
		ufo_b200_geometry_plane(v_1.data(), v_2.data(), v_3.data(), p);
		normal = Point(p[0], p[1], p[2]);
		distance = p[3];
	}
};

struct Ray {
	Point origin;
	Point direction;
	Ray() : direction(0.0, 0.0, 1.0) {}
	// the direction is normalised
	Ray(Point const& origin, Point const& direction)
	{
		double r[6];
		ufo_b200_geometry_ray(origin.data(), direction.data(), r);
		this->origin = Point(r[0], r[1], r[2]);
		this->direction = Point(r[3], r[4], r[5]);
	}
};

struct LineSegment {
	Point start;
	Point end;
	LineSegment() {}
	LineSegment(Point const& start, Point const& end) : start(start), end(end) {}
};

struct Frustum {
	std::array<Plane, 6> planes;
	Frustum() {}
	Frustum(Point const& pos, Point const& target, Point const& up, double vertical_angle, double horizontal_angle,
	        double near_distance, double far_distance)
	{
		double p[24];
		ufo_b200_geometry_frustum(pos.data(), target.data(), up.data(), vertical_angle, horizontal_angle, near_distance,
		                          far_distance, p);
		for (int i = 0; i < 6; ++i) planes[i] = Plane(Point(p[4 * i], p[4 * i + 1], p[4 * i + 2]), p[4 * i + 3]);
	}
	Plane const& top() const { return planes[0]; }
	Plane& top() { return planes[0]; }
	Plane const& bottom() const { return planes[1]; }
	Plane& bottom() { return planes[1]; }
	Plane const& left() const { return planes[2]; }
	Plane& left() { return planes[2]; }
	Plane const& right() const { return planes[3]; }
	Plane& right() { return planes[3]; }
	Plane const& near() const { return planes[4]; }
	Plane& near() { return planes[4]; }
	Plane const& far() const { return planes[5]; }
	Plane& far() { return planes[5]; }
};

// geometry/types.h: the shapes in this order (the C ABI's ufo_b200_volume type numbers)
using BoundingVar = std::variant<AABB, Frustum, LineSegment, OBB, Plane, Point, Ray, Sphere>;

// geometry/bounding_volume.h: a union of shapes; empty = the whole map
class BoundingVolume
{
 public:
	void add(BoundingVar const& bv) { bounding_volume_.push_back(bv); }
	std::size_t size() const { return bounding_volume_.size(); }
	bool empty() const { return bounding_volume_.empty(); }
	std::vector<BoundingVar>::iterator begin() { return bounding_volume_.begin(); }
	std::vector<BoundingVar>::const_iterator begin() const { return bounding_volume_.begin(); }
	std::vector<BoundingVar>::const_iterator cbegin() const { return bounding_volume_.cbegin(); }
	std::vector<BoundingVar>::iterator end() { return bounding_volume_.end(); }
	std::vector<BoundingVar>::const_iterator end() const { return bounding_volume_.end(); }
	std::vector<BoundingVar>::const_iterator cend() const { return bounding_volume_.cend(); }

 private:
	std::vector<BoundingVar> bounding_volume_;
};

// one shape as the C ABI's record
inline ufo_b200_volume toRecord(BoundingVar const& bv)
{
	ufo_b200_volume r{};
	r.type = (std::uint32_t)bv.index();
	double* v = r.v;
	auto put = [&v](Point const& p) {
		*v++ = p[0];
		*v++ = p[1];
		*v++ = p[2];
	};
	std::visit(
	    [&](auto const& s) {
		    using T = std::decay_t<decltype(s)>;
		    if constexpr (std::is_same_v<T, AABB>) {
			    put(s.center);
			    put(s.half_size);
		    } else if constexpr (std::is_same_v<T, Frustum>) {
			    for (Plane const& p : s.planes) {
				    put(p.normal);
				    *v++ = p.distance;
			    }
		    } else if constexpr (std::is_same_v<T, LineSegment>) {
			    put(s.start);
			    put(s.end);
		    } else if constexpr (std::is_same_v<T, OBB>) {
			    put(s.center);
			    put(s.half_size);
			    *v++ = s.rotation.w();
			    *v++ = s.rotation.x();
			    *v++ = s.rotation.y();
			    *v++ = s.rotation.z();
		    } else if constexpr (std::is_same_v<T, Plane>) {
			    put(s.normal);
			    *v++ = s.distance;
		    } else if constexpr (std::is_same_v<T, Point>) {
			    put(s);
		    } else if constexpr (std::is_same_v<T, Ray>) {
			    put(s.origin);
			    put(s.direction);
		    } else {
			    put(s.center);
			    *v++ = s.radius;
		    }
	    },
	    bv);
	return r;
}

inline std::vector<ufo_b200_volume> toRecords(BoundingVolume const& bv)
{
	std::vector<ufo_b200_volume> out;
	out.reserve(bv.size());
	for (BoundingVar const& b : bv) out.push_back(toRecord(b));
	return out;
}
}  // namespace ufo::geometry

namespace ufo::map
{
using CodeType = std::uint64_t;
using KeyType = unsigned int;
using DepthType = unsigned int;
using ColorType = std::uint8_t;
using Point3 = ufo::math::Vector3;

struct Color {
	ColorType r = 0, g = 0, b = 0;
	Color() {}
	Color(ColorType r_, ColorType g_, ColorType b_) : r(r_), g(g_), b(b_) {}
	bool operator==(Color const& o) const { return r == o.r && g == o.g && b == o.b; }
	bool operator!=(Color const& o) const { return !(*this == o); }
	bool isSet() const { return r || g || b; }
};

class Point3Color : public Point3
{
 public:
	Point3Color() {}
	Point3Color(Point3 const& p, Color const& c = Color()) : Point3(p), color_(c) {}
	Point3Color(double x, double y, double z, ColorType r = 0, ColorType g = 0, ColorType b = 0)
	    : Point3(x, y, z), color_(r, g, b)
	{
	}
	Color const& getColor() const { return color_; }
	Color& getColor() { return color_; }
	void setColor(Color const& c) { color_ = c; }
	void setColor(ColorType r, ColorType g, ColorType b) { color_ = Color(r, g, b); }

 private:
	Color color_;
};

template <typename T, typename = std::enable_if_t<std::is_base_of_v<Point3, T>>>
class PointCloudT
{
 public:
	using iterator = typename std::vector<T>::iterator;
	using const_iterator = typename std::vector<T>::const_iterator;
	T& operator[](std::size_t i) { return pts_[i]; }
	T const& operator[](std::size_t i) const { return pts_[i]; }
	void clear() { pts_.clear(); }
	void reserve(std::size_t n) { pts_.reserve(n); }
	void resize(std::size_t n) { pts_.resize(n); }
	std::size_t size() const { return pts_.size(); }
	bool empty() const { return pts_.empty(); }
	void push_back(T const& p) { pts_.push_back(p); }
	void push_back(PointCloudT const& other) { pts_.insert(pts_.end(), other.begin(), other.end()); }
	iterator begin() { return pts_.begin(); }
	iterator end() { return pts_.end(); }
	const_iterator begin() const { return pts_.begin(); }
	const_iterator end() const { return pts_.end(); }
	const_iterator cbegin() const { return pts_.cbegin(); }
	const_iterator cend() const { return pts_.cend(); }
	T const* data() const { return pts_.data(); }
	// point_cloud.h:150-166 (the `parallel` hint is accepted and ignored)
	void transform(ufo::math::Pose6 const& pose, bool /*parallel*/ = false)
	{
		// batched through the library (exact arithmetic, see Quaternion): one call per 1024 points
		double f[7], in[3 * 1024], out[3 * 1024];
		pose.pack(f);
		for (std::size_t base = 0; base < pts_.size(); base += 1024) {
			std::size_t m = std::min<std::size_t>(1024, pts_.size() - base);
			for (std::size_t i = 0; i < m; ++i) {
				in[3 * i] = pts_[base + i].x();
				in[3 * i + 1] = pts_[base + i].y();
				in[3 * i + 2] = pts_[base + i].z();
			}
			ufo_b200_transform_points(f, in, m, UFO_B200_XYZ_F64, out);
			for (std::size_t i = 0; i < m; ++i) {
				pts_[base + i].x() = out[3 * i];
				pts_[base + i].y() = out[3 * i + 1];
				pts_[base + i].z() = out[3 * i + 2];
			}
		}
	}

 private:
	std::vector<T> pts_;
};
using PointCloud = PointCloudT<Point3>;
using PointCloudColor = PointCloudT<Point3Color>;

class Key
{
 public:
	Key() : k_{0, 0, 0}, depth_(0) {}
	Key(KeyType x, KeyType y, KeyType z, DepthType depth) : k_{x, y, z}, depth_(depth) {}
	DepthType getDepth() const { return depth_; }
	bool operator==(Key const& o) const { return depth_ == o.depth_ && k_ == o.k_; }
	bool operator!=(Key const& o) const { return !(*this == o); }
	bool equals(Key const& o, DepthType depth = 0) const
	{
		return (k_[0] >> depth) == (o.k_[0] >> depth) && (k_[1] >> depth) == (o.k_[1] >> depth) &&
		       (k_[2] >> depth) == (o.k_[2] >> depth);
	}
	KeyType& operator[](std::size_t i) { return k_[i]; }
	KeyType const& operator[](std::size_t i) const { return k_[i]; }
	KeyType const& x() const { return k_[0]; }
	KeyType const& y() const { return k_[1]; }
	KeyType const& z() const { return k_[2]; }

 private:
	std::array<KeyType, 3> k_;
	DepthType depth_;
};
using KeyRay = std::vector<Key>;

class Code
{
 public:
	Code() : code_(0), depth_(0) {}
	Code(CodeType code, DepthType depth = 0) : code_(code), depth_(depth) {}
	Code(Key const& key) : depth_(key.getDepth())
	{
		std::uint32_t k[3] = {key[0], key[1], key[2]};
		code_ = ufo_b200_key_to_code(k);
	}
	bool operator==(Code const& o) const { return code_ == o.code_ && depth_ == o.depth_; }
	bool operator!=(Code const& o) const { return !(*this == o); }
	CodeType getCode() const { return code_; }
	DepthType getDepth() const { return depth_; }
	Code toDepth(DepthType depth) const
	{
		CodeType s = 3 * depth;
		return Code((code_ >> s) << s, depth);
	}
	std::size_t getChildIdx(DepthType depth) const { return (code_ >> (3 * depth)) & CodeType(7); }
	Code getChild(std::size_t idx) const
	{
		if (0 == depth_) return *this;
		return Code(code_ + (CodeType(idx) << (3 * (depth_ - 1))), depth_ - 1);
	}
	Key toKey() const
	{
		std::uint32_t k[3];
		ufo_b200_code_to_key(code_, k);
		return Key(k[0], k[1], k[2], depth_);
	}
	KeyType toKey(std::size_t axis) const { return toKey()[axis]; }
	struct Hash {
		std::size_t operator()(Code const& c) const { return static_cast<std::size_t>(c.code_); }
	};

 private:
	CodeType code_;
	DepthType depth_;
};
using CodeRay = std::vector<Code>;

enum class OccupancyState { unknown, free, occupied };

// what an iterator dereferences to (map/occupancy_map_node.h: OccupancyNode / ColorOccupancyNode value)
struct OccupancyValue {
	float occupancy = 0.0f;  // log-odds
};
struct ColorOccupancyValue {
	float occupancy = 0.0f;  // log-odds
	Color color;
};

namespace detail
{
// Common implementation of OccupancyMap / OccupancyMapColor over the C ABI.
template <bool COLOR>
class MapFacade
{
 public:
	MapFacade(double resolution, DepthType depth_levels = 16, bool automatic_pruning = true,
	          double occupied_thres = 0.5, double free_thres = 0.5, double prob_hit = 0.7,
	          double prob_miss = 0.4, double clamping_thres_min = 0.1192,
	          double clamping_thres_max = 0.971)
	{
		ufo_b200_params p;
		ufo_b200_default_params(&p);
		p.resolution = resolution;
		p.depth_levels = depth_levels;
		p.automatic_pruning = automatic_pruning;
		p.occupied_thres = occupied_thres;
		p.free_thres = free_thres;
		p.prob_hit = prob_hit;
		p.prob_miss = prob_miss;
		p.clamping_thres_min = clamping_thres_min;
		p.clamping_thres_max = clamping_thres_max;
		p.color = COLOR ? 1 : 0;
		params_ = p;
		int rc = ufo_b200_create(&p, &map_);
		if (UFO_B200_E_INVALID == rc) {
			// octree.h:931-935
			throw std::invalid_argument("depth_levels has to be [2, 21]");
		}
		if (UFO_B200_OK != rc) {
			throw std::runtime_error("ufomap_b200: no usable CUDA device (there is no CPU fallback)");
		}
	}
	// The file constructors (occupancy_map_base.h:878-886): a map of resolution 0.1 and 16 depth
	// levels that then reads the file.  A failed read leaves that map and its status in lastStatus().
	MapFacade(std::string const& filename, bool automatic_pruning = true, double occupied_thres = 0.5,
	          double free_thres = 0.5, double prob_hit = 0.7, double prob_miss = 0.4,
	          double clamping_thres_min = 0.1192, double clamping_thres_max = 0.971)
	    : MapFacade(0.1, 16, automatic_pruning, occupied_thres, free_thres, prob_hit, prob_miss, clamping_thres_min,
	                clamping_thres_max)
	{
		read(filename);
	}
	// The copy constructor (occupancy_map_base.h:888-897) without its file round trip: the map is
	// copied on its device (ufo_b200_clone).  As in the reference, whose copy passes the source's
	// probability getters to its constructor, the copy's sensor model is toLogit(toProb(x)) of the
	// source's.  Change detection, min/max change detection, the early-stopping opt-in and a stream set
	// on the source start as on a new map.  Throws std::runtime_error when the device copy fails.
	MapFacade(MapFacade const& other) : map_(copyOf(other)), params_(other.params_) {}
	// Copy assignment, an extension: the reference's is deleted (its map holds a std::future,
	// occupancy_map_base.h:1553).  Same meaning as the copy constructor; when the copy fails this map is
	// unchanged and the error is thrown.
	MapFacade& operator=(MapFacade const& other)
	{
		if (this != &other) {
			MapFacade copy(other);
			std::swap(map_, copy.map_);
			params_ = copy.params_;
			changes_.clear();
			change_enabled_ = false;
			change_depth_ = 0;
			minmax_enabled_ = false;
			last_status_ = 0;
		}
		return *this;
	}
	virtual ~MapFacade() { ufo_b200_destroy(map_); }

	virtual std::string getTreeType() const noexcept { return COLOR ? "occupancy_map_color" : "occupancy_map"; }

	//
	// Iteration (occupancy_map_base.h:93-163, iterator/octree.h, iterator/occupancy_map.h): the nodes
	// come from one ufo_b200_iterate call -- computed on the device, in the reference iterator's order --
	// and the iterator walks that snapshot, so a map changed after begin*() does not change an
	// iteration in progress.  Forward iterator; copies share the snapshot.
	//
	class Iterator
	{
	 public:
		using value_type = std::conditional_t<COLOR, ColorOccupancyValue, OccupancyValue>;
		using difference_type = std::ptrdiff_t;
		using pointer = value_type const*;
		using reference = value_type const&;
		using iterator_category = std::forward_iterator_tag;

		Iterator() {}  // the end iterator

		// Equal when both are exhausted, or when both walk the same snapshot and are at the same node.
		// (The reference's operator== compares the tree pointers only, so two live iterators of one map
		// compare equal there whatever node they are at; that is not reproduced.)
		bool operator==(Iterator const& o) const
		{
			return (atEnd() && o.atEnd()) || (!atEnd() && !o.atEnd() && s_ == o.s_ && i_ == o.i_);
		}
		bool operator!=(Iterator const& o) const { return !(*this == o); }
		Iterator& operator++()
		{
			++i_;
			load();
			return *this;
		}
		Iterator operator++(int)
		{
			Iterator r = *this;
			++(*this);
			return r;
		}
		reference operator*() const { return value_; }
		pointer operator->() const { return &value_; }

		// Code::getChild from the root: Code(code, max(getDepth(), depth)) with the bits below zero
		Code getCode(DepthType depth = 0) const
		{
			DepthType d = std::min(std::max(getDepth(), depth), s_->levels);
			CodeType s = CodeType(3) * d;
			return Code((s_->codes[i_] >> s) << s, d);
		}
		DepthType getDepth() const { return s_->depths[i_]; }
		Point3 getCenter() const { return center_; }
		double getX() const { return center_.x(); }
		double getY() const { return center_.y(); }
		double getZ() const { return center_.z(); }
		double getSize() const { return 2.0 * getHalfSize(); }
		double getHalfSize() const { return s_->half_size[getDepth()]; }
		ufo::geometry::AABB getBoundingVolume() const { return ufo::geometry::AABB(center_, getHalfSize()); }
		bool isLeaf() const { return s_->flags[i_] & 4u; }
		bool isPureLeaf() const { return 0 == getDepth(); }
		bool hasChildren() const { return !isLeaf(); }
		// occupancy_map_base.h:926-980 on the node's value and flags
		bool isOccupied() const { return s_->occupied_thres_log < value_.occupancy; }
		bool isFree() const { return s_->free_thres_log > value_.occupancy; }
		bool isUnknown() const { return !isOccupied() && !isFree(); }
		bool containsOccupied() const { return isOccupied(); }
		bool containsFree() const { return s_->flags[i_] & 1u; }
		bool containsUnknown() const { return s_->flags[i_] & 2u; }
		double getOccupancy() const { return toProb(value_.occupancy); }

	 private:
		friend class MapFacade;
		struct Snapshot {
			std::vector<std::uint64_t> codes;
			std::vector<std::uint8_t> depths, flags, rgb;
			std::vector<float> logodds;
			double half_size[22];
			DepthType levels;
			double occupied_thres_log, free_thres_log;
		};
		explicit Iterator(std::shared_ptr<Snapshot const> s) : s_(std::move(s)) { load(); }
		bool atEnd() const { return !s_ || i_ >= s_->codes.size(); }
		void load()
		{
			if (atEnd()) return;
			value_.occupancy = s_->logodds[i_];
			if constexpr (COLOR) value_.color = Color(s_->rgb[3 * i_], s_->rgb[3 * i_ + 1], s_->rgb[3 * i_ + 2]);
			// getChildCenter from the root down (octree.h:625-633), as the reference iterator accumulates it
			Point3 c(0.0, 0.0, 0.0);
			for (DepthType d = s_->levels; d > getDepth(); --d) {
				unsigned idx = unsigned(s_->codes[i_] >> (3 * (d - 1))) & 7u;
				double hs = s_->half_size[d - 1];
				c[0] += (idx & 1u) ? hs : -hs;
				c[1] += (idx & 2u) ? hs : -hs;
				c[2] += (idx & 4u) ? hs : -hs;
			}
			center_ = c;
		}
		std::shared_ptr<Snapshot const> s_;
		std::size_t i_ = 0;
		value_type value_{};
		Point3 center_;
	};
	using TreeIterator = Iterator;
	using LeafIterator = Iterator;

	// beginTree / beginLeaves with the reference's overloads and defaults.  A call that fails (no
	// device, depth_levels < 5) gives an empty sequence; lastError() says why.
	Iterator beginTree(bool occupied_space = true, bool free_space = true, bool unknown_space = false,
	                   bool contains = false, DepthType min_depth = 0) const
	{
		return iterate(false, {}, occupied_space, free_space, unknown_space, contains, min_depth);
	}
	Iterator beginTree(ufo::geometry::BoundingVar const& bounding_volume, bool occupied_space = true,
	                   bool free_space = true, bool unknown_space = false, bool contains = false,
	                   DepthType min_depth = 0) const
	{
		return iterate(false, {ufo::geometry::toRecord(bounding_volume)}, occupied_space, free_space, unknown_space, contains,
		               min_depth);
	}
	Iterator beginTree(ufo::geometry::BoundingVolume const& bounding_volume, bool occupied_space = true,
	                   bool free_space = true, bool unknown_space = false, bool contains = false,
	                   DepthType min_depth = 0) const
	{
		return iterate(false, ufo::geometry::toRecords(bounding_volume), occupied_space, free_space, unknown_space, contains,
		               min_depth);
	}
	Iterator endTree() const noexcept { return Iterator(); }
	Iterator beginLeaves(bool occupied_space = true, bool free_space = true, bool unknown_space = false,
	                     bool contains = false, DepthType min_depth = 0) const
	{
		return iterate(true, {}, occupied_space, free_space, unknown_space, contains, min_depth);
	}
	Iterator beginLeaves(ufo::geometry::BoundingVar const& bounding_volume, bool occupied_space = true,
	                     bool free_space = true, bool unknown_space = false, bool contains = false,
	                     DepthType min_depth = 0) const
	{
		return iterate(true, {ufo::geometry::toRecord(bounding_volume)}, occupied_space, free_space, unknown_space, contains,
		               min_depth);
	}
	Iterator beginLeaves(ufo::geometry::BoundingVolume const& bounding_volume, bool occupied_space = true,
	                     bool free_space = true, bool unknown_space = false, bool contains = false,
	                     DepthType min_depth = 0) const
	{
		return iterate(true, ufo::geometry::toRecords(bounding_volume), occupied_space, free_space, unknown_space, contains,
		               min_depth);
	}
	Iterator endLeaves() const noexcept { return Iterator(); }

	//
	// Nearest-first iteration (occupancy_map_base.h:169-245) with the intended semantics (DESIGN §8):
	// the nodes of beginTree / beginLeaves with the same arguments, in non-decreasing squared distance
	// from a point, equal distances in beginTree / beginLeaves order.  The iterator fetches the sequence
	// lazily in distance shells (ufo_b200_nearest): the first holds at least 8 nodes, each next one at
	// least twice as many as the one before.  A map changed after begin*() ends the iteration at the next
	// shell fetch and sets lastStatus() to UFO_B200_E_INVALID: it never mixes two states of the map.
	// Forward iterator; copies share the fetched shells.  The map must outlive it.
	//
	class NNIterator
	{
	 public:
		using value_type = std::conditional_t<COLOR, ColorOccupancyValue, OccupancyValue>;
		using difference_type = std::ptrdiff_t;
		using pointer = value_type const*;
		using reference = value_type const&;
		using iterator_category = std::forward_iterator_tag;

		NNIterator() {}  // the end iterator

		// as Iterator: equal when both are exhausted, or at the same node of the same sequence
		bool operator==(NNIterator const& o) const
		{
			return (atEnd() && o.atEnd()) || (!atEnd() && !o.atEnd() && s_ == o.s_ && i_ == o.i_);
		}
		bool operator!=(NNIterator const& o) const { return !(*this == o); }
		NNIterator& operator++()
		{
			++i_;
			load();
			return *this;
		}
		NNIterator operator++(int)
		{
			NNIterator r = *this;
			++(*this);
			return r;
		}
		reference operator*() const { return value_; }
		pointer operator->() const { return &value_; }

		double getDistance() const { return std::sqrt(getSquaredDistance()); }
		double getSquaredDistance() const { return s_->d2[i_]; }
		// an extension: the reference's nearest iterators have no getCode
		Code getCode() const { return Code(s_->codes[i_], getDepth()); }
		DepthType getDepth() const { return s_->depths[i_]; }
		Point3 getCenter() const { return center_; }
		double getX() const { return center_.x(); }
		double getY() const { return center_.y(); }
		double getZ() const { return center_.z(); }
		double getSize() const { return 2.0 * getHalfSize(); }
		double getHalfSize() const { return s_->half_size[getDepth()]; }
		ufo::geometry::AABB getAABB() const { return ufo::geometry::AABB(center_, getHalfSize()); }
		bool isLeaf() const { return s_->flags[i_] & 4u; }
		bool isPureLeaf() const { return 0 == getDepth(); }
		bool hasChildren() const { return !isLeaf(); }
		bool isOccupied() const { return s_->occupied_thres_log < value_.occupancy; }
		bool isFree() const { return s_->free_thres_log > value_.occupancy; }
		bool isUnknown() const { return !isOccupied() && !isFree(); }
		bool containsOccupied() const { return isOccupied(); }
		bool containsFree() const { return s_->flags[i_] & 1u; }
		bool containsUnknown() const { return s_->flags[i_] & 2u; }
		double getOccupancy() const { return toProb(value_.occupancy); }

	 private:
		friend class MapFacade;
		struct State {
			MapFacade const* map;
			double point[3];
			std::vector<ufo_b200_volume> bv;
			bool leaves, occupied, free_space, unknown, contains;
			DepthType min_depth;
			std::uint64_t revision = 0;
			double d2_next = 0.0;  // where the next shell starts; +inf: none left
			std::size_t want = 8;
			std::vector<std::uint64_t> codes;
			std::vector<std::uint8_t> depths, flags, rgb;
			std::vector<float> logodds;
			std::vector<double> d2;
			double half_size[22];
			DepthType levels;
			double occupied_thres_log, free_thres_log;

			// appends the next shell; false when none is left, the map changed or the call failed
			bool fetch()
			{
				if (!(d2_next < HUGE_VAL)) return false;
				ufo_b200_map* m = map->map_;
				auto call = [&](std::size_t at, std::size_t cap, std::size_t* n, double* next) {
					return ufo_b200_nearest(m, point, bv.data(), bv.size(), leaves, occupied, free_space, unknown, contains,
					                        min_depth, d2_next, want, cap ? codes.data() + at : nullptr,
					                        cap ? depths.data() + at : nullptr, cap ? logodds.data() + at : nullptr,
					                        cap ? flags.data() + at : nullptr, cap && COLOR ? rgb.data() + 3 * at : nullptr,
					                        cap ? d2.data() + at : nullptr, cap, n, next);
				};
				auto fail = [&](int status) {
					map->last_status_ = status;
					d2_next = HUGE_VAL;
					return false;
				};
				std::size_t n = 0;
				double next = HUGE_VAL;
				int rc = call(0, 0, &n, &next);
				ufo_b200_nearest_stats st{};
				if (UFO_B200_OK != rc) return fail(rc);
				ufo_b200_last_nearest_stats(m, &st);
				if (0 == revision) revision = st.revision;
				if (st.revision != revision) return fail(UFO_B200_E_INVALID);
				const std::size_t at = codes.size();
				codes.resize(at + n);
				depths.resize(at + n);
				logodds.resize(at + n);
				flags.resize(at + n);
				d2.resize(at + n);
				if (COLOR) rgb.resize(3 * (at + n));
				if (n) {
					rc = call(at, n, &n, &next);
					if (UFO_B200_OK != rc) return fail(rc);
					ufo_b200_last_nearest_stats(m, &st);
					if (st.revision != revision) return fail(UFO_B200_E_INVALID);
				}
				d2_next = next;
				want *= 2;
				return n > 0 || fetch();
			}
		};
		explicit NNIterator(std::shared_ptr<State> s) : s_(std::move(s)) { load(); }
		bool atEnd() const { return !s_ || i_ >= s_->codes.size(); }
		void load()
		{
			if (s_ && i_ >= s_->codes.size() && !s_->fetch()) return;
			if (atEnd()) return;
			value_.occupancy = s_->logodds[i_];
			if constexpr (COLOR) value_.color = Color(s_->rgb[3 * i_], s_->rgb[3 * i_ + 1], s_->rgb[3 * i_ + 2]);
			// getChildCenter from the root down (octree.h:625-633), as the reference iterator accumulates it
			Point3 c(0.0, 0.0, 0.0);
			for (DepthType d = s_->levels; d > getDepth(); --d) {
				unsigned idx = unsigned(s_->codes[i_] >> (3 * (d - 1))) & 7u;
				double hs = s_->half_size[d - 1];
				c[0] += (idx & 1u) ? hs : -hs;
				c[1] += (idx & 2u) ? hs : -hs;
				c[2] += (idx & 4u) ? hs : -hs;
			}
			center_ = c;
		}
		std::shared_ptr<State> s_;
		std::size_t i_ = 0;
		value_type value_{};
		Point3 center_;
	};
	using NNTreeIterator = NNIterator;
	using NNLeafIterator = NNIterator;

	// beginNNTree / beginNNLeaves with the reference's overloads and defaults (the point comes before the
	// volume).  A first shell that fails (no device, depth_levels < 5, a non-finite point) gives an empty
	// sequence with its status in lastStatus().
	NNIterator beginNNTree(Point3 const& coord, bool occupied_space = true, bool free_space = true,
	                       bool unknown_space = false, bool contains = false, DepthType min_depth = 0) const
	{
		return nearest(false, coord, {}, occupied_space, free_space, unknown_space, contains, min_depth);
	}
	NNIterator beginNNTree(Point3 const& coord, ufo::geometry::BoundingVar const& bounding_volume,
	                       bool occupied_space = true, bool free_space = true, bool unknown_space = false,
	                       bool contains = false, DepthType min_depth = 0) const
	{
		return nearest(false, coord, {ufo::geometry::toRecord(bounding_volume)}, occupied_space, free_space, unknown_space,
		               contains, min_depth);
	}
	NNIterator beginNNTree(Point3 const& coord, ufo::geometry::BoundingVolume const& bounding_volume,
	                       bool occupied_space = true, bool free_space = true, bool unknown_space = false,
	                       bool contains = false, DepthType min_depth = 0) const
	{
		return nearest(false, coord, ufo::geometry::toRecords(bounding_volume), occupied_space, free_space, unknown_space,
		               contains, min_depth);
	}
	NNIterator endNNTree() const noexcept { return NNIterator(); }
	NNIterator beginNNLeaves(Point3 const& coord, bool occupied_space = true, bool free_space = true,
	                         bool unknown_space = false, bool contains = false, DepthType min_depth = 0) const
	{
		return nearest(true, coord, {}, occupied_space, free_space, unknown_space, contains, min_depth);
	}
	NNIterator beginNNLeaves(Point3 const& coord, ufo::geometry::BoundingVar const& bounding_volume,
	                         bool occupied_space = true, bool free_space = true, bool unknown_space = false,
	                         bool contains = false, DepthType min_depth = 0) const
	{
		return nearest(true, coord, {ufo::geometry::toRecord(bounding_volume)}, occupied_space, free_space, unknown_space,
		               contains, min_depth);
	}
	NNIterator beginNNLeaves(Point3 const& coord, ufo::geometry::BoundingVolume const& bounding_volume,
	                         bool occupied_space = true, bool free_space = true, bool unknown_space = false,
	                         bool contains = false, DepthType min_depth = 0) const
	{
		return nearest(true, coord, ufo::geometry::toRecords(bounding_volume), occupied_space, free_space, unknown_space,
		               contains, min_depth);
	}
	NNIterator endNNLeaves() const noexcept { return NNIterator(); }

	//
	// File / wire format (octree.h:776-864): whole map or the part inside an AABB, truncated at
	// min_depth (0..4); compress = true packs the node stream as one LZ4 block like the reference
	// (needs liblz4.so.1 at run time, else false).
	//
	bool write(std::string const& filename, bool compress = false, DepthType min_depth = 0,
	           int compression_acceleration_level = 1, int compression_level = 0) const
	{
		if (compress) {
			std::ofstream f(filename.c_str(), std::ios_base::out | std::ios_base::binary);
			return f.is_open() && writeCompressed(f, nullptr, false, min_depth, compression_acceleration_level, compression_level) >= 0;
		}
		return UFO_B200_OK == ufo_b200_write_file(map_, filename.c_str(), nullptr, min_depth, 0);
	}
	bool write(std::string const& filename, ufo::geometry::AABB const& bounding_volume, bool compress = false,
	           DepthType min_depth = 0, int compression_acceleration_level = 1,
	           int compression_level = 0) const
	{
		double box[6];
		packBox(bounding_volume, box);
		if (compress) {
			std::ofstream f(filename.c_str(), std::ios_base::out | std::ios_base::binary);
			return f.is_open() && writeCompressed(f, box, false, min_depth, compression_acceleration_level, compression_level) >= 0;
		}
		return UFO_B200_OK == ufo_b200_write_file(map_, filename.c_str(), box, min_depth, 0);
	}
	bool write(std::ostream& s, bool compress = false, DepthType min_depth = 0,
	           int compression_acceleration_level = 1, int compression_level = 0) const
	{
		if (compress) return writeCompressed(s, nullptr, false, min_depth, compression_acceleration_level, compression_level) >= 0;
		std::size_t n = 0;
		if (UFO_B200_OK != ufo_b200_write(map_, nullptr, min_depth, 0, nullptr, 0, &n)) return false;
		std::vector<char> image(n);
		if (UFO_B200_OK != ufo_b200_write(map_, nullptr, min_depth, 0, image.data(), n, &n)) return false;
		s.write(image.data(), (std::streamsize)n);
		return s.good();
	}

	// Octree::write with a BoundingVolume (octree.h:796-864): the save_map service (server.cpp:381-390)
	bool write(std::string const& filename, ufo::geometry::BoundingVolume const& bounding_volume, bool compress = false,
	           DepthType min_depth = 0, int compression_acceleration_level = 1, int compression_level = 0) const
	{
		std::ofstream f(filename.c_str(), std::ios_base::out | std::ios_base::binary);
		return f.is_open() && write(f, bounding_volume, compress, min_depth, compression_acceleration_level, compression_level) &&
		       (f.close(), !f.fail());
	}
	bool write(std::ostream& s, ufo::geometry::BoundingVolume const& bounding_volume, bool compress = false,
	           DepthType min_depth = 0, int compression_acceleration_level = 1, int compression_level = 0) const
	{
		auto const bv = ufo::geometry::toRecords(bounding_volume);
		if (compress)
			return writeCompressedBv(s, bv, false, min_depth, compression_acceleration_level, compression_level) >= 0;
		std::size_t n = 0;
		if (UFO_B200_OK != ufo_b200_write_bv(map_, bv.data(), bv.size(), min_depth, 0, nullptr, 0, &n)) return false;
		std::vector<char> image(n ? n : 1);
		if (UFO_B200_OK != ufo_b200_write_bv(map_, bv.data(), bv.size(), min_depth, 0, image.data(), n, &n)) return false;
		s.write(image.data(), (std::streamsize)n);
		return s.good();
	}

	// EXTENSIONS (no counterpart in the reference): a map in bounded memory (ufomap_b200.h,
	// ufo_b200_retain_bv).  retain removes every brick (16^3 voxels) the volume does not keep and gives
	// its memory back; pageOut returns those bricks as a page blob without changing the map; pageIn puts
	// a blob's bricks back and fails if any of them exists.  An empty BoundingVolume keeps everything.
	// They take an AABB, one shape or a volume, like write; the status is left in lastStatus().
	bool retain(ufo::geometry::BoundingVolume const& bounding_volume, ufo_b200_retain_stats* stats = nullptr)
	{
		auto const bv = ufo::geometry::toRecords(bounding_volume);
		last_status_ = ufo_b200_retain_bv(map_, bv.data(), bv.size(), stats);
		return UFO_B200_OK == last_status_;
	}
	bool retain(ufo::geometry::BoundingVar const& bounding_volume, ufo_b200_retain_stats* stats = nullptr)
	{
		ufo_b200_volume const r = ufo::geometry::toRecord(bounding_volume);
		last_status_ = ufo_b200_retain_bv(map_, &r, 1, stats);
		return UFO_B200_OK == last_status_;
	}
	bool retain(ufo::geometry::AABB const& bounding_volume, ufo_b200_retain_stats* stats = nullptr)
	{
		return retain(ufo::geometry::BoundingVar(bounding_volume), stats);
	}
	std::vector<std::uint8_t> pageOut(ufo::geometry::BoundingVolume const& bounding_volume)
	{
		return pageOutRecords(ufo::geometry::toRecords(bounding_volume));
	}
	std::vector<std::uint8_t> pageOut(ufo::geometry::BoundingVar const& bounding_volume)
	{
		return pageOutRecords({ufo::geometry::toRecord(bounding_volume)});
	}
	std::vector<std::uint8_t> pageOut(ufo::geometry::AABB const& bounding_volume)
	{
		return pageOut(ufo::geometry::BoundingVar(bounding_volume));
	}
	bool pageIn(std::vector<std::uint8_t> const& blob, ufo_b200_retain_stats* stats = nullptr)
	{
		last_status_ = ufo_b200_page_in(map_, blob.data(), blob.size(), stats);
		return UFO_B200_OK == last_status_;
	}
	// getKnownBBX() (occupancy_map_base.h:828-852) and the node counters of octree.h:411-443 for the
	// pruned tree, computed on the device (ufo_b200_tree_info).  The memoryUsage members apply the
	// reference's formula to the sizes of ITS node types on LP64 (inner / leaf: 16 / 4 bytes, colour
	// 24 / 8): they say what the reference would hold for this map, not what this library holds, which
	// poolStats() reports.  A routed or sharded map reports its own part.
	ufo::geometry::AABB getKnownBBX() const
	{
		const ufo_b200_tree_stats t = treeStats();
		if (!t.known) return ufo::geometry::AABB(Point3(0, 0, 0), 0);
		return ufo::geometry::AABB(Point3(t.known_min[0], t.known_min[1], t.known_min[2]),
		                           Point3(t.known_max[0], t.known_max[1], t.known_max[2]));
	}
	std::size_t getNumInnerNodes() const { return treeStats().num_inner_nodes; }
	std::size_t getNumLeafNodes() const { return treeStats().num_leaf_nodes; }
	std::size_t memoryUsageInnerNode() const noexcept { return COLOR ? 24 : 16; }
	std::size_t memoryUsageLeafNode() const noexcept { return COLOR ? 8 : 4; }
	std::size_t memoryUsage() const
	{
		const ufo_b200_tree_stats t = treeStats();
		return t.num_inner_nodes * memoryUsageInnerNode() + t.num_leaf_nodes * memoryUsageLeafNode();
	}
	std::size_t size() const
	{
		const ufo_b200_tree_stats t = treeStats();
		return t.num_inner_nodes + t.num_leaf_nodes;
	}

	// live bricks / upper nodes, pool capacities and device bytes of the map right now
	ufo_b200_pool_counts poolStats()
	{
		ufo_b200_pool_counts c{};
		last_status_ = ufo_b200_pool_stats(map_, &c);
		return c;
	}

	// setValueVolume (occupancy_map_base.h:492-518) for any one shape: the clear_volume service loops
	// over the shapes of its BoundingVolume (server.cpp:345-354).  min_depth 0..4, colour maps at 0;
	// other cases, and more than 2^22 nodes of one level inside the shape, set lastStatus() to
	// UFO_B200_E_UNSUPPORTED.
	void setValueVolume(ufo::geometry::BoundingVar const& bounding_volume, double occupancy_value,
	                    DepthType min_depth = 0)
	{
		const ufo_b200_volume r = ufo::geometry::toRecord(bounding_volume);
		last_status_ = ufo_b200_set_value_volume_bv(map_, &r, occupancy_value, min_depth);
	}

	// setValueVolume (occupancy_map_base.h:492-518) for the bounding volume the mapping server uses
	// (robot clearing server.cpp:152-154, clear_volume service :354): AABB, min_depth 0..4; colour
	// maps at min_depth 0.  Other cases set lastStatus() to UFO_B200_E_UNSUPPORTED.
	void setValueVolume(ufo::geometry::AABB const& bounding_volume, double occupancy_value,
	                    DepthType min_depth = 0)
	{
		double box[6];
		packBox(bounding_volume, box);
		last_status_ = ufo_b200_set_value_volume(map_, box, occupancy_value, min_depth);
	}

	//
	// Per-node writes (occupancy_map_base.h:524-593) and ray insertion (:251-268).  Each call is a
	// batch of one on the device (ufo_b200_update_nodes / ufo_b200_insert_rays); depth 0..6.  Like the
	// inserts they return nothing and leave their status in lastStatus().
	//
	void setOccupancy(Code const& code, double occupancy_value) { writeNode(code, 1, (float)toLogit(occupancy_value)); }
	void setOccupancy(Point3 const& coord, double occupancy_value, DepthType depth = 0)
	{
		setOccupancy(toCode(coord, depth), occupancy_value);
	}
	void setOccupancy(double x, double y, double z, double occupancy_value, DepthType depth = 0)
	{
		setOccupancy(toCode(x, y, z, depth), occupancy_value);
	}
	void updateOccupancy(Code const& code, double occupancy_value_update)
	{
		writeNode(code, 0, (float)toLogit(occupancy_value_update));
	}
	void updateOccupancy(Point3 const& coord, double occupancy_value_update, DepthType depth = 0)
	{
		updateOccupancy(toCode(coord, depth), occupancy_value_update);
	}
	void updateOccupancy(double x, double y, double z, double occupancy_value_update, DepthType depth = 0)
	{
		updateOccupancy(toCode(x, y, z, depth), occupancy_value_update);
	}
	void integrateHit(Code const& code) { writeNode(code, 0, (float)model()[2]); }
	void integrateHit(Point3 const& coord, DepthType depth = 0) { integrateHit(toCode(coord, depth)); }
	void integrateHit(double x, double y, double z, DepthType depth = 0) { integrateHit(toCode(x, y, z, depth)); }
	void integrateMiss(Code const& code) { writeNode(code, 0, (float)model()[3]); }
	void integrateMiss(Point3 const& coord, DepthType depth = 0) { integrateMiss(toCode(coord, depth)); }
	void integrateMiss(double x, double y, double z, DepthType depth = 0) { integrateMiss(toCode(x, y, z, depth)); }
	void insertMissOnRay(Point3 const& origin, Point3 const& end, double max_range = -1, DepthType depth = 0)
	{
		last_status_ = ufo_b200_insert_rays(map_, origin.data(), end.data(), 1, max_range, depth, 0, 0);
	}
	void insertRay(Point3 const& origin, Point3 const& end, double max_range = -1, DepthType depth = 0)
	{
		last_status_ = ufo_b200_insert_rays(map_, origin.data(), end.data(), 1, max_range, depth, 1, 0);
	}

	// Octree::writeData (octree.h:866-917): the node stream of a UFOMap message, whole map or the
	// part inside an AABB, truncated at min_depth (0..4).  Returns the number of bytes written, -1
	// on error (as the reference does).
	int writeData(std::ostream& s, bool compress = false, DepthType min_depth = 0,
	              int compression_acceleration_level = 1, int compression_level = 0) const
	{
		if (compress) return writeCompressed(s, nullptr, true, min_depth, compression_acceleration_level, compression_level);
		return writeDataImpl(s, nullptr, compress, min_depth);
	}
	int writeData(std::ostream& s, ufo::geometry::AABB const& bounding_volume, bool compress = false,
	              DepthType min_depth = 0, int compression_acceleration_level = 1,
	              int compression_level = 0) const
	{
		double box[6];
		packBox(bounding_volume, box);
		if (compress) return writeCompressed(s, box, true, min_depth, compression_acceleration_level, compression_level);
		return writeDataImpl(s, box, compress, min_depth);
	}

	// Octree::writeData with a BoundingVolume (octree.h:885-917): what ufoToMsg publishes for the
	// get_map service (server.cpp:327-336, ufomap_msgs/conversions.h:161-185)
	int writeData(std::ostream& s, ufo::geometry::BoundingVolume const& bounding_volume, bool compress = false,
	              DepthType min_depth = 0, int compression_acceleration_level = 1, int compression_level = 0) const
	{
		auto const bv = ufo::geometry::toRecords(bounding_volume);
		if (compress) return writeCompressedBv(s, bv, true, min_depth, compression_acceleration_level, compression_level);
		std::size_t n = 0;
		if (UFO_B200_OK != ufo_b200_write_data_bv(map_, bv.data(), bv.size(), min_depth, nullptr, 0, &n)) return -1;
		std::vector<char> data(n ? n : 1);
		if (UFO_B200_OK != ufo_b200_write_data_bv(map_, bv.data(), bv.size(), min_depth, data.data(), n, &n)) return -1;
		s.write(data.data(), (std::streamsize)n);
		return s.good() ? (int)n : -1;
	}

	// Octree::readType (octree.h:639-688): the id of a file's header, "" when the first line is not
	// the file mark or the file cannot be opened.  Reads the stream up to the end of its header.
	static std::string readType(std::string const& filename)
	{
		std::ifstream file(filename.c_str(), std::ios_base::in | std::ios_base::binary);
		return file.is_open() ? readType(file) : std::string();
	}
	static std::string readType(std::istream& s)
	{
		std::string head;
		char buf[4096];
		ufo_b200_file_header h;
		while (s.good()) {
			s.read(buf, sizeof buf);
			head.append(buf, (std::size_t)s.gcount());
			ufo_b200_read_header(head.data(), head.size(), &h);
			if (h.data_offset && h.data_offset < head.size()) return h.id;  // the "data" line is complete
		}
		ufo_b200_read_header(head.data(), head.size(), &h);
		return h.id;
	}

	// Octree::read (octree.h:690-729): the file image (header + node stream) into the map.  A file of
	// another resolution / depth_levels re-creates the map with the file's (ufo_b200_read); a failed
	// read changes nothing and leaves its status in lastStatus().
	bool read(std::string const& filename)
	{
		std::ifstream file(filename.c_str(), std::ios_base::in | std::ios_base::binary);
		if (!file.is_open()) {
			last_status_ = UFO_B200_E_INVALID;
			return false;
		}
		return read(file);
	}
	bool read(std::istream& s)
	{
		std::vector<char> image((std::istreambuf_iterator<char>(s)), std::istreambuf_iterator<char>());
		last_status_ = ufo_b200_read(map_, image.data(), image.size());
		if (UFO_B200_OK != last_status_) return false;
		ufo_b200_file_header h;
		ufo_b200_read_header(image.data(), image.size(), &h);
		// the geometry getters read params_
		params_.resolution = h.resolution;
		params_.depth_levels = h.depth_levels;
		return true;
	}

	// Octree::readData with a BoundingVolume (octree.h:751-774; msgToUfo, conversions.h:122-134)
	bool readData(std::istream& s, ufo::geometry::BoundingVolume const& bounding_volume, double resolution,
	              DepthType depth_levels, int uncompressed_data_size = 1, bool compressed = false)
	{
		if (getResolution() != resolution || getTreeDepthLevels() != depth_levels) clear(resolution, depth_levels);
		auto const bv = ufo::geometry::toRecords(bounding_volume);
		std::vector<char> data((std::istreambuf_iterator<char>(s)), std::istreambuf_iterator<char>());
		return UFO_B200_OK == ufo_b200_read_data_bv(map_, bv.data(), bv.size(), data.data(), data.size(), compressed,
		                                            compressed ? (std::size_t)uncompressed_data_size : 0);
	}

	// Octree::readData (octree.h:733-770): merges a node stream (the data of a UFOMap message,
	// ufomap_msgs/conversions.h:122-134) into the map.  Like the reference, a stream written for
	// another resolution / depth clears and resizes the map first.
	bool readData(std::istream& s, double resolution, DepthType depth_levels, int uncompressed_data_size = 1,
	              bool compressed = false)
	{
		return readDataImpl(s, nullptr, resolution, depth_levels, uncompressed_data_size, compressed);
	}
	bool readData(std::istream& s, ufo::geometry::AABB const& bounding_volume, double resolution,
	              DepthType depth_levels, int uncompressed_data_size = 1, bool compressed = false)
	{
		double box[6];
		packBox(bounding_volume, box);
		return readDataImpl(s, box, resolution, depth_levels, uncompressed_data_size, compressed);
	}

	// castRay (occupancy_map_base.h:449-486), intended semantics (DESIGN.md section 8)
	std::optional<Code> castRay(Point3 origin, Point3 direction, bool ignore_unknown = false, double max_range = -1,
	                            DepthType depth = 0) const
	{
		std::uint64_t code = 0;
		std::uint8_t hit = 0;
		if (UFO_B200_OK != ufo_b200_cast_rays(map_, origin.data(), direction.data(), 1, ignore_unknown, max_range, depth, &code, &hit) || !hit)
			return std::nullopt;
		return Code(code, depth);
	}

	//
	// Integration (occupancy_map_base.h:270-443, occupancy_map_color.h:87-267)
	//
	template <typename T>
	void insertPointCloud(Point3 const& sensor_origin, T const& cloud, double max_range = -1,
	                      DepthType depth = 0, bool simple_ray_casting = false,
	                      unsigned int early_stopping = 0, bool async = false)
	{
		insert(sensor_origin, cloud, max_range, depth, simple_ray_casting, early_stopping, false, async);
	}

	template <typename T>
	void insertPointCloud(Point3 const& sensor_origin, T cloud, ufo::math::Pose6 const& frame_origin,
	                      double max_range = -1, DepthType depth = 0, bool simple_ray_casting = false,
	                      unsigned int early_stopping = 0, bool async = false)
	{
		// the transform is fused into the device-side point read (ufo_b200_insert_pointcloud_frame)
		insert(sensor_origin, cloud, max_range, depth, simple_ray_casting, early_stopping, false, async,
		       &frame_origin);
	}

	template <typename T>
	void insertPointCloudDiscrete(Point3 const& sensor_origin, T const& cloud, double max_range = -1,
	                              DepthType depth = 0, bool simple_ray_casting = false,
	                              unsigned int early_stopping = 0, bool async = false)
	{
		insert(sensor_origin, cloud, max_range, depth, simple_ray_casting, early_stopping, true, async);
	}

	template <typename T>
	void insertPointCloudDiscrete(Point3 const& sensor_origin, T cloud, ufo::math::Pose6 const& frame_origin,
	                              double max_range = -1, DepthType depth = 0,
	                              bool simple_ray_casting = false, unsigned int early_stopping = 0,
	                              bool async = false)
	{
		insert(sensor_origin, cloud, max_range, depth, simple_ray_casting, early_stopping, true, async,
		       &frame_origin);
	}

	bool insertPointCloudDone() const
	{
		int done = 1;
		ufo_b200_done(map_, &done);
		return done != 0;
	}
	void insertPointCloudWait() const { ufo_b200_wait(map_); }

	//
	// Indexing and rays (octree.h:299-496)
	//
	Code toCode(Key const& key) const noexcept { return Code(key); }
	Code toCode(Point3 const& coord, DepthType depth = 0) const noexcept { return Code(toKey(coord, depth)); }
	Code toCode(double x, double y, double z, DepthType depth = 0) const noexcept { return toCode(Point3(x, y, z), depth); }
	Key toKey(Code const& code) const noexcept { return code.toKey(); }
	Key toKey(Point3 const& coord, DepthType depth = 0) const noexcept
	{
		std::uint32_t k[3];
		ufo_b200_to_key(map_, coord.data(), depth, k);
		return Key(k[0], k[1], k[2], depth);
	}
	Key toKey(double x, double y, double z, DepthType depth = 0) const noexcept { return toKey(Point3(x, y, z), depth); }
	Point3 toCoord(Key const& key) const noexcept
	{
		std::uint32_t k[3] = {key[0], key[1], key[2]};
		double p[3];
		ufo_b200_key_to_coord(map_, k, key.getDepth(), p);
		return Point3(p[0], p[1], p[2]);
	}
	Point3 toCoord(Code const& code) const noexcept { return toCoord(code.toKey()); }

	CodeRay computeRay(Point3 const& origin, Point3 const& end, double max_range = -1, DepthType depth = 0) const
	{
		std::size_t n = 0;
		ufo_b200_compute_ray(map_, origin.data(), end.data(), max_range, depth, nullptr, 0, &n);
		std::vector<std::uint64_t> codes(n);
		if (n) ufo_b200_compute_ray(map_, origin.data(), end.data(), max_range, depth, codes.data(), n, &n);
		CodeRay ray;
		ray.reserve(n);
		for (std::uint64_t c : codes) ray.emplace_back(c, depth);
		return ray;
	}

	//
	// Geometry of the tree (octree.h:522-600)
	//
	double getResolution() const noexcept { return params_.resolution; }
	DepthType getTreeDepthLevels() const noexcept { return params_.depth_levels; }
	double getNodeSize(DepthType depth) const { return std::ldexp(params_.resolution, int(depth)); }
	double getNodeHalfSize(DepthType depth) const { return getNodeSize(depth) / 2.0; }
	Point3 getMin() const noexcept
	{
		double h = -getNodeHalfSize(getTreeDepthLevels());
		return Point3(h, h, h);
	}
	Point3 getMax() const noexcept
	{
		double h = getNodeHalfSize(getTreeDepthLevels());
		return Point3(h, h, h);
	}
	bool isInside(Point3 const& p) const
	{
		Point3 lo = getMin(), hi = getMax();
		return lo.x() <= p.x() && hi.x() >= p.x() && lo.y() <= p.y() && hi.y() >= p.y() && lo.z() <= p.z() &&
		       hi.z() >= p.z();
	}

	//
	// State queries (occupancy_map_base.h:599-728) with the intended node semantics
	//
	double getOccupancy(Code const& code) const { return toProb(node(code).logodds); }
	double getOccupancy(Point3 const& coord, DepthType depth = 0) const { return getOccupancy(toCode(coord, depth)); }
	OccupancyState getState(Code const& code) const
	{
		float v = node(code).logodds;
		double const* m = model();
		if (m[0] < v) return OccupancyState::occupied;
		if (m[1] > v) return OccupancyState::free;
		return OccupancyState::unknown;
	}
	OccupancyState getState(Point3 const& coord, DepthType depth = 0) const { return getState(toCode(coord, depth)); }
	bool isOccupied(Code const& code) const { return OccupancyState::occupied == getState(code); }
	bool isFree(Code const& code) const { return OccupancyState::free == getState(code); }
	bool isUnknown(Code const& code) const { return OccupancyState::unknown == getState(code); }
	bool isOccupied(Point3 const& c, DepthType d = 0) const { return isOccupied(toCode(c, d)); }
	bool isFree(Point3 const& c, DepthType d = 0) const { return isFree(toCode(c, d)); }
	bool isUnknown(Point3 const& c, DepthType d = 0) const { return isUnknown(toCode(c, d)); }
	bool containsOccupied(Code const& code) const { return isOccupied(code); }
	bool containsFree(Code const& code) const { return node(code).flags & 1u; }
	bool containsUnknown(Code const& code) const { return node(code).flags & 2u; }

	//
	// Sensor model (occupancy_map_base.h:734-773)
	//
	double getOccupiedThres() const { return toProb(model()[0]); }
	double getFreeThres() const { return toProb(model()[1]); }
	double getProbHit() const { return toProb(model()[2]); }
	double getProbMiss() const { return toProb(model()[3]); }
	double getClampingThresMin() const { return toProb(model()[4]); }
	double getClampingThresMax() const { return toProb(model()[5]); }
	// each setter stores toLogit(p) into ONE parameter; the other stored log-odds stay bit for bit
	// (occupancy_map_base.h:748-773) -- no probability round trip
	void setOccupiedFreeThres(double occupied, double free)
	{
		ufo_b200_set_sensor_model_field(map_, 0, occupied);
		ufo_b200_set_sensor_model_field(map_, 1, free);
	}
	void setProbHit(double p) { ufo_b200_set_sensor_model_field(map_, 2, p); }
	void setProbMiss(double p) { ufo_b200_set_sensor_model_field(map_, 3, p); }
	void setClampingThresMin(double p) { ufo_b200_set_sensor_model_field(map_, 4, p); }
	void setClampingThresMax(double p) { ufo_b200_set_sensor_model_field(map_, 5, p); }

	//
	// Change detection (occupancy_map_base.h:779-790): the nodes whose value changed since the last
	// reset, recorded per voxel on the device and read out at the depth of the last insert (0 for
	// the server's default), unordered like the reference's CodeSet
	//
	using ChangeSet = std::vector<Code>;
	void enableChangeDetection(bool enable) noexcept
	{
		ufo_b200_enable_change_detection(map_, enable);
		change_enabled_ = enable;
	}
	bool isChangeDetectionEnabled() const noexcept { return change_enabled_; }
	void resetChangeDetection() noexcept
	{
		ufo_b200_reset_change_detection(map_);
		changes_.clear();
	}
	std::size_t numChangedDetected() const { return changes().size(); }
	ChangeSet::const_iterator changesBegin() const { return changes().begin(); }
	ChangeSet::const_iterator changesEnd() const { return changes_.end(); }

	//
	// Min/max change detection (occupancy_map_base.h:792-822); always recorded on the device
	//
	void enableMinMaxChangeDetection(bool enable) noexcept
	{
		if (!minmax_enabled_ && enable) resetMinMaxChangeDetection();
		minmax_enabled_ = enable;
	}
	bool isMinMaxChangeDetectionEnabled() const noexcept { return minmax_enabled_; }
	Point3 minChange() const
	{
		double mn[3], mx[3];
		ufo_b200_change_bbox(map_, mn, mx);
		return Point3(mn[0], mn[1], mn[2]);
	}
	Point3 maxChange() const
	{
		double mn[3], mx[3];
		ufo_b200_change_bbox(map_, mn, mx);
		return Point3(mx[0], mx[1], mx[2]);
	}
	void resetMinMaxChangeDetection() noexcept { ufo_b200_reset_change_bbox(map_); }
	bool validMinMaxChange() const
	{
		Point3 a = minChange(), b = maxChange();
		return a.x() <= b.x() && a.y() <= b.y() && a.z() <= b.z();
	}

	void clear() { ufo_b200_clear(map_); }
	// Octree::clear(resolution, depth_levels) octree.h:541-560 (the server's reset service)
	void clear(double new_resolution, DepthType new_depth_levels)
	{
		if (UFO_B200_E_INVALID == ufo_b200_clear_resize(map_, new_resolution, new_depth_levels))
			throw std::invalid_argument("depth_levels has to be [2, 21]");
		// the geometry getters (getResolution, getTreeDepthLevels, getMin/getMax, isInside ...) read params_
		params_.resolution = new_resolution;
		params_.depth_levels = new_depth_levels;
	}

	// status of the last insert (the reference's insert functions are void and never throw)
	int lastStatus() const noexcept { return last_status_; }
	std::string lastError() const { return ufo_b200_last_error(map_); }
	ufo_b200_map* handle() noexcept { return map_; }
	// early_stopping != 0 is rejected (lastStatus() == UFO_B200_E_UNSUPPORTED) unless the map opts in:
	// then the reference's sequential result is computed on the device, at extra cost
	// (ufo_b200_set_early_stopping)
	void setEarlyStoppingExact(bool exact) { last_status_ = ufo_b200_set_early_stopping(map_, exact ? 1 : 0); }

 protected:
	struct NodeValue {
		float logodds;
		std::uint8_t flags;
		std::uint8_t rgb[3];
	};
	NodeValue node(Code const& code) const
	{
		NodeValue v{};
		std::uint64_t c = code.getCode();
		std::uint32_t d = code.getDepth();
		ufo_b200_query(map_, &c, &d, 1, &v.logodds, &v.flags, COLOR ? v.rgb : nullptr);
		return v;
	}
	NNIterator nearest(bool leaves, Point3 const& coord, std::vector<ufo_b200_volume> bv, bool occupied, bool free_space,
	                   bool unknown, bool contains, DepthType min_depth) const
	{
		auto s = std::make_shared<typename NNIterator::State>();
		s->map = this;
		for (int i = 0; i < 3; ++i) s->point[i] = coord[i];
		s->bv = std::move(bv);
		s->leaves = leaves;
		s->occupied = occupied;
		s->free_space = free_space;
		s->unknown = unknown;
		s->contains = contains;
		s->min_depth = min_depth;
		s->levels = getTreeDepthLevels();
		for (DepthType d = 0; d < 22; ++d) s->half_size[d] = getNodeHalfSize(d);
		s->occupied_thres_log = model()[0];
		s->free_thres_log = model()[1];
		return NNIterator(std::move(s));
	}
	Iterator iterate(bool leaves, std::vector<ufo_b200_volume> const& bv, bool occupied, bool free_space, bool unknown,
	                 bool contains, DepthType min_depth) const
	{
		auto s = std::make_shared<typename Iterator::Snapshot>();
		auto call = [&](std::size_t cap, std::size_t* n) {
			return ufo_b200_iterate(map_, leaves, occupied, free_space, unknown, contains, min_depth, bv.data(), bv.size(),
			                        cap ? s->codes.data() : nullptr, cap ? s->depths.data() : nullptr,
			                        cap ? s->logodds.data() : nullptr, cap ? s->flags.data() : nullptr,
			                        cap && COLOR ? s->rgb.data() : nullptr, cap, n);
		};
		std::size_t n = 0;
		if (UFO_B200_OK != call(0, &n) || 0 == n) return Iterator();
		s->codes.resize(n);
		s->depths.resize(n);
		s->logodds.resize(n);
		s->flags.resize(n);
		if (COLOR) s->rgb.resize(3 * n);
		if (UFO_B200_OK != call(n, &n) || n != s->codes.size()) return Iterator();
		s->levels = getTreeDepthLevels();
		for (DepthType d = 0; d < 22; ++d) s->half_size[d] = getNodeHalfSize(d);
		s->occupied_thres_log = model()[0];
		s->free_thres_log = model()[1];
		return Iterator(std::move(s));
	}
	// occupancy_map_base.h:911 -- LogitType is float there: the argument narrows to float and the
	// exponential is the float one, for the sensor-model getters as well as for getOccupancy
	static double toProb(float logit) { return 1.0 / (1.0 + std::exp(-logit)); }
	// occupancy_map_base.h:909: in double; the callers narrow to float (LogitType)
	static double toLogit(double prob) { return std::log(prob / (1.0 - prob)); }
	void writeNode(Code const& code, std::uint8_t op, float value)
	{
		std::uint64_t c = code.getCode();
		std::uint32_t d = code.getDepth();
		last_status_ = ufo_b200_update_nodes(map_, &c, &d, &op, &value, 1, 0);
	}
	double const* model() const
	{
		ufo_b200_sensor_model_logit(map_, model_);
		return model_;
	}
	ufo_b200_tree_stats treeStats() const
	{
		ufo_b200_tree_stats t{};
		if (UFO_B200_OK != ufo_b200_tree_info(map_, &t)) throw std::runtime_error("ufomap_b200: " + lastError());
		return t;
	}
	static ufo_b200_map* copyOf(MapFacade const& other)
	{
		ufo_b200_map* m = nullptr;
		if (UFO_B200_OK != ufo_b200_clone(other.map_, &m))
			throw std::runtime_error("ufomap_b200: the map could not be copied on its device: " + other.lastError());
		const double p[6] = {other.getOccupiedThres(), other.getFreeThres(),         other.getProbHit(),
		                     other.getProbMiss(),      other.getClampingThresMin(), other.getClampingThresMax()};
		// one call for all six: the flags are rebuilt once
		if (UFO_B200_OK != ufo_b200_set_sensor_model(m, p)) {
			const std::string why = ufo_b200_last_error(m);
			ufo_b200_destroy(m);
			throw std::runtime_error("ufomap_b200: the copy's sensor model could not be set: " + why);
		}
		return m;
	}

	template <typename T>
	void insert(Point3 const& origin, T const& cloud, double max_range, DepthType depth, bool simple,
	            unsigned int early_stopping, bool discrete, bool async,
	            ufo::math::Pose6 const* frame = nullptr)
	{
		using P = std::decay_t<decltype(cloud[0])>;
		change_depth_ = depth;
		double pose[7];
		if (frame) frame->pack(pose);
		constexpr bool has_color = std::is_base_of_v<Point3Color, P>;
		// repack into the C-ABI layout (the reference takes the cloud by value, i.e. copies it too)
		std::size_t n = cloud.size();
		if constexpr (has_color) {
			struct Rec {
				double x, y, z;
				std::uint8_t r, g, b, pad[5];
			};
			static_assert(sizeof(Rec) == 32);
			std::vector<Rec> buf(n);
			for (std::size_t i = 0; i < n; ++i) {
				P const& p = cloud[i];
				buf[i] = Rec{p.x(), p.y(), p.z(), p.getColor().r, p.getColor().g, p.getColor().b, {0, 0, 0, 0, 0}};
			}
			last_status_ =
			    frame ? ufo_b200_insert_pointcloud_frame(map_, origin.data(), buf.data(), n, UFO_B200_XYZRGB_F64,
			                                             pose, max_range, depth, simple, early_stopping,
			                                             discrete, async)
			          : ufo_b200_insert_pointcloud(map_, origin.data(), buf.data(), n, UFO_B200_XYZRGB_F64,
			                                       max_range, depth, simple, early_stopping, discrete, async);
		} else {
			std::vector<double> buf(3 * n);
			for (std::size_t i = 0; i < n; ++i) {
				buf[3 * i] = cloud[i].x();
				buf[3 * i + 1] = cloud[i].y();
				buf[3 * i + 2] = cloud[i].z();
			}
			last_status_ =
			    frame ? ufo_b200_insert_pointcloud_frame(map_, origin.data(), buf.data(), n, UFO_B200_XYZ_F64,
			                                             pose, max_range, depth, simple, early_stopping,
			                                             discrete, async)
			          : ufo_b200_insert_pointcloud(map_, origin.data(), buf.data(), n, UFO_B200_XYZ_F64,
			                                       max_range, depth, simple, early_stopping, discrete, async);
		}
	}

	static void packBox(ufo::geometry::AABB const& b, double box[6])
	{
		box[0] = b.center.x();
		box[1] = b.center.y();
		box[2] = b.center.z();
		box[3] = b.half_size.x();
		box[4] = b.half_size.y();
		box[5] = b.half_size.z();
	}
	// compressed stream (data_only) or file image; returns the UNCOMPRESSED data size like the
	// reference's writeData, -1 on error
	int writeCompressed(std::ostream& s, double const* box, bool data_only, DepthType min_depth, int accel, int level) const
	{
		std::size_t n = 0, u = 0;
		if (UFO_B200_OK != ufo_b200_write_compressed(map_, box, min_depth, data_only, accel, level, nullptr, 0, &n, &u)) return -1;
		std::vector<char> data(n ? n : 1);
		if (UFO_B200_OK != ufo_b200_write_compressed(map_, box, min_depth, data_only, accel, level, data.data(), n, &n, &u)) return -1;
		s.write(data.data(), (std::streamsize)n);
		return s.good() ? (int)u : -1;
	}
	std::vector<std::uint8_t> pageOutRecords(std::vector<ufo_b200_volume> const& bv)
	{
		std::size_t n = 0;
		std::vector<std::uint8_t> blob;
		last_status_ = ufo_b200_page_out_bv(map_, bv.data(), bv.size(), nullptr, 0, &n);
		if (UFO_B200_OK != last_status_) return blob;
		blob.resize(n);
		last_status_ = ufo_b200_page_out_bv(map_, bv.data(), bv.size(), blob.data(), n, &n);
		if (UFO_B200_OK != last_status_) blob.clear();
		return blob;
	}
	int writeCompressedBv(std::ostream& s, std::vector<ufo_b200_volume> const& bv, bool data_only, DepthType min_depth,
	                      int accel, int level) const
	{
		std::size_t n = 0, u = 0;
		if (UFO_B200_OK != ufo_b200_write_compressed_bv(map_, bv.data(), bv.size(), min_depth, data_only, accel, level, nullptr,
		                                                0, &n, &u))
			return -1;
		std::vector<char> data(n ? n : 1);
		if (UFO_B200_OK != ufo_b200_write_compressed_bv(map_, bv.data(), bv.size(), min_depth, data_only, accel, level,
		                                                data.data(), n, &n, &u))
			return -1;
		s.write(data.data(), (std::streamsize)n);
		return s.good() ? (int)u : -1;
	}
	bool readDataImpl(std::istream& s, double const* box, double resolution, DepthType depth_levels, int uncompressed_data_size,
	                  bool compressed)
	{
		if (getResolution() != resolution || getTreeDepthLevels() != depth_levels) clear(resolution, depth_levels);
		std::vector<char> data((std::istreambuf_iterator<char>(s)), std::istreambuf_iterator<char>());
		return UFO_B200_OK == ufo_b200_read_data(map_, box, data.data(), data.size(), compressed,
		                                         compressed ? (std::size_t)uncompressed_data_size : 0);
	}
	int writeDataImpl(std::ostream& s, double const* box, bool compress, DepthType min_depth) const
	{
		if (compress) return -1;
		std::size_t n = 0;
		if (UFO_B200_OK != ufo_b200_write_data(map_, box, min_depth, nullptr, 0, &n)) return -1;
		std::vector<char> data(n ? n : 1);
		if (UFO_B200_OK != ufo_b200_write_data(map_, box, min_depth, data.data(), n, &n)) return -1;
		s.write(data.data(), (std::streamsize)n);
		return s.good() ? (int)n : -1;
	}

	ChangeSet const& changes() const
	{
		std::size_t n = 0;
		ufo_b200_changed_codes(map_, change_depth_, nullptr, 0, &n);
		std::vector<std::uint64_t> raw(n ? n : 1);
		ufo_b200_changed_codes(map_, change_depth_, raw.data(), n, &n);
		changes_.clear();
		changes_.reserve(n);
		for (std::size_t i = 0; i < n; ++i) changes_.emplace_back(raw[i], change_depth_);
		return changes_;
	}

	ufo_b200_map* map_ = nullptr;
	mutable ChangeSet changes_;
	bool change_enabled_ = false;
	DepthType change_depth_ = 0;
	ufo_b200_params params_{};
	mutable double model_[6] = {0, 0, 0, 0, 0, 0};
	bool minmax_enabled_ = false;
	mutable int last_status_ = 0;  // mutable: a nearest-first iterator reports a map changed under it
};
}  // namespace detail

class OccupancyMap : public detail::MapFacade<false>
{
 public:
	using detail::MapFacade<false>::MapFacade;
};

class OccupancyMapColor : public detail::MapFacade<true>
{
 public:
	using detail::MapFacade<true>::MapFacade;

	// occupancy_map_color.h:269-287 and :304-314.  Each call is a batch of one on the device
	// (ufo_b200_update_nodes_color) at depth 0 only; the status is left in lastStatus().
	void updateValue(Code const& code, float update, Color color) { writeColorNode(code, 2, update, color); }
	void setColor(Code const& code, Color color) { writeColorNode(code, 3, 0.0f, color); }
	void setColor(Point3 const& coord, Color color, DepthType depth = 0) { setColor(toCode(coord, depth), color); }
	void setColor(double x, double y, double z, Color color, DepthType depth = 0)
	{
		setColor(toCode(x, y, z, depth), color);
	}

	// occupancy_map_color.h:320-330
	Color getColor(Code const& code) const
	{
		NodeValue v = node(code);
		return Color(v.rgb[0], v.rgb[1], v.rgb[2]);
	}
	Color getColor(Point3 const& coord, DepthType depth = 0) const { return getColor(toCode(coord, depth)); }
	Color getColor(double x, double y, double z, DepthType depth = 0) const { return getColor(toCode(x, y, z, depth)); }

 private:
	void writeColorNode(Code const& code, std::uint8_t op, float value, Color color)
	{
		std::uint64_t c = code.getCode();
		std::uint32_t d = code.getDepth();
		const std::uint8_t rgb[3] = {color.r, color.g, color.b};
		last_status_ = ufo_b200_update_nodes_color(map_, &c, &d, &op, &value, rgb, 1, 0);
	}
};
}  // namespace ufo::map
