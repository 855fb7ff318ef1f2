// The mapping server's get_map, clear_volume and save_map service bodies (server.cpp:327-390), without
// ROS, against the facade: the request's bounding volume is built the way msgToUfo builds it
// (ufomap_msgs/conversions.cpp:46-124) and the map calls are the server's own.  Built and run by
// tests/test_facade_volumes.py.
#include <ufo/geometry/bounding_volume.h>
#include <ufo/geometry/frustum.h>
#include <ufo/geometry/line_segment.h>
#include <ufo/geometry/obb.h>
#include <ufo/geometry/plane.h>
#include <ufo/geometry/ray.h>
#include <ufo/geometry/sphere.h>
#include <ufo/geometry/types.h>
#include <ufo/map/occupancy_map.h>
#include <ufo/map/occupancy_map_color.h>

#include <cstdio>
#include <cstring>
#include <sstream>
#include <string>
#include <type_traits>
#include <variant>

using namespace ufo::map;
namespace geo = ufo::geometry;

struct Request {
	geo::BoundingVolume bounding_volume;
	bool compress = false;
	unsigned depth = 0;
	std::string filename;
	int compression_level = 0;
};
struct Response {
	bool success = false;
	std::string data;
	int uncompressed_data_size = 0;
};

// what ufoToMsg does with the map (ufomap_msgs/conversions.h:161-185), the message left out
template <class TreeType>
bool ufoToMsg(TreeType const& tree, Response& msg, geo::BoundingVolume const& bounding_volume, bool compress = false,
              unsigned depth = 0, int compression_acceleration_level = 1, int compression_level = 0)
{
	std::stringstream data_stream(std::ios_base::in | std::ios_base::out | std::ios_base::binary);
	msg.uncompressed_data_size =
	    tree.writeData(data_stream, bounding_volume, compress, depth, compression_acceleration_level, compression_level);
	if (0 > msg.uncompressed_data_size) return false;
	msg.data = data_stream.str();
	return true;
}

struct Server {
	std::variant<std::monostate, OccupancyMap, OccupancyMapColor> map_;

	// server.cpp:327-343
	bool getMapCallback(Request& request, Response& response)
	{
		std::visit(
		    [this, &request, &response](auto& map) {
			    if constexpr (!std::is_same_v<std::decay_t<decltype(map)>, std::monostate>) {
				    geo::BoundingVolume bv = request.bounding_volume;
				    response.success = ufoToMsg(map, response, bv, request.compress, request.depth);
			    } else {
				    response.success = false;
			    }
		    },
		    map_);
		return true;
	}

	// server.cpp:345-363
	bool clearVolumeCallback(Request& request, Response& response)
	{
		std::visit(
		    [this, &request, &response](auto& map) {
			    if constexpr (!std::is_same_v<std::decay_t<decltype(map)>, std::monostate>) {
				    geo::BoundingVolume bv = request.bounding_volume;
				    for (auto& b : bv) {
					    map.setValueVolume(b, map.getClampingThresMin(), request.depth);
				    }
				    response.success = true;
			    } else {
				    response.success = false;
			    }
		    },
		    map_);
		return true;
	}

	// server.cpp:381-397
	bool saveMapCallback(Request& request, Response& response)
	{
		std::visit(
		    [this, &request, &response](auto& map) {
			    if constexpr (!std::is_same_v<std::decay_t<decltype(map)>, std::monostate>) {
				    geo::BoundingVolume bv = request.bounding_volume;
				    response.success =
				        map.write(request.filename, bv, request.compress, request.depth, 1, request.compression_level);
			    } else {
				    response.success = false;
			    }
		    },
		    map_);
		return true;
	}
};

// msgToUfo's constructors (conversions.cpp:46-92)
static geo::BoundingVolume every_shape(geo::Point c)
{
	geo::BoundingVolume bv;
	geo::AABB a;
	a.center = c;
	a.half_size = geo::Point(0.2, 0.3, 0.1);
	bv.add(a);
	bv.add(geo::Frustum(c - geo::Point(1, 0, 0), c, geo::Point(0, 0, 1), 0.8, 1.0, 0.1, 2.0));
	bv.add(geo::LineSegment(c, c + geo::Point(0.5, 0.2, 0.1)));
	bv.add(geo::OBB(c, geo::Point(0.3, 0.1, 0.2), geo::Point(0.1, 0.2, 0.3)));
	bv.add(geo::Plane(geo::Point(0, 0, 1), c.z()));
	bv.add(c);
	bv.add(geo::Ray(c, geo::Point(1, 1, 0)));
	bv.add(geo::Sphere(c, 0.25));
	return bv;
}

static void print_doubles(char const* name, double const* v, int n)
{
	std::printf("%s", name);
	for (int i = 0; i < n; ++i) {
		std::uint64_t u;
		std::memcpy(&u, v + i, 8);
		std::printf(" %016llx", (unsigned long long)u);
	}
	std::printf("\n");
}

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) {
		// the constructors' doubles (compared with the reference's by the test)
		geo::Frustum f(geo::Point(0.5, -1, 0.25), geo::Point(0.5, 2, 0.25), geo::Point(0, 0, 1), 0.7, 1.1, 0.1, 3.0);
		double fp[24];
		for (int i = 0; i < 6; ++i) {
			for (int k = 0; k < 3; ++k) fp[4 * i + k] = f.planes[i].normal[k];
			fp[4 * i + 3] = f.planes[i].distance;
		}
		print_doubles("frustum", fp, 24);
		geo::Plane p(geo::Point(0.1, 0.2, 0.3), geo::Point(1.3, -0.2, 0.7), geo::Point(-0.4, 0.9, 1.1));
		double pp[4] = {p.normal[0], p.normal[1], p.normal[2], p.distance};
		print_doubles("plane", pp, 4);
		geo::Ray r(geo::Point(0.1, 0.2, 0.3), geo::Point(0.3, -0.7, 2.9));
		double rp[6] = {r.origin[0], r.origin[1], r.origin[2], r.direction[0], r.direction[1], r.direction[2]};
		print_doubles("ray", rp, 6);
		geo::OBB o(geo::Point(0, 0, 0), geo::Point(1, 1, 1), geo::Point(0.3, -0.2, 1.1));
		double op[4] = {o.rotation.w(), o.rotation.x(), o.rotation.y(), o.rotation.z()};
		print_doubles("obb", op, 4);
		// rejections before any device work (a geometry-only handle has no device)
		ufo_b200_params prm;
		ufo_b200_default_params(&prm);
		prm.device = -2;
		ufo_b200_map* h = nullptr;
		if (ufo_b200_create(&prm, &h) != UFO_B200_OK) return 2;
		ufo_b200_volume bad{};
		bad.type = 8;
		if (ufo_b200_set_value_volume_bv(h, &bad, 0.2, 0) != UFO_B200_E_INVALID) return 3;
		ufo_b200_volume s = geo::toRecord(geo::Sphere(geo::Point(0, 0, 0), 1.0));
		if (ufo_b200_set_value_volume_bv(h, &s, 0.2, 5) != UFO_B200_E_UNSUPPORTED) return 4;
		std::size_t n = 0;
		if (ufo_b200_write_data_bv(h, &bad, 1, 0, nullptr, 0, &n) != UFO_B200_E_INVALID) return 5;
		ufo_b200_destroy(h);
		std::puts("facade volumes ok (no device)");
		return 0;
	}

	Server srv;
	auto& map = srv.map_.emplace<OccupancyMap>(0.05);
	geo::Point c(0.52, -0.31, 0.18);
	for (int i = 0; i < 5; ++i) map.setOccupancy(c + geo::Point(0.05 * i, 0, 0), 0.9);
	if (map.lastStatus() != UFO_B200_OK) return 10;

	Request req;
	Response res;
	// get_map: the whole map, a volume around the voxels, a volume that misses the map
	srv.getMapCallback(req, res);
	std::string const whole = res.data;
	if (!res.success || whole.empty()) return 11;
	req.bounding_volume = every_shape(c);
	srv.getMapCallback(req, res);
	if (!res.success || res.data.empty() || res.data.size() > whole.size()) return 12;
	std::string const part = res.data;
	Request far_req;
	far_req.bounding_volume.add(geo::Sphere(geo::Point(1e6, 1e6, 1e6), 1.0));
	srv.getMapCallback(far_req, res);
	if (!res.success || !res.data.empty()) return 13;
	// msgToUfo on the other side: the partial stream read back with its volume gives the voxels
	OccupancyMap back(0.05);
	std::stringstream in(part, std::ios_base::in | std::ios_base::binary);
	if (!back.readData(in, req.bounding_volume, 0.05, 16)) return 14;
	if (!back.isOccupied(c)) return 15;

	// save_map with the volume: a UFOMap file
	req.filename = argc > 1 ? argv[1] : "facade_volumes.ufo";
	srv.saveMapCallback(req, res);
	if (!res.success) return 16;
	std::FILE* fp = std::fopen(req.filename.c_str(), "rb");
	if (!fp) return 17;
	char head[13] = {0};
	std::size_t got = std::fread(head, 1, 12, fp);
	std::fclose(fp);
	if (got != 12 || std::strncmp(head, "# UFOMap file", 12) != 0) return 18;

	// clear_volume: a sphere around the first voxel clears it to the lower clamp (free), the others
	// outside it stay occupied; a depth the device does not support is refused
	Request clr;
	clr.bounding_volume.add(geo::Sphere(c, 0.02));
	srv.clearVolumeCallback(clr, res);
	if (!res.success || map.lastStatus() != UFO_B200_OK) return 19;
	if (!map.isFree(c) || !map.isOccupied(c + geo::Point(0.15, 0, 0))) return 20;
	clr.depth = 5;
	srv.clearVolumeCallback(clr, res);
	if (map.lastStatus() != UFO_B200_E_UNSUPPORTED) return 21;
	std::puts("facade volumes ok");
	return 0;
}
