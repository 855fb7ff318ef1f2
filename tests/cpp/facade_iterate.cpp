// The RViz plugin's map loop (ufomap_rviz_plugins/src/ufomap_display.cpp:267-303) against the facade,
// written as the plugin writes it; the Qt / Ogre / rviz types are replaced by plain structs of the
// same shape.  Built and run by tests/test_facade_iterate.py.
//
//   facade_iterate --no-device       the loop compiles for both map types; argument checks of
//                                    ufo_b200_iterate that need no device
//   facade_iterate DATA RES DEPTH_LEVELS COLOR MIN_DEPTH OCC FREE UNK MINX MINY MINZ MAXX MAXY MAXZ
//                                    reads the node stream DATA (writeData) into a map, runs the loop
//                                    over the box and prints one line per node and the per-type extents
#include <ufo/map/occupancy_map.h>
#include <ufo/map/occupancy_map_color.h>

#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <type_traits>
#include <vector>

namespace
{
enum VoxelType { OCCUPIED, FREE, UNKNOWN };

// rviz::PointCloud::Point
struct RvizPoint {
	double r = 0, g = 0, b = 0, a = 0;
	void setColor(double r_, double g_, double b_, double a_)
	{
		r = r_;
		g = g_;
		b = b_;
		a = a_;
	}
};

std::uint64_t bits(double d)
{
	std::uint64_t u;
	std::memcpy(&u, &d, 8);
	return u;
}

// what the plugin's addPoint receives, printed bit for bit
void addPoint(VoxelType type, int min_depth, RvizPoint const& point, double occupancy, unsigned depth,
              ufo::geometry::AABB const& box)
{
	auto mn = box.getMin(), mx = box.getMax();
	std::printf("node %d %d %u %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64
	            " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 "\n",
	            (int)type, min_depth, depth, bits(occupancy), bits(mn[0]), bits(mn[1]), bits(mn[2]), bits(mx[0]), bits(mx[1]),
	            bits(mx[2]), bits(point.r), bits(point.g), bits(point.b), bits(point.a));
}

template <typename T>
void renderMap(T const& map, ufo::map::Point3 min_value, ufo::map::Point3 max_value, int min_depth, bool occupied, bool free,
               bool unknown)
{
	std::map<VoxelType, ufo::map::Point3> min_coord;
	std::map<VoxelType, ufo::map::Point3> max_coord;

	ufo::geometry::AABB aabb_bbx(min_value, max_value);
	for (auto it = map.beginLeaves(aabb_bbx, occupied, free, unknown, false, min_depth), end = map.endLeaves(); it != end;
	     ++it) {
		VoxelType type;
		if (it.isOccupied()) {
			type = OCCUPIED;
		} else if (it.isFree()) {
			type = FREE;
		} else {
			type = UNKNOWN;
		}

		ufo::geometry::AABB it_aabb = it.getBoundingVolume();
		ufo::map::Point3 it_min = it_aabb.getMin();
		ufo::map::Point3 it_max = it_aabb.getMax();

		if (min_coord.count(type)) {
			for (int i : {0, 1, 2}) {
				min_coord[type][i] = std::min(min_coord[type][i], it_min[i]);
				max_coord[type][i] = std::max(max_coord[type][i], it_max[i]);
			}
		} else {
			min_coord[type] = it_min;
			max_coord[type] = it_max;
		}

		RvizPoint point;
		if constexpr (std::is_same_v<T, ufo::map::OccupancyMapColor>) {
			point.setColor(it->color.r / 255.0, it->color.g / 255.0, it->color.b / 255.0, it.getOccupancy());
		}

		addPoint(type, min_depth, point, it.getOccupancy(), it.getDepth(), it.getBoundingVolume());
	}
	for (auto const& [type, mn] : min_coord) {
		auto const& mx = max_coord[type];
		std::printf("extent %d %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 "\n",
		            (int)type, bits(mn[0]), bits(mn[1]), bits(mn[2]), bits(mx[0]), bits(mx[1]), bits(mx[2]));
	}
}

int fail(const char* what)
{
	std::printf("FAILED: %s\n", what);
	return 1;
}

int noDevice()
{
	// the loop instantiates for both map types (never called here: creating a map needs a device)
	void (*mono)(ufo::map::OccupancyMap const&, ufo::map::Point3, ufo::map::Point3, int, bool, bool, bool) =
	    &renderMap<ufo::map::OccupancyMap>;
	void (*color)(ufo::map::OccupancyMapColor const&, ufo::map::Point3, ufo::map::Point3, int, bool, bool, bool) =
	    &renderMap<ufo::map::OccupancyMapColor>;
	if (!mono || !color) return fail("instantiation");
	// end iterators compare equal; a default iterator is an end iterator
	ufo::map::OccupancyMap::Iterator a, b;
	if (!(a == b) || a != b) return fail("end == end");

	ufo_b200_params p;
	ufo_b200_default_params(&p);
	p.device = -2;  // geometry-only handle
	ufo_b200_map* m = nullptr;
	if (UFO_B200_OK != ufo_b200_create(&p, &m)) return fail("geometry-only handle");
	std::size_t n = 7;
	std::uint64_t codes[1];
	std::uint8_t depths[1], flags[1];
	float occ[1];
	ufo_b200_volume bad{};
	bad.type = 99;
	if (UFO_B200_E_INVALID != ufo_b200_iterate(nullptr, 1, 1, 1, 0, 0, 0, nullptr, 0, nullptr, nullptr, nullptr, nullptr,
	                                           nullptr, 0, &n))
		return fail("NULL map");
	if (UFO_B200_E_INVALID != ufo_b200_iterate(m, 1, 1, 1, 0, 0, 0, nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
	                                           nullptr))
		return fail("NULL count");
	if (UFO_B200_E_INVALID != ufo_b200_iterate(m, 1, 1, 1, 0, 0, 0, &bad, 1, nullptr, nullptr, nullptr, nullptr, nullptr, 0, &n))
		return fail("unknown volume type");
	if (UFO_B200_E_INVALID != ufo_b200_iterate(m, 1, 1, 1, 0, 0, 0, nullptr, 1, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
	                                           &n))
		return fail("NULL volume with n_bv > 0");
	if (UFO_B200_E_INVALID != ufo_b200_iterate(m, 1, 1, 1, 0, 0, 0, nullptr, 0, codes, nullptr, occ, flags, nullptr, 1, &n))
		return fail("cap > 0 without arrays");
	if (UFO_B200_E_CUDA != ufo_b200_iterate(m, 1, 1, 1, 0, 0, 0, nullptr, 0, codes, depths, occ, flags, nullptr, 1, &n) ||
	    n != 0)
		return fail("geometry-only handle must refuse");
	ufo_b200_destroy(m);
	std::printf("facade iterate ok (no device)\n");
	return 0;
}
}  // namespace

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) return noDevice();
	if (argc != 15) return fail("usage");
	double res = std::atof(argv[2]);
	unsigned levels = (unsigned)std::atoi(argv[3]);
	bool color = std::atoi(argv[4]) != 0;
	int min_depth = std::atoi(argv[5]);
	bool occ = std::atoi(argv[6]) != 0, fre = std::atoi(argv[7]) != 0, unk = std::atoi(argv[8]) != 0;
	ufo::map::Point3 mn(std::atof(argv[9]), std::atof(argv[10]), std::atof(argv[11]));
	ufo::map::Point3 mx(std::atof(argv[12]), std::atof(argv[13]), std::atof(argv[14]));
	auto run = [&](auto& map) {
		std::ifstream f(argv[1], std::ios_base::in | std::ios_base::binary);
		if (!f.is_open() || !map.readData(f, res, levels)) return fail("readData");
		// the plugin clamps its box to the map (ufomap_display.cpp:244-260)
		ufo::map::Point3 lo = map.getMin(), hi = map.getMax();
		for (int i = 0; i < 3; ++i) {
			lo[i] = std::max(lo[i], mn[i]);
			hi[i] = std::min(hi[i], mx[i]);
		}
		renderMap(map, lo, hi, min_depth, occ, fre, unk);
		std::printf("facade iterate ok\n");
		return 0;
	};
	if (color) {
		ufo::map::OccupancyMapColor map(res, levels);
		return run(map);
	}
	ufo::map::OccupancyMap map(res, levels);
	return run(map);
}
