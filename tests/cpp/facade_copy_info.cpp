// Copies of facade maps and the RViz plugin's updateInfo call (ufomap_rviz_plugins/src/ufomap_display.cpp:
// 508-516) against the facade, written as a caller writes them.  Built and run by
// tests/test_facade_copy_info.py.
//
//   facade_copy_info --no-device     everything compiles for both map types; argument checks of
//                                    ufo_b200_clone / ufo_b200_tree_info that need no device
//   facade_copy_info DATA RES DEPTH_LEVELS COLOR
//                                    reads the node stream DATA (writeData) into a map held in a
//                                    std::variant, copies it four ways and prints one "info" line per map
#include <ufo/map/occupancy_map.h>
#include <ufo/map/occupancy_map_color.h>

#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <type_traits>
#include <variant>

namespace
{
using MapVariant = std::variant<std::monostate, ufo::map::OccupancyMap, ufo::map::OccupancyMapColor>;

int fail(char const* what)
{
	std::printf("FAIL %s\n", what);
	return 1;
}

std::uint64_t bits(double d)
{
	std::uint64_t u;
	std::memcpy(&u, &d, 8);
	return u;
}

// the plugin's info panel (UFOMapDisplay::updateInfo)
void updateInfo(double resolution, std::size_t num_leaf_nodes, std::size_t num_inner_nodes, std::size_t memory_usage)
{
	std::printf("updateInfo %016" PRIx64 " %zu %zu %zu\n", bits(resolution), num_leaf_nodes, num_inner_nodes, memory_usage);
}

template <typename T>
void printInfo(char const* name, T const& map)
{
	const ufo::geometry::AABB b = map.getKnownBBX();
	std::printf("info %s %zu %zu %zu %zu", name, map.getNumLeafNodes(), map.getNumInnerNodes(), map.size(), map.memoryUsage());
	for (int i = 0; i < 3; ++i) std::printf(" %016" PRIx64, bits(b.center[i]));
	for (int i = 0; i < 3; ++i) std::printf(" %016" PRIx64, bits(b.half_size[i]));
	// the stored log-odds of the sensor model
	double o[6];
	ufo_b200_sensor_model_logit(const_cast<T&>(map).handle(), o);
	for (double x : o) std::printf(" %016" PRIx64, bits(x));
	std::printf("\n");
}

// a function that takes a map by value
template <typename T>
void byValue(T map)
{
	printInfo("by_value", map);
}

int noDevice()
{
	static_assert(std::is_copy_constructible_v<ufo::map::OccupancyMap>);
	static_assert(std::is_copy_constructible_v<ufo::map::OccupancyMapColor>);
	static_assert(std::is_copy_assignable_v<ufo::map::OccupancyMap>);
	static_assert(std::is_copy_assignable_v<ufo::map::OccupancyMapColor>);
	static_assert(std::is_copy_constructible_v<MapVariant> && std::is_copy_assignable_v<MapVariant>);
	ufo_b200_params p;
	ufo_b200_default_params(&p);
	p.device = -2;  // geometry-only handle
	ufo_b200_map* m = nullptr;
	if (UFO_B200_OK != ufo_b200_create(&p, &m)) return fail("geometry-only handle");
	ufo_b200_map* c = reinterpret_cast<ufo_b200_map*>(&p);
	ufo_b200_tree_stats t{};
	if (UFO_B200_E_INVALID != ufo_b200_clone(nullptr, &c) || c) return fail("NULL source");
	if (UFO_B200_E_INVALID != ufo_b200_clone(m, nullptr)) return fail("NULL out");
	if (UFO_B200_E_CUDA != ufo_b200_clone(m, &c) || c) return fail("geometry-only handle must refuse the copy");
	if (UFO_B200_E_INVALID != ufo_b200_tree_info(nullptr, &t)) return fail("NULL map");
	if (UFO_B200_E_INVALID != ufo_b200_tree_info(m, nullptr)) return fail("NULL stats");
	if (UFO_B200_E_CUDA != ufo_b200_tree_info(m, &t)) return fail("geometry-only handle must refuse the counters");
	ufo_b200_destroy(m);
	std::printf("facade copy info ok (no device)\n");
	return 0;
}
}  // namespace

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) return noDevice();
	if (argc != 5) return fail("usage");
	double res = std::atof(argv[2]);
	unsigned levels = (unsigned)std::atoi(argv[3]);
	bool color = std::atoi(argv[4]) != 0;
	MapVariant map_;
	if (color) map_.emplace<ufo::map::OccupancyMapColor>(res, levels);
	else map_.emplace<ufo::map::OccupancyMap>(res, levels);
	bool ok = std::visit(
	    [&](auto& map) -> bool {
		    if constexpr (!std::is_same_v<std::decay_t<decltype(map)>, std::monostate>) {
			    std::ifstream f(argv[1], std::ios_base::in | std::ios_base::binary);
			    if (!f.is_open() || !map.readData(f, res, levels)) return false;
			    // a sensor model whose probability round trip is not exact in every bit
			    map.setProbHit(0.7123456789);
			    // ufomap_display.cpp:512-513, line for line
			    updateInfo(map.getResolution(), map.getNumLeafNodes(),
			               map.getNumInnerNodes(), map.memoryUsage());
			    return true;
		    }
		    return false;
	    },
	    map_);
	if (!ok) return fail("readData");
	MapVariant copied = map_;  // the variant's copy constructor
	MapVariant assigned;
	assigned = map_;  // the variant's copy assignment
	return std::visit(
	    [&](auto& map) -> int {
		    using M = std::decay_t<decltype(map)>;
		    if constexpr (std::is_same_v<M, std::monostate>) {
			    return fail("empty variant");
		    } else {
			    printInfo("source", map);
			    printInfo("variant_copy", std::get<M>(copied));
			    printInfo("variant_assign", std::get<M>(assigned));
			    auto snapshot = map;
			    printInfo("snapshot", snapshot);
			    M target(res, levels);
			    target = map;
			    printInfo("assigned", target);
			    byValue(map);
			    // a change to a copy leaves the source as it was
			    ufo::map::PointCloud cloud;
			    cloud.push_back(ufo::map::Point3(1.0, 0.5, 0.25));
			    snapshot.insertPointCloud(ufo::map::Point3(0, 0, 0), cloud);
			    printInfo("snapshot_after", snapshot);
			    printInfo("source_after", map);
			    std::printf("facade copy info ok\n");
			    return 0;
		    }
	    },
	    map_);
}
