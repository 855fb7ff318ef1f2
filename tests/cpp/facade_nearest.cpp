// A planner's nearest-occupied query and the six nearest-first overloads against the facade.  Built and
// run by tests/test_facade_nearest.py.
//
//   facade_nearest --no-device   the loops compile for both map types; argument checks of
//                                ufo_b200_nearest that need no device
//   facade_nearest DATA RES DEPTH_LEVELS COLOR PX PY PZ
//                                reads the node stream DATA (writeData) into a map and prints, per
//                                overload, one line per node; then the planner loop's distance and a
//                                map changed in the middle of an iteration
#include <ufo/map/occupancy_map.h>
#include <ufo/map/occupancy_map_color.h>

#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <type_traits>

namespace
{
namespace geo = ufo::geometry;

std::uint64_t bits(double d)
{
	std::uint64_t u;
	std::memcpy(&u, &d, 8);
	return u;
}

std::uint32_t fbits(float f)
{
	std::uint32_t u;
	std::memcpy(&u, &f, 4);
	return u;
}

int fail(const char* what)
{
	std::printf("FAILED: %s\n", what);
	return 1;
}

// one line per node: overload, code, depth, log-odds bits, colour, isLeaf / contains flags, d2 bits,
// and the AABB's min and max bits
template <typename It>
void dump(const char* name, It it, It end)
{
	for (; it != end; ++it) {
		unsigned r = 0, g = 0, b = 0;
		if constexpr (std::is_same_v<std::decay_t<decltype(*it)>, ufo::map::ColorOccupancyValue>) {
			r = it->color.r;
			g = it->color.g;
			b = it->color.b;
		}
		const unsigned fl = (it.containsFree() ? 1u : 0u) | (it.containsUnknown() ? 2u : 0u) | (it.isLeaf() ? 4u : 0u);
		const auto box = it.getAABB();
		const auto mn = box.getMin(), mx = box.getMax();
		if (it.getDistance() != std::sqrt(it.getSquaredDistance()) || it.getCenter()[0] != it.getX() ||
		    it.getSize() != 2.0 * it.getHalfSize() || it.hasChildren() == it.isLeaf() ||
		    it.isPureLeaf() != (0 == it.getDepth()) || it.getCode().getDepth() != it.getDepth())
			std::printf("FAILED: accessors disagree\n");
		std::printf("%s %" PRIu64 " %u %08" PRIx32 " %u %u %u %u %016" PRIx64 " %016" PRIx64 " %016" PRIx64 " %016" PRIx64
		            " %016" PRIx64 " %016" PRIx64 " %016" PRIx64 "\n",
		            name, (std::uint64_t)it.getCode().getCode(), (unsigned)it.getDepth(), fbits(it->occupancy), r, g, b, fl,
		            bits(it.getSquaredDistance()), bits(mn[0]), bits(mn[1]), bits(mn[2]), bits(mx[0]), bits(mx[1]), bits(mx[2]));
	}
}

// the planner's question: how far is the nearest occupied voxel
template <typename T>
double nearestOccupied(T const& map, ufo::map::Point3 const& p)
{
	double d = -1.0;
	for (auto it = map.beginNNLeaves(p, true, false, false); it != map.endNNLeaves(); ++it) {
		d = it.getDistance();
		break;
	}
	return d;
}

template <typename T>
int run(T& map, ufo::map::Point3 const& p)
{
	geo::Sphere const sphere(p, 1.5);
	geo::AABB const box(ufo::map::Point3(p[0] - 0.7, p[1] - 0.4, p[2] - 0.3), ufo::map::Point3(p[0] + 0.6, p[1] + 0.9, p[2] + 0.5));
	geo::BoundingVolume volume;
	volume.add(box);
	volume.add(sphere);
	dump("tree", map.beginNNTree(p, true, false, false, false, 1), map.endNNTree());
	dump("tree_var", map.beginNNTree(p, geo::BoundingVar(sphere), true, true, false, true, 0), map.endNNTree());
	dump("tree_volume", map.beginNNTree(p, volume), map.endNNTree());
	dump("leaves", map.beginNNLeaves(p, true, false, false), map.endNNLeaves());
	dump("leaves_var", map.beginNNLeaves(p, geo::BoundingVar(box), false, true, false, false, 2), map.endNNLeaves());
	dump("leaves_volume", map.beginNNLeaves(p, volume, true, true, true), map.endNNLeaves());
	std::printf("planner %016" PRIx64 "\n", bits(nearestOccupied(map, p)));

	// equality as the facade's Iterator: copies at the same node are equal, end == end
	auto a = map.beginNNLeaves(p, true, true, false);
	auto b = a;
	if (a != b || !(map.endNNLeaves() == map.endNNLeaves())) return fail("equality");
	if (a != map.endNNLeaves()) {
		++b;
		if (a == b) return fail("advanced copy compares equal");
	}

	// a map changed in the middle of an iteration: the next shell fetch ends it
	std::size_t seen = 0;
	bool changed = false;
	auto it = map.beginNNLeaves(p, true, true, false);
	for (; it != map.endNNLeaves(); ++it, ++seen) {
		if (!changed && seen == 3) {
			map.integrateHit(ufo::map::Point3(p[0] + 0.05, p[1] + 0.05, p[2] + 0.05));
			changed = true;
		}
		if (seen > 100000) break;
	}
	std::printf("changed %zu %d\n", seen, map.lastStatus());
	return 0;
}

int noDevice()
{
	int (*mono)(ufo::map::OccupancyMap&, ufo::map::Point3 const&) = &run<ufo::map::OccupancyMap>;
	int (*color)(ufo::map::OccupancyMapColor&, ufo::map::Point3 const&) = &run<ufo::map::OccupancyMapColor>;
	if (!mono || !color) return fail("instantiation");
	ufo::map::OccupancyMap::NNIterator a, b;
	if (!(a == b) || a != b) return fail("end == end");

	ufo_b200_params prm;
	ufo_b200_default_params(&prm);
	prm.device = -2;  // geometry-only handle
	ufo_b200_map* m = nullptr;
	if (UFO_B200_OK != ufo_b200_create(&prm, &m)) return fail("geometry-only handle");
	const double p[3] = {0.1, 0.2, 0.3}, bad_p[3] = {0.0, NAN, 0.0};
	std::size_t n = 7;
	double next = 0.0;
	std::uint64_t codes[1];
	std::uint8_t depths[1], flags[1];
	float occ[1];
	double d2[1];
	if (UFO_B200_E_INVALID != ufo_b200_nearest(nullptr, p, nullptr, 0, 1, 1, 1, 0, 0, 0, 0.0, 1, nullptr, nullptr, nullptr,
	                                           nullptr, nullptr, nullptr, 0, &n, &next))
		return fail("NULL map");
	if (UFO_B200_E_INVALID != ufo_b200_nearest(m, bad_p, nullptr, 0, 1, 1, 1, 0, 0, 0, 0.0, 1, nullptr, nullptr, nullptr, nullptr,
	                                           nullptr, nullptr, 0, &n, &next))
		return fail("non-finite point");
	if (UFO_B200_E_INVALID != ufo_b200_nearest(m, p, nullptr, 0, 1, 1, 1, 0, 0, 0, NAN, 1, nullptr, nullptr, nullptr, nullptr,
	                                           nullptr, nullptr, 0, &n, &next))
		return fail("NaN d2_from");
	if (UFO_B200_E_INVALID != ufo_b200_nearest(m, p, nullptr, 0, 1, 1, 1, 0, 0, 0, 0.0, 1, codes, depths, occ, flags, nullptr,
	                                           nullptr, 1, &n, &next))
		return fail("cap > 0 without d2");
	if (UFO_B200_E_CUDA != ufo_b200_nearest(m, p, nullptr, 0, 1, 1, 1, 0, 0, 0, 0.0, 1, codes, depths, occ, flags, nullptr, d2,
	                                        1, &n, &next) ||
	    n != 0)
		return fail("geometry-only handle must refuse");
	ufo_b200_destroy(m);
	std::printf("facade nearest ok (no device)\n");
	return 0;
}
}  // namespace

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) return noDevice();
	if (argc != 8) return fail("usage");
	double res = std::atof(argv[2]);
	unsigned levels = (unsigned)std::atoi(argv[3]);
	bool color = std::atoi(argv[4]) != 0;
	ufo::map::Point3 p(std::atof(argv[5]), std::atof(argv[6]), std::atof(argv[7]));
	auto go = [&](auto& map) {
		std::ifstream f(argv[1], std::ios_base::in | std::ios_base::binary);
		if (!f.is_open() || !map.readData(f, res, levels)) return fail("readData");
		if (run(map, p)) return 1;
		std::printf("facade nearest ok\n");
		return 0;
	};
	if (color) {
		ufo::map::OccupancyMapColor map(res, levels);
		return go(map);
	}
	ufo::map::OccupancyMap map(res, levels);
	return go(map);
}
