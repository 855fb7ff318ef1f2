// A planner or viewer that loads a saved map, written against the facade as against the reference:
// the file constructors, read(std::istream&) and readType.  Built and run by tests/test_facade_read.py.
//
//   facade_read --no-device   compiles for both map types; readType needs no device
//   facade_read DIR           writes a map to DIR/site.um, opens it with OccupancyMap map(filename),
//                             reads it again through read(istream) and iterates the leaves of both
#include <ufo/map/occupancy_map.h>
#include <ufo/map/occupancy_map_color.h>

#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>

using namespace ufo::map;

namespace
{
template <typename T>
std::size_t leaves(T const& map)
{
	std::size_t n = 0;
	for (auto it = map.beginLeaves(true, true, false, false, 0), end = map.endLeaves(); it != end; ++it) ++n;
	return n;
}

int no_device()
{
	std::istringstream good(
	    "# UFOMap file\n# comment\nversion 1.0.0\nid occupancy_map_color\nresolution 0.05\ndepth_levels 16\n"
	    "compressed 0\nuncompressed_data_size 0\ndata\n");
	if (OccupancyMapColor::readType(good) != "occupancy_map_color") return 2;
	std::istringstream no_version("# UFOMap file\nid occupancy_map\nresolution 0.05\ndata\n");
	if (OccupancyMap::readType(no_version) != "occupancy_map") return 3;  // readType checks nothing else
	std::istringstream not_a_file("# UFOMap\nid occupancy_map\ndata\n");
	if (!OccupancyMap::readType(not_a_file).empty()) return 4;
	if (!OccupancyMap::readType(std::string("/nonexistent/site.um")).empty()) return 5;
	std::puts("facade read ok (no device)");
	return 0;
}
}  // namespace

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) return no_device();
	if (argc < 2) return 1;
	const std::string path = std::string(argv[1]) + "/site.um";
	{
		OccupancyMap map(0.08);
		PointCloud cloud;
		for (int i = 0; i < 400; ++i) cloud.push_back(Point3(2.0 + 0.013 * i, -1.0 + 0.007 * i, 0.3 - 0.002 * i));
		map.insertPointCloud(Point3(0, 0, 0), cloud, 10.0);
		if (!map.write(path)) return 6;
	}
	if (OccupancyMap::readType(path) != "occupancy_map") return 7;
	OccupancyMap map(path);
	if (UFO_B200_OK != map.lastStatus() || map.getResolution() != 0.08 || map.getTreeDepthLevels() != 16) return 8;
	const std::size_t n = leaves(map);
	if (0 == n) return 9;
	std::ifstream file(path, std::ios_base::in | std::ios_base::binary);
	OccupancyMap again(0.2, 12);
	if (!again.read(file) || again.getResolution() != 0.08 || leaves(again) != n) return 10;
	std::ostringstream a, b;
	map.write(a);
	again.write(b);
	if (a.str() != b.str()) return 11;
	// a mono file does not go into a colour map: the constructor leaves the empty map of 0.1
	OccupancyMapColor cmap(path);
	if (UFO_B200_E_INVALID != cmap.lastStatus() || cmap.getResolution() != 0.1 || leaves(cmap) != 0) return 12;
	std::printf("facade read ok: %zu leaves\n", n);
	return 0;
}
