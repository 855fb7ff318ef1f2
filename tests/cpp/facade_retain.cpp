// A window that follows the sensor, written against the facade: page out what a box does not keep,
// retain the box, bring the page back.  Built and run by tests/test_facade_retain.py (no device) and
// tests/test_gpu_retain.py (on a device).
//
//   facade_retain --no-device   retain / pageOut / pageIn compile for both map types and every volume
//                               form; argument checks of the C ABI that need no device
//   facade_retain               runs the round trip on the current device, both map types
#include <ufo/map/occupancy_map.h>
#include <ufo/map/occupancy_map_color.h>

#include <cstdio>
#include <cstring>
#include <sstream>
#include <vector>

namespace
{
int fail(char const* what)
{
	std::printf("facade retain FAILED: %s\n", what);
	return 1;
}

template <typename T>
std::string image(T const& map)
{
	std::ostringstream s;
	map.write(s);
	return s.str();
}

template <typename T>
int roundTrip(T& map)
{
	namespace geo = ufo::geometry;
	for (int i = 0; i < 40; ++i)
		map.insertRay(ufo::map::Point3(0.05, 0.05, 0.05), ufo::map::Point3(6.0 - 0.3 * i, 0.2 * i - 4.0, 0.5), -1, 0);
	std::string const before = image(map);
	auto const pools = map.poolStats();
	geo::AABB const box(ufo::map::Point3(-1, -1, -1), ufo::map::Point3(1.5, 1.5, 1.5));
	geo::Sphere const sphere(ufo::map::Point3(0, 0, 0), 2.0);
	geo::BoundingVolume volume;
	volume.add(box);
	volume.add(sphere);

	std::vector<std::uint8_t> const blob = map.pageOut(volume);
	ufo_b200_page_header h{};
	if (UFO_B200_OK != ufo_b200_page_info(blob.data(), blob.size(), &h) || h.bytes != blob.size() || 0 == h.n_bricks)
		return fail("pageOut");
	if (image(map) != before) return fail("pageOut changed the map");
	if (map.pageIn(blob) || UFO_B200_E_INVALID != map.lastStatus()) return fail("pageIn of bricks that exist must be refused");
	ufo_b200_retain_stats st{};
	if (!map.retain(volume, &st) || st.bricks_removed != h.n_bricks || st.bricks_kept + st.bricks_removed != pools.bricks)
		return fail("retain(BoundingVolume)");
	if (image(map) == before) return fail("retain removed nothing");
	if (!map.pageIn(blob) || image(map) != before) return fail("pageIn");
	// the single-shape forms keep a subset of what the union keeps
	if (!map.retain(geo::BoundingVar(sphere), &st) || 0 == st.bricks_kept) return fail("retain(BoundingVar)");
	if (!map.retain(box, &st) || 0 == st.bricks_kept) return fail("retain(AABB)");
	if (map.pageOut(box).size() != map.pageOut(geo::BoundingVar(box)).size()) return fail("pageOut(AABB)");
	return 0;
}

int noDevice()
{
	ufo_b200_params p;
	ufo_b200_default_params(&p);
	p.device = -2;  // geometry-only handle
	ufo_b200_map* m = nullptr;
	if (UFO_B200_OK != ufo_b200_create(&p, &m)) return fail("geometry-only handle");
	double const box6[6] = {0, 0, 0, 1, 1, 1};
	ufo_b200_volume bad{};
	bad.type = 99;
	std::size_t n = 0;
	ufo_b200_retain_stats st{};
	ufo_b200_pool_counts pools{};
	ufo_b200_page_header h{};
	std::uint8_t hdr[64] = {};
	if (UFO_B200_E_INVALID != ufo_b200_retain_bv(nullptr, nullptr, 0, &st)) return fail("NULL map");
	if (UFO_B200_E_INVALID != ufo_b200_retain_bv(m, &bad, 1, &st)) return fail("unknown volume type");
	if (UFO_B200_E_INVALID != ufo_b200_retain_bv(m, nullptr, 1, &st)) return fail("NULL volume with n_bv > 0");
	if (UFO_B200_E_INVALID != ufo_b200_retain(m, nullptr, &st)) return fail("NULL box");
	if (UFO_B200_E_INVALID != ufo_b200_page_out_bv(m, nullptr, 0, nullptr, 0, nullptr)) return fail("NULL size");
	if (UFO_B200_E_INVALID != ufo_b200_page_in(m, nullptr, 64, &st)) return fail("NULL blob");
	if (UFO_B200_E_INVALID != ufo_b200_page_info(hdr, sizeof(hdr), &h)) return fail("bad magic");
	if (UFO_B200_E_INVALID != ufo_b200_pool_stats(m, nullptr)) return fail("NULL stats");
	if (UFO_B200_E_CUDA != ufo_b200_retain(m, box6, &st) || UFO_B200_E_CUDA != ufo_b200_page_out_bv(m, nullptr, 0, nullptr, 0, &n) ||
	    UFO_B200_E_CUDA != ufo_b200_page_in(m, hdr, sizeof(hdr), &st) || UFO_B200_E_CUDA != ufo_b200_pool_stats(m, &pools))
		return fail("geometry-only handle must refuse");
	ufo_b200_destroy(m);
	std::printf("facade retain ok (no device)\n");
	return 0;
}
}  // namespace

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) return noDevice();
	ufo::map::OccupancyMap mono(0.1);
	if (int rc = roundTrip(mono)) return rc;
	ufo::map::OccupancyMapColor color(0.1);
	if (int rc = roundTrip(color)) return rc;
	std::printf("facade retain ok\n");
	return 0;
}
