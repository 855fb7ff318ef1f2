// Per-node writes and ray insertion through the facade, written like a program against the
// reference.  Built and run by tests/test_facade_writes.py.
#include <ufo/map/occupancy_map.h>
#include <ufo/map/occupancy_map_color.h>

#include <cstdio>
#include <cstring>

using namespace ufo::map;

// every overload the reference offers (occupancy_map_base.h:251-268, :524-593)
template <class MAP>
void use_all(MAP& m, Code c, Point3 p)
{
	m.setOccupancy(c, 0.3);
	m.setOccupancy(p, 0.3);
	m.setOccupancy(p, 0.3, 2);
	m.setOccupancy(0.1, 0.2, 0.3, 0.3, 1);
	m.updateOccupancy(c, 0.6);
	m.updateOccupancy(p, 0.6, 3);
	m.updateOccupancy(0.1, 0.2, 0.3, 0.6);
	m.integrateHit(c);
	m.integrateHit(p);
	m.integrateHit(0.1, 0.2, 0.3, 4);
	m.integrateMiss(c);
	m.integrateMiss(p, 5);
	m.integrateMiss(0.1, 0.2, 0.3);
	m.insertMissOnRay(Point3(0, 0, 0), p);
	m.insertMissOnRay(Point3(0, 0, 0), p, 2.0, 1);
	m.insertRay(Point3(0, 0, 0), p);
	m.insertRay(Point3(0, 0, 0), p, 2.0, 3);
}

static std::uint32_t bits(double p)
{
	float f = (float)std::log(p / (1.0 - p));
	std::uint32_t u;
	std::memcpy(&u, &f, 4);
	return u;
}

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) {
		// depth > 6 is rejected before any device work (a geometry-only handle has no device)
		ufo_b200_params p;
		ufo_b200_default_params(&p);
		p.device = -2;
		ufo_b200_map* h = nullptr;
		if (ufo_b200_create(&p, &h) != UFO_B200_OK) return 2;
		const double o[3] = {0, 0, 0}, e[3] = {1, 0, 0};
		std::uint64_t c = 0;
		std::uint32_t d = 7;
		std::uint8_t op = 0;
		float v = 0.5f;
		if (ufo_b200_insert_rays(h, o, e, 1, -1, 7, 1, 0) != UFO_B200_E_UNSUPPORTED) return 3;
		if (ufo_b200_update_nodes(h, &c, &d, &op, &v, 1, 0) != UFO_B200_E_UNSUPPORTED) return 4;
		ufo_b200_destroy(h);
		std::puts("facade writes ok (no device)");
		return 0;
	}

	OccupancyMap map(0.02);
	Point3 p(0.5, 0.5, 0.5);
	use_all(map, map.toCode(p), p);
	if (map.lastStatus() != UFO_B200_OK) return 10;
	OccupancyMapColor cmap(0.02);
	use_all(cmap, cmap.toCode(p), p);
	if (cmap.lastStatus() != UFO_B200_OK) return 11;  // the last call is insertRay at depth 3

	// SURVEY.md 8(c): integrateHit then integrateMiss on one voxel, then repeated hits stop at the clamp
	OccupancyMap kat(0.02);
	Point3 q(0.31, -0.17, 0.05);
	kat.integrateHit(q);
	kat.integrateMiss(q);
	std::uint64_t c = kat.toCode(q).getCode();
	std::uint32_t d = 0;
	float lo;
	std::uint8_t fl;
	ufo_b200_query(kat.handle(), &c, &d, 1, &lo, &fl, nullptr);
	std::uint32_t u;
	std::memcpy(&u, &lo, 4);
	if (u != 0x3EE237E7u) return 12;
	for (int i = 0; i < 20; ++i) kat.integrateHit(q);
	ufo_b200_query(kat.handle(), &c, &d, 1, &lo, &fl, nullptr);
	std::memcpy(&u, &lo, 4);
	if (u != 0x4060B4BAu) return 13;

	// one insertRay: the computeRay codes become free, the end occupied
	OccupancyMap ray(0.02);
	Point3 a(0, 0, 0), b(0.7, 0.3, -0.2);
	ray.insertRay(a, b);
	for (Code const& k : ray.computeRay(a, b))
		if (!ray.isFree(k)) return 14;
	if (!ray.isOccupied(b)) return 15;
	ray.insertMissOnRay(a, b, -1, 7);
	if (ray.lastStatus() != UFO_B200_E_UNSUPPORTED) return 16;
	// setOccupancy: the node takes the clamped value
	ray.setOccupancy(b, 0.999);
	c = ray.toCode(b).getCode();
	ufo_b200_query(ray.handle(), &c, &d, 1, &lo, &fl, nullptr);
	std::memcpy(&u, &lo, 4);
	if (u != bits(0.971)) return 17;
	std::puts("facade writes ok");
	return 0;
}
