// The colour map's writers through the facade, written like a program against the reference.  Built
// and run by tests/test_facade_color_writes.py.
#include <ufo/map/occupancy_map_color.h>

#include <cmath>
#include <cstdio>
#include <cstring>

using namespace ufo::map;

// every overload the reference offers (occupancy_map_color.h:269-287, :304-330)
void use_all(OccupancyMapColor& map, Code code, Point3 p)
{
	map.setColor(code, Color(10, 20, 30));
	map.setColor(Point3(0.1, 0.2, 0.3), Color(40, 50, 60));
	map.setColor(p, Color(1, 2, 3), 0);
	map.setColor(0.1, 0.2, 0.3, Color(70, 80, 90), 0);
	map.updateValue(code, 0.85f, Color(200, 100, 0));
	map.updateValue(map.toCode(p), 0.85, Color(200, 100, 0));
	Color c = map.getColor(code);
	c = map.getColor(p);
	c = map.getColor(p, 1);
	c = map.getColor(0.1, 0.2, 0.3);
	c = map.getColor(0.1, 0.2, 0.3, 2);
	(void)c;
}

// updateNodeColor (occupancy_map_color.cpp:142-171) of one channel, weight toProb(update)
static int blend(int cur, int upd, float update, float occ)
{
	double prob = 1.0 / (1.0 + std::exp(-update));
	prob /= prob + 1.0 / (1.0 + std::exp(-occ));
	return (int)(unsigned char)std::sqrt(((double)cur * cur) * (1.0 - prob) + ((double)upd * upd) * prob);
}

static int expect(ufo_b200_map* h, std::uint64_t c, std::uint32_t d, std::uint8_t op, const std::uint8_t* rgb, int status)
{
	float v = 0.5f;
	return ufo_b200_update_nodes_color(h, &c, &d, &op, &v, rgb, 1, 0) == status ? 0 : 1;
}

int main(int argc, char** argv)
{
	if (argc > 1 && 0 == std::strcmp(argv[1], "--no-device")) {
		// every rejection is decided before any device work (a geometry-only handle has no device)
		ufo_b200_params p;
		ufo_b200_default_params(&p);
		p.device = -2;
		ufo_b200_map* mono = nullptr;
		ufo_b200_map* col = nullptr;
		if (ufo_b200_create(&p, &mono) != UFO_B200_OK) return 2;
		p.color = 1;
		if (ufo_b200_create(&p, &col) != UFO_B200_OK) return 2;
		const std::uint8_t rgb[3] = {1, 2, 3};
		const std::uint64_t c = 0, out = 1ull << 48;  // key x = 2^16: outside a 16-level tree
		int bad = 0;
		bad += expect(col, c, 0, 4, rgb, UFO_B200_E_INVALID) << 0;
		bad += expect(mono, c, 0, 2, rgb, UFO_B200_E_INVALID) << 1;
		bad += expect(mono, c, 0, 3, rgb, UFO_B200_E_INVALID) << 2;
		bad += expect(col, c, 0, 2, nullptr, UFO_B200_E_INVALID) << 3;
		bad += expect(col, out, 0, 3, rgb, UFO_B200_E_INVALID) << 4;
		bad += expect(col, c, 1, 2, rgb, UFO_B200_E_UNSUPPORTED) << 5;
		bad += expect(col, c, 3, 3, rgb, UFO_B200_E_UNSUPPORTED) << 6;
		bad += expect(col, c, 7, 0, rgb, UFO_B200_E_UNSUPPORTED) << 7;
		bad += expect(col, c, 1, 1, rgb, UFO_B200_E_UNSUPPORTED) << 8;
		if (ufo_b200_update_nodes_color(nullptr, &c, nullptr, nullptr, nullptr, rgb, 1, 0) != UFO_B200_E_INVALID) bad |= 1 << 9;
		ufo_b200_destroy(mono);
		ufo_b200_destroy(col);
		if (bad) {
			std::printf("rejections wrong: mask %#x\n", bad);
			return 3;
		}
		std::puts("facade colour writes ok (no device)");
		return 0;
	}

	OccupancyMapColor map(0.02);
	Point3 p(0.5, 0.5, 0.5);
	use_all(map, map.toCode(p), p);
	if (map.lastStatus() != UFO_B200_OK) return 10;

	// setColor on untouched space: the voxel is created with log-odds 0 and the colour
	OccupancyMapColor kat(0.02);
	Point3 q(0.31, -0.17, 0.05);
	kat.setColor(q, Color(200, 10, 30));
	if (kat.lastStatus() != UFO_B200_OK || kat.getColor(q) != Color(200, 10, 30)) return 11;
	if (kat.getColor(0.31, -0.17, 0.05) != Color(200, 10, 30)) return 12;
	// one hit with a colour onto a set colour at log-odds 0
	const float hit = 0.85f;
	Code code = kat.toCode(q);
	kat.updateValue(code, hit, Color(10, 250, 90));
	Color want(blend(200, 10, hit, 0.0f), blend(10, 250, hit, 0.0f), blend(30, 90, hit, 0.0f));
	if (kat.getColor(code) != want) return 13;
	// the colour of a depth-1 node is the root-mean-square of its set children: here the one voxel
	if (kat.getColor(q, 1) != want) return 14;
	// rejected calls leave their status and change nothing
	kat.setColor(q, Color(1, 1, 1), 1);
	if (kat.lastStatus() != UFO_B200_E_UNSUPPORTED || kat.getColor(code) != want) return 15;
	// setColor (0,0,0) unsets the colour
	kat.setColor(code, Color());
	if (kat.lastStatus() != UFO_B200_OK || kat.getColor(code).isSet()) return 16;
	std::puts("facade colour writes ok");
	return 0;
}
