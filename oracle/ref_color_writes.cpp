// oracle/ref_color_writes.cpp -- TEST INFRASTRUCTURE ONLY.
//
// ref_writes.cpp (included whole, with the reference shim) plus the colour map's two public writers,
// built into oracle/_ref/libufo_ref_color_writes.so by oracle/color_writes.mk from the UNMODIFIED
// reference sources.  Every ufo_ref_* entry point of libufo_ref_writes.so is exported as well, so one
// handle serves all (tests/color_writes_lib.py).  Nothing in the product path may link or load it.
#include "ref_writes.cpp"

extern "C" {

// Colour writes in array order, one reference call per entry:
//   ops[i] == 0 -> updateValue(Code(code, depth), value)            occupancy_map_base.h:1063-1083
//   ops[i] == 2 -> OccupancyMapColor::updateValue(Code, value, Color) occupancy_map_color.h:269-287
//   ops[i] == 3 -> OccupancyMapColor::setColor(Code, Color)         occupancy_map_color.cpp:74-81
// rgb[n][3].  setNodeValue (op 1) does not compile in the reference, and the colour calls do not
// exist on a map without colour: such a batch is refused (-1) before anything is applied.
int ufo_ref_update_nodes_color(void* h, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                               const float* values, const uint8_t* rgb, size_t n)
{
	RefMap* m = static_cast<RefMap*>(h);
	for (size_t i = 0; i < n; ++i)
		if (ops[i] == 1 || ops[i] > 3 || (ops[i] >= 2 && !m->color)) return -1;
	if (!m->color) return ufo_ref_update_nodes(h, codes, depths, ops, values, n);
	ufo::map::OccupancyMapColor& map = *m->col;
	for (size_t i = 0; i < n; ++i) {
		const Code code(codes[i], depths[i]);
		const ufo::map::Color c(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
		if (ops[i] == 0) UpdateValue<ufo::map::OccupancyMapColor>::call(map, code, values[i]);
		else if (ops[i] == 2) map.updateValue(code, values[i], c);
		else map.setColor(code, c);
	}
	return 0;
}

}  // extern "C"
