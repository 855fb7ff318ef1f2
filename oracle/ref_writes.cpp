// oracle/ref_writes.cpp -- TEST INFRASTRUCTURE ONLY.
//
// The reference shim (ref_harness.cpp, included whole) plus the reference's per-node writes and
// ray insertion, built into oracle/_ref/libufo_ref_writes.so by oracle/writes.mk from the UNMODIFIED
// reference sources.  Every ufo_ref_* entry point of libufo_ref.so is exported as well, so one
// handle serves both (tests/writes_lib.py).  Nothing in the product path may link or load it.
#include "ref_harness.cpp"

namespace
{
template <class MAP>
struct NodeOf {
	using type = ufo::map::OccupancyNode<float>;
};
template <>
struct NodeOf<ufo::map::OccupancyMapColor> {
	using type = ufo::map::ColorOccupancyNode<float>;
};

// updateValue (occupancy_map_base.h:1063-1083) is protected, and the colour map hides it behind its
// own three-argument overload.  A class derived from the map may name it and form a pointer to it,
// through which it is called on the shim's map unchanged, so that any float update passes exactly.
template <class MAP>
struct UpdateValue : MAP {
	using Base = ufo::map::OccupancyMapBase<typename NodeOf<MAP>::type>;
	using Base::updateValue;
	static void call(MAP& m, Code const& code, float value)
	{
		void (Base::*f)(Code const&, float const&) = &UpdateValue::updateValue;
		(m.*f)(code, value);
	}
};
}  // namespace

extern "C" {

// Per-node writes, one reference call per entry in array order: ops[i] == 0 -> updateValue(Code(code,
// depth), value) (the body of integrateHit / integrateMiss / updateOccupancy,
// occupancy_map_base.h:544-593).  setNodeValue does not compile in the reference: a batch with
// ops[i] != 0 is refused (-1) before anything is applied.
int ufo_ref_update_nodes(void* h, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                         const float* values, size_t n)
{
	for (size_t i = 0; i < n; ++i)
		if (ops[i]) return -1;
	RefMap* m = static_cast<RefMap*>(h);
	if (m->color) {
		for (size_t i = 0; i < n; ++i)
			UpdateValue<ufo::map::OccupancyMapColor>::call(*m->col, Code(codes[i], depths[i]), values[i]);
	} else {
		for (size_t i = 0; i < n; ++i)
			UpdateValue<ufo::map::OccupancyMap>::call(*m->mono, Code(codes[i], depths[i]), values[i]);
	}
	return 0;
}

// insertMissOnRay(origin, end, max_range, depth) (occupancy_map_base.h:251-258) per ray; hit_end
// adds integrateHit(end), the rest of insertRay's body (:260-268, which itself does not compile).
void ufo_ref_insert_rays(void* h, const double* origins, const double* ends, size_t n, double max_range,
                         unsigned depth, int hit_end)
{
	RefMap* m = static_cast<RefMap*>(h);
	withMap(m, [&](auto& map) {
		for (size_t i = 0; i < n; ++i) {
			const Point3 o(origins[3 * i], origins[3 * i + 1], origins[3 * i + 2]);
			const Point3 e(ends[3 * i], ends[3 * i + 1], ends[3 * i + 2]);
			map.insertMissOnRay(o, e, max_range, depth);
			if (hit_end) map.integrateHit(e);
		}
	});
}

}  // extern "C"
