// oracle/ref_iterate.cpp -- TEST INFRASTRUCTURE ONLY.
//
// The bounding-volume checker (ref_volumes.cpp, included whole) plus a dump of the reference's own
// iterators: beginTree / beginLeaves(BoundingVolume, occupied, free, unknown, contains, min_depth)
// (occupancy_map_base.h:120-163) with everything a caller reads per node.  Built into
// oracle/_ref/libufo_ref_iterate.so by oracle/iterate.mk from the UNMODIFIED reference sources
// (tests/iterate_lib.py).  Nothing in the product path may link or load it.
#include "ref_volumes.cpp"

#include <type_traits>

extern "C" {

// Per node, in the iterator's order: getCode().getCode(), getDepth(), the float log-odds bits of
// it->occupancy, it->color (colour maps; zeros otherwise), flags = containsFree | containsUnknown << 1
// | isLeaf << 2 | isOccupied << 3 | isFree << 4 | isUnknown << 5 | containsOccupied << 6,
// getCenter() (3 doubles) and getOccupancy().  Returns the number of nodes; fills the arrays up to cap.
size_t ufo_ref_iterate(void* h, int leaves, int occupied, int free_space, int unknown, int contains, unsigned min_depth,
                       const VolumeRecord* recs, size_t n_recs, uint64_t* codes, uint8_t* depths, float* occ, uint8_t* flags,
                       uint8_t* rgb, double* centres, double* probs, size_t cap)
{
	RefMap* m = static_cast<RefMap*>(h);
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	return withMap(m, [&](auto& map) {
		using M = std::decay_t<decltype(map)>;
		size_t n = 0;
		auto dump = [&](auto it, auto end) {
			for (; it != end; ++it, ++n) {
				if (!codes || n >= cap) continue;
				codes[n] = it.getCode().getCode();
				depths[n] = (uint8_t)it.getDepth();
				occ[n] = (float)it->occupancy;
				rgb[3 * n] = rgb[3 * n + 1] = rgb[3 * n + 2] = 0;
				if constexpr (std::is_base_of_v<ufo::map::OccupancyMapColor, M>) {
					rgb[3 * n] = it->color.r;
					rgb[3 * n + 1] = it->color.g;
					rgb[3 * n + 2] = it->color.b;
				}
				flags[n] = (uint8_t)((it.containsFree() ? 1 : 0) | (it.containsUnknown() ? 2 : 0) | (it.isLeaf() ? 4 : 0) |
				                     (it.isOccupied() ? 8 : 0) | (it.isFree() ? 16 : 0) | (it.isUnknown() ? 32 : 0) |
				                     (it.containsOccupied() ? 64 : 0));
				const auto c = it.getCenter();
				put(c, centres + 3 * n);
				probs[n] = it.getOccupancy();
			}
		};
		if (leaves)
			dump(map.beginLeaves(bv, occupied != 0, free_space != 0, unknown != 0, contains != 0, min_depth), map.endLeaves());
		else
			dump(map.beginTree(bv, occupied != 0, free_space != 0, unknown != 0, contains != 0, min_depth), map.endTree());
		return n;
	});
}

}  // extern "C"
