// oracle/ref_info.cpp -- TEST INFRASTRUCTURE ONLY.
//
// The colour-writes checker (ref_color_writes.cpp, included whole: the reference shim, write batches
// and colour batches) plus the reference's tree counters, its known box and its copy constructor's steps.
// Built into oracle/_ref/libufo_ref_info.so by oracle/info.mk from the UNMODIFIED reference sources
// (tests/info_lib.py).  Nothing in the product path may link or load it.
#include "ref_color_writes.cpp"

#include <type_traits>

extern "C" {

// out4: getNumLeafNodes(), getNumInnerNodes(), size(), memoryUsage() (octree.h:411-443);
// box6: getKnownBBX() (occupancy_map_base.h:828-852) as the AABB holds it, centre xyz then half size xyz.
void ufo_ref_tree_info(void* h, uint64_t* out4, double* box6)
{
	RefMap* m = static_cast<RefMap*>(h);
	withMap(m, [&](auto& map) {
		out4[0] = map.getNumLeafNodes();
		out4[1] = map.getNumInnerNodes();
		out4[2] = map.size();
		out4[3] = map.memoryUsage();
		const ufo::geometry::AABB b = map.getKnownBBX();
		for (int i = 0; i < 3; ++i) {
			box6[i] = b.center[i];
			box6[3 + i] = b.half_size[i];
		}
	});
}

// A new handle holding a copy of the map made the way its copy constructor makes one
// (occupancy_map_base.h:888-897, occupancy_map.cpp:65, occupancy_map_color.cpp:65-68): a map constructed
// from the source's resolution, depth levels, pruning setting and probability getters, then
// write(stream) of the source and read(stream).  The constructor itself cannot be called: it runs read
// while the base class is still under construction, where read's virtual calls are pure ("pure virtual
// method called").  So the same steps run here once the new map is complete.  NULL on an exception.
void* ufo_ref_copy(void* h)
{
	RefMap* m = static_cast<RefMap*>(h);
	try {
		RefMap* c = new RefMap;
		c->color = m->color;
		withMap(m, [&](auto& map) {
			using P = std::decay_t<decltype(map)>;
			P* copy = new P(map.getResolution(), map.getTreeDepthLevels(), map.isAutomaticPruningEnabled(),
			                map.getOccupiedThres(), map.getFreeThres(), map.getProbHit(), map.getProbMiss(),
			                map.getClampingThresMin(), map.getClampingThresMax());
			if constexpr (std::is_same_v<P, Probe<ufo::map::OccupancyMapColor>>) c->col = copy;
			else c->mono = copy;
			std::stringstream s(std::ios_base::in | std::ios_base::out | std::ios_base::binary);
			map.write(s);
			copy->read(s);
		});
		return c;
	} catch (std::exception const&) {
		return nullptr;
	}
}

}  // extern "C"
