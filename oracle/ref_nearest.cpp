// oracle/ref_nearest.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Two CPU checkers of the nearest-first iteration (beginNNTree / beginNNLeaves with the intended
// semantics: the nodes of beginTree / beginLeaves in non-decreasing squared distance from a point).
// The reference's own nearest iterators cannot be used: beginNNTree does not compile and beginNNLeaves
// expands the node after the one it pops (iterator/octree_nearest.h:236-241).
//
//   ufo_ref_nearest_sorted    the reference's beginTree / beginLeaves, each node's distance computed with
//                             the reference's Point3::clamp and squaredNorm (octree_nearest.h:198-202),
//                             then stable-sorted by distance: equal distances keep the iterator's order.
//   ufo_ref_nearest_bestfirst the reference's best-first search restated with the popped-node test fixed:
//                             a priority queue of (distance, node) over the reference's own pointer tree
//                             (getRoot / getChild / isLeaf), with the iterators' validNode and
//                             validReturnNode.  Equal distances come in the queue's order.
//
// Built into oracle/_ref/libufo_ref_nearest.so by oracle/nearest.mk from the UNMODIFIED reference
// sources (tests/nearest_lib.py).  Nothing in the product path may link or load it.
#include "ref_volumes.cpp"

#include <algorithm>
#include <numeric>
#include <queue>
#include <type_traits>

namespace
{
struct NearRec {
	uint64_t code;
	uint8_t depth, flags;
	float occ;
	uint8_t rgb[3];
	double centre[3];
	double d2;
};

double squaredDistance(Point3 const& p, ufo::geometry::AABB const& aabb)
{
	Point3 closest = Point3::clamp(p, aabb.getMin(), aabb.getMax());
	return (p - closest).squaredNorm();
}

size_t put_out(std::vector<NearRec> const& v, uint64_t* codes, uint8_t* depths, float* occ, uint8_t* flags, uint8_t* rgb,
               double* centres, double* d2, size_t cap)
{
	if (codes && v.size() <= cap) {
		for (size_t i = 0; i < v.size(); ++i) {
			codes[i] = v[i].code;
			depths[i] = v[i].depth;
			occ[i] = v[i].occ;
			flags[i] = v[i].flags;
			for (int k = 0; k < 3; ++k) {
				rgb[3 * i + k] = v[i].rgb[k];
				centres[3 * i + k] = v[i].centre[k];
			}
			d2[i] = v[i].d2;
		}
	}
	return v.size();
}

// The best-first search over the reference's tree, with the popped node's own depth and leaf state
// deciding whether it is expanded.
template <class MAP>
class NearestProbe : public MAP
{
 public:
	using Leaf = typename MAP::LEAF_NODE;
	using Inner = typename MAP::INNER_NODE;

	std::vector<NearRec> search(Point3 const& p, geo::BoundingVolume const& bv, bool leaves, bool occupied, bool free_space,
	                            bool unknown, bool contains, unsigned min_depth) const
	{
		struct Item {
			double d2;
			Leaf const* node;
			unsigned depth;
			uint64_t code;
			Point3 centre;
			bool operator>(Item const& o) const { return d2 > o.d2; }
		};
		std::vector<NearRec> out;
		const unsigned L = this->getTreeDepthLevels();
		if (min_depth > L) return out;
		auto valid = [&](Item const& it) {
			ufo::geometry::AABB box(it.centre, this->getNodeHalfSize(it.depth));
			if (!bv.empty() && !bv.intersects(box)) return false;
			if (contains || min_depth != it.depth)
				return (occupied && this->containsOccupied(*it.node, it.depth)) ||
				       (unknown && this->containsUnknown(*it.node, it.depth)) ||
				       (free_space && this->containsFree(*it.node, it.depth));
			return (occupied && this->isOccupied(*it.node)) || (unknown && this->isUnknown(*it.node)) ||
			       (free_space && this->isFree(*it.node));
		};
		auto returns = [&](Item const& it) {
			const bool leaf = MAP::isLeaf(it.node, it.depth);
			if (leaves && !(min_depth == it.depth || leaf)) return false;
			if (!leaves && contains)
				return (occupied && this->containsOccupied(*it.node, it.depth)) ||
				       (unknown && this->containsUnknown(*it.node, it.depth)) ||
				       (free_space && this->containsFree(*it.node, it.depth));
			return (occupied && this->isOccupied(*it.node)) || (unknown && this->isUnknown(*it.node)) ||
			       (free_space && this->isFree(*it.node));
		};
		std::priority_queue<Item, std::vector<Item>, std::greater<Item>> q;
		Item root{0.0, &this->getRoot(), L, 0, Point3(0, 0, 0)};
		root.d2 = squaredDistance(p, ufo::geometry::AABB(root.centre, this->getNodeHalfSize(L)));
		if (valid(root)) q.push(root);
		while (!q.empty()) {
			const Item it = q.top();
			q.pop();
			if (returns(it)) out.push_back(record(it.node, it.depth, it.code, it.centre, it.d2));
			if (it.depth <= min_depth || MAP::isLeaf(it.node, it.depth)) continue;
			auto const& inner = static_cast<Inner const&>(*it.node);
			const unsigned cd = it.depth - 1;
			const double chs = this->getNodeHalfSize(cd);
			for (unsigned i = 0; i < 8; ++i) {
				Item c;
				c.node = &MAP::getChild(inner, cd, i);
				c.depth = cd;
				c.code = it.code | (uint64_t(i) << (3 * cd));
				c.centre = MAP::getChildCenter(it.centre, chs, i);
				c.d2 = squaredDistance(p, ufo::geometry::AABB(c.centre, chs));
				if (valid(c)) q.push(c);
			}
		}
		return out;
	}

 private:
	NearRec record(Leaf const* node, unsigned depth, uint64_t code, Point3 const& c, double d2) const
	{
		NearRec r{};
		r.code = code;
		r.depth = (uint8_t)depth;
		r.occ = (float)node->value.occupancy;
		if constexpr (std::is_base_of_v<ufo::map::OccupancyMapColor, MAP>) {
			r.rgb[0] = node->value.color.r;
			r.rgb[1] = node->value.color.g;
			r.rgb[2] = node->value.color.b;
		}
		r.flags = (uint8_t)((this->containsFree(*node, depth) ? 1 : 0) | (this->containsUnknown(*node, depth) ? 2 : 0) |
		                    (MAP::isLeaf(node, depth) ? 4 : 0));
		for (int k = 0; k < 3; ++k) r.centre[k] = c[k];
		r.d2 = d2;
		return r;
	}
};
}  // namespace

extern "C" {

// Per node, in non-decreasing distance: code, depth, log-odds bits, colour, flags (containsFree |
// containsUnknown << 1 | isLeaf << 2), centre (3 doubles) and the squared distance.  Returns the number
// of nodes; fills the arrays when it is <= cap.
size_t ufo_ref_nearest_sorted(void* h, const double* point, int leaves, int occupied, int free_space, int unknown,
                              int contains, unsigned min_depth, const VolumeRecord* recs, size_t n_recs, uint64_t* codes,
                              uint8_t* depths, float* occ, uint8_t* flags, uint8_t* rgb, double* centres, double* d2,
                              size_t cap)
{
	RefMap* m = static_cast<RefMap*>(h);
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	const Point3 p(point[0], point[1], point[2]);
	std::vector<NearRec> v;
	withMap(m, [&](auto& map) {
		using M = std::decay_t<decltype(map)>;
		auto dump = [&](auto it, auto end) {
			for (; it != end; ++it) {
				NearRec r{};
				r.code = it.getCode().getCode();
				r.depth = (uint8_t)it.getDepth();
				r.occ = (float)it->occupancy;
				if constexpr (std::is_base_of_v<ufo::map::OccupancyMapColor, M>) {
					r.rgb[0] = it->color.r;
					r.rgb[1] = it->color.g;
					r.rgb[2] = it->color.b;
				}
				r.flags = (uint8_t)((it.containsFree() ? 1 : 0) | (it.containsUnknown() ? 2 : 0) | (it.isLeaf() ? 4 : 0));
				const auto c = it.getCenter();
				for (int k = 0; k < 3; ++k) r.centre[k] = c[k];
				r.d2 = squaredDistance(p, ufo::geometry::AABB(c, it.getHalfSize()));
				v.push_back(r);
			}
		};
		if (leaves)
			dump(map.beginLeaves(bv, occupied != 0, free_space != 0, unknown != 0, contains != 0, min_depth), map.endLeaves());
		else
			dump(map.beginTree(bv, occupied != 0, free_space != 0, unknown != 0, contains != 0, min_depth), map.endTree());
	});
	std::stable_sort(v.begin(), v.end(), [](NearRec const& a, NearRec const& b) { return a.d2 < b.d2; });
	return put_out(v, codes, depths, occ, flags, rgb, centres, d2, cap);
}

size_t ufo_ref_nearest_bestfirst(void* h, const double* point, int leaves, int occupied, int free_space, int unknown,
                                 int contains, unsigned min_depth, const VolumeRecord* recs, size_t n_recs, uint64_t* codes,
                                 uint8_t* depths, float* occ, uint8_t* flags, uint8_t* rgb, double* centres, double* d2,
                                 size_t cap)
{
	RefMap* m = static_cast<RefMap*>(h);
	const geo::BoundingVolume bv = to_volume(recs, n_recs);
	const Point3 p(point[0], point[1], point[2]);
	std::vector<NearRec> v;
	if (m->color)
		v = static_cast<NearestProbe<ufo::map::OccupancyMapColor> const*>(
		        static_cast<ufo::map::OccupancyMapColor const*>(m->col))
		        ->search(p, bv, leaves, occupied, free_space, unknown, contains, min_depth);
	else
		v = static_cast<NearestProbe<ufo::map::OccupancyMap> const*>(static_cast<ufo::map::OccupancyMap const*>(m->mono))
		        ->search(p, bv, leaves, occupied, free_space, unknown, contains, min_depth);
	return put_out(v, codes, depths, occ, flags, rgb, centres, d2, cap);
}

}  // extern "C"
