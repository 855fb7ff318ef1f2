/* oracle/ufo_oracle_writes.c -- TEST INFRASTRUCTURE ONLY.
 *
 * The CPU restatement (ufo_oracle.c, included whole so that the tree helpers are reachable) plus the
 * per-node writes and ray insertion of the reference, built into oracle/libufo_oracle_writes.so by
 * oracle/writes.mk.  Every ufo_oracle_* entry point of libufo_oracle.so is exported as well, so one
 * handle serves both (tests/writes_lib.py).
 */
#include "ufo_oracle.c"

void ufo_oracle_update_nodes(void* h, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                             const float* values, size_t n);
void ufo_oracle_insert_rays(void* h, const double* origins, const double* ends, size_t n, double max_range,
                            unsigned depth, int hit_end);

/* ---- per-node writes, one after the other in array order:
 * op 0: updateValue(Code(code, depth), value)  OMB:1063-1120 (integrateHit / integrateMiss /
 *       updateOccupancy are this with a fixed or converted value, OMB:544-593);
 * op 1: setNodeValue(code, value) OMB:1037-1057 as intended -- the node takes clamp(value) and loses
 *       its children.  The reference returns early when the deepest EXISTING node on the path already
 *       holds the value (its getNodePath stops one level short, SURVEY.md Appendix B); that early
 *       return is not restated, the node is always written. */
static void set_node_value(omap* m, uint64_t code, unsigned depth, float value)
{
	node* path[MAX_LEVELS + 1];
	create_path(m, code, depth, path);
	node* n = path[depth];
	set_occ(m, &n->occ, value);
	if (depth > 0 && !n->is_leaf) delete_children(m, n, depth);
	update_parents(m, path, depth);
}

void ufo_oracle_update_nodes(void* h, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                             const float* values, size_t n)
{
	omap* m = (omap*)h;
	for (size_t i = 0; i < n; ++i) {
		if (ops[i]) set_node_value(m, mask_code(m, codes[i]), depths[i], values[i]);
		else update_value(m, mask_code(m, codes[i]), depths[i], values[i]);
	}
}

/* insertMissOnRay (OMB:251-258): integrateMiss on every code computeRay returns; insertRay
 * (OMB:260-268, which does not compile: it calls Base::insertMissOnRay) additionally integrateHit on
 * the depth-0 voxel of the end point as given. */
void ufo_oracle_insert_rays(void* h, const double* origins, const double* ends, size_t n, double max_range,
                            unsigned depth, int hit_end)
{
	omap* m = (omap*)h;
	const float miss = (float)m->miss, hit = (float)m->hit;
	size_t cap = 1024;
	uint64_t* codes = (uint64_t*)malloc(cap * sizeof(uint64_t));
	for (size_t i = 0; i < n; ++i) {
		size_t k = ufo_oracle_compute_ray(h, origins + 3 * i, ends + 3 * i, max_range, depth, codes, cap);
		if (k > cap) {
			cap = k;
			codes = (uint64_t*)realloc(codes, cap * sizeof(uint64_t));
			k = ufo_oracle_compute_ray(h, origins + 3 * i, ends + 3 * i, max_range, depth, codes, cap);
		}
		for (size_t j = 0; j < k; ++j) update_value(m, mask_code(m, codes[j]), depth, miss);
		if (hit_end) update_value(m, mask_code(m, ufo_oracle_to_code(h, ends + 3 * i, 0)), 0, hit);
	}
	free(codes);
}
