/* oracle/ufo_oracle_color_writes.c -- TEST INFRASTRUCTURE ONLY.
 *
 * ufo_oracle_writes.c (included whole, with the CPU restatement) plus the colour map's two public
 * writers, built into oracle/libufo_oracle_color_writes.so by oracle/color_writes.mk.  Every
 * ufo_oracle_* entry point of libufo_oracle_writes.so is exported as well, so one handle serves all
 * (tests/color_writes_lib.py).
 */
#include "ufo_oracle_writes.c"

void ufo_oracle_update_nodes_color(void* h, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                                   const float* values, const uint8_t* rgb, size_t n, uint8_t* changed);

/* OMC.cpp:74-81: createNode, the node takes the colour, updateParents */
static void set_color(omap* m, uint64_t code, const uint8_t rgb[3])
{
	node* path[MAX_LEVELS + 1];
	create_path(m, code, 0, path);
	memcpy(path[0]->rgb, rgb, 3);
	update_parents(m, path, 0);
}

/* the log-odds of the depth-0 voxel of `code` (a collapsed leaf above it holds it) */
static float voxel_occ(void* h, uint64_t code)
{
	float occ;
	uint8_t rgb[3], flags;
	unsigned found;
	ufo_oracle_node(h, code, 0, &occ, rgb, &flags, &found);
	return occ;
}

/* Writes in array order: ops 0 / 1 as ufo_oracle_update_nodes; op 2 updateValue(code, value,
 * Color) OMC.h:269-287 (blend weighted by toProb(value) against the voxel's occupancy before the
 * add, then the add); op 3 setColor(code, Color).  Ops 2 and 3 at depth 0.  changed (may be NULL):
 * changed[i] = 1 when a depth-0 entry of op 0 or 2 changed its voxel's log-odds -- the reference's
 * change detection records exactly those codes. */
void ufo_oracle_update_nodes_color(void* h, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                                   const float* values, const uint8_t* rgb, size_t n, uint8_t* changed)
{
	omap* m = (omap*)h;
	for (size_t i = 0; i < n; ++i) {
		const uint64_t code = mask_code(m, codes[i]);
		const int track = changed && 0 == depths[i] && (ops[i] == 0 || ops[i] == 2);
		const float before = track ? voxel_occ(h, code) : 0.0f;
		if (ops[i] == 3) set_color(m, code, rgb + 3 * i);
		else if (ops[i] == 2) update_value_color(m, code, values[i], rgb + 3 * i);
		else ufo_oracle_update_nodes(h, codes + i, depths + i, ops + i, values + i, 1);
		if (changed) {
			const float after = track ? voxel_occ(h, code) : before;
			changed[i] = memcmp(&before, &after, sizeof(float)) != 0;
		}
	}
}
