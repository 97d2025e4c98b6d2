// state.h -- which resident item of a b2tex_ctx is derived from which.  Plain C++ (no CUDA): the CPU tests compile it.
//
// Every upload and every stage result held by a context is one item.  An item is valid while the items it was computed
// from are unchanged; changing an item (an upload, a stage run) invalidates everything derived from it, transitively.
// The helpers that apply the table to a context (invalidate, mark_valid, require) are in common.cuh.
#pragma once

#include <stdint.h>

namespace b2 {

enum Item : uint32_t {
    MESH = 1u << 0,          // verts, faces, face normals, F, Vn
    PREP = 1u << 1,          // vertex normals and kept face ids of prepare_mesh
    BVH = 1u << 2,
    ADJ = 1u << 3,           // face adjacency
    RINGS = 1u << 4,         // vertex -> faces, vertex -> vertices
    VIEWS = 1u << 5,         // cameras, K
    PIXELS = 1u << 6,        // rgb images
    IMAGES = 1u << 7,        // camera block, gradients, validity masks (prepare_images)
    COSTS = 1u << 8,         // data costs
    MRF = 1u << 9,           // forest state that mrf_iterate, mrf_energy and mrf_sample_forest read
    LABELS = 1u << 10,
    SEAM_SYSTEM = 1u << 11,  // the assembled seam leveling system
    SEAM = 1u << 12,         // its solution
    PATCHES = 1u << 13,      // texture patches
};
constexpr int NUM_ITEMS = 14;
constexpr uint32_t ALL_ITEMS = (1u << NUM_ITEMS) - 1;

inline const char *item_name(int i)
{
    static const char *const names[NUM_ITEMS] = {"mesh", "prepared mesh", "BVH", "face adjacency", "vertex rings", "views",
                                                 "pixels", "prepared images", "data costs", "view selection state",
                                                 "labels", "seam system", "seam solution", "texture patches"};
    return names[i];
}

// the items item i is computed from
constexpr uint32_t inputs_of(int i)
{
    switch (1u << i) {
        case PREP: return MESH;
        case BVH: return MESH;
        case ADJ: return MESH;
        case RINGS: return MESH;
        case PIXELS: return VIEWS;
        case IMAGES: return PIXELS;
        case COSTS: return MESH | PIXELS;
        case MRF: return COSTS | ADJ;
        case LABELS: return MESH | VIEWS;
        case SEAM_SYSTEM: return MESH | PIXELS | RINGS | LABELS;
        case SEAM: return SEAM_SYSTEM;
        case PATCHES: return MESH | PIXELS | ADJ | LABELS;
        default: return 0;
    }
}

// every item derived, directly or through other items, from one of `bits`
constexpr uint32_t dependents_of(uint32_t bits)
{
    uint32_t out = 0;
    for (bool grew = true; grew;) {
        grew = false;
        for (int i = 0; i < NUM_ITEMS; ++i)
            if (!(out & (1u << i)) && (inputs_of(i) & (bits | out))) {
                out |= 1u << i;
                grew = true;
            }
    }
    return out;
}

}  // namespace b2
