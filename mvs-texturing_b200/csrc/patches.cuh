// patches.cuh -- device-resident state of the texture-patch stages (patches.cu, localseam.cu)
#pragma once
#include "common.cuh"
#include "patches_host.h"

namespace b2 {

struct PatchState {
    PatchPlan plan;
    std::vector<uint32_t> faces;          // face id per final slot
    DevBuf<uint32_t> comp_faces, slot_comp0, slot_src, slot_comp, slot_patch, slot_face, comp_chain, comp_wh, key;
    DevBuf<int32_t> comp_bbox, comp_min, desc;
    DevBuf<uint64_t> pix_off;
    DevBuf<float> px, tex, chain, adj, img;
    DevBuf<uint8_t> valid, blend;
    uint64_t total_pixels = 0;
    // local seam leveling (localseam.cu)
    DevBuf<float> orig;                   // images before the seam colours are stamped (Poisson source)
    DevBuf<float> edge_proj, edge_color, vert_color, vert_proj;
    DevBuf<uint32_t> edge_info, sample_edge, vert_info, line_info, pixw_info;
    DevBuf<uint32_t> plan_face_slot, plan_cnt_a, plan_cnt_b, plan_off_a, plan_off_b, plan_edges, plan_flags;   // seam planning on the device
    DevBuf<uint8_t> layer;
    DevBuf<uint32_t> uflag, uidx, ulist;
    DevBuf<int32_t> unb;
    DevBuf<float> cg_b, cg_x, cg_r, cg_t;
    DevBuf<float4> cg_p;
    DevBuf<double> cg_partials;
    DevBuf<uint32_t> cg_status;
    bool leveled = false;
};

}  // namespace b2
