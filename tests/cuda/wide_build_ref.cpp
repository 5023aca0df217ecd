// wide_build_ref.cpp — TEST INFRASTRUCTURE: hkw::build_wide (bevy_hikari_b200/csrc/wide_build.h) behind a C function, so that a test can
// derive the 4-wide TLAS of a flat TLAS exactly as hk_scene_upload does on the host and compare it with what kc_build_wide_tlas
// derived on the device (tests/test_gpu_wide_tlas_device.py).  Compiled for the host by the test against tests/emu/include.
#include <string.h>

#include "wide_build.h"

// `nodes` holds room for max(shapes - 1, 1) nodes, `rank` for `shapes` ranks.  A tree the host cannot derive is reported the way
// context.cu upload_wide_tlas uploads it: no nodes, every rank 0.  Returns 1 when the tree could be derived.
extern "C" int wide_build_ref(const hk_node* flat, uint32_t count, uint32_t shapes, hkd::hk_wide_node* nodes, uint32_t* node_count,
                              uint32_t* rank, uint32_t* root, uint32_t* stack_need) {
    hkw::WideTree t = hkw::build_wide(flat, count, shapes, nullptr);
    if (!t.ok) { t.nodes.clear(); t.rank.assign(shapes, 0u); }
    *node_count = (uint32_t)t.nodes.size();
    if (!t.nodes.empty()) memcpy(nodes, t.nodes.data(), sizeof(hkd::hk_wide_node) * t.nodes.size());
    if (!t.rank.empty()) memcpy(rank, t.rank.data(), sizeof(uint32_t) * t.rank.size());
    *root = t.root;
    *stack_need = t.stack_need;
    return t.ok ? 1 : 0;
}
