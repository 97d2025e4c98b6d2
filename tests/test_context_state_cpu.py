"""The dependency table of the resident context (csrc/state.h), compiled with g++: every item invalidates exactly the items
derived from it, directly or through other items, as include/b2tex.h states it."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mvs-texturing_b200", "csrc")

ITEMS = ["MESH", "PREP", "BVH", "ADJ", "RINGS", "VIEWS", "PIXELS", "IMAGES", "COSTS", "MRF", "LABELS", "SEAM_SYSTEM",
         "SEAM", "PATCHES"]

# what a change of each item leaves out of date, spelled out rather than derived
INVALIDATES = {
    "MESH": {"PREP", "BVH", "ADJ", "RINGS", "COSTS", "MRF", "LABELS", "SEAM_SYSTEM", "SEAM", "PATCHES"},
    "PREP": set(),
    "BVH": set(),
    "ADJ": {"MRF", "PATCHES"},
    "RINGS": {"SEAM_SYSTEM", "SEAM"},
    "VIEWS": {"PIXELS", "IMAGES", "COSTS", "MRF", "LABELS", "SEAM_SYSTEM", "SEAM", "PATCHES"},
    "PIXELS": {"IMAGES", "COSTS", "MRF", "SEAM_SYSTEM", "SEAM", "PATCHES"},
    "IMAGES": set(),
    "COSTS": {"MRF"},
    "MRF": set(),
    "LABELS": {"SEAM_SYSTEM", "SEAM", "PATCHES"},
    "SEAM_SYSTEM": {"SEAM"},
    "SEAM": set(),
    "PATCHES": set(),
}

PROGRAM = r"""
#include <stdio.h>
#include "state.h"
using namespace b2;
static_assert(dependents_of(MESH | VIEWS) == (ALL_ITEMS & ~(MESH | VIEWS)), "everything derives from the mesh or the views");
int main()
{
    const uint32_t items[] = {%s};
    static_assert(sizeof(items) / sizeof(items[0]) == NUM_ITEMS, "one bit per item");
    for (int i = 0; i < NUM_ITEMS; ++i) {
        if (items[i] != 1u << i) return 1;
        printf("%%u %%s\n", dependents_of(items[i]), item_name(i));
    }
    printf("%%u all\n", dependents_of(ALL_ITEMS));
    return 0;
}
""" % ", ".join(ITEMS)


def test_every_item_invalidates_what_is_derived_from_it(tmp_path):
    src, exe = tmp_path / "state.cpp", tmp_path / "state"
    src.write_text(PROGRAM)
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I" + CSRC, str(src), "-o", str(exe)])
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(lines) == len(ITEMS) + 1
    names = set()
    for item, line in zip(ITEMS, lines):
        mask, name = line.split(" ", 1)
        got = {ITEMS[b] for b in range(len(ITEMS)) if int(mask) >> b & 1}
        assert got == INVALIDATES[item], item
        names.add(name)
    assert len(names) == len(ITEMS)   # every item has a name of its own for the error messages
    derived = set().union(*INVALIDATES.values())
    assert int(lines[-1].split()[0]) == sum(1 << ITEMS.index(i) for i in derived)
