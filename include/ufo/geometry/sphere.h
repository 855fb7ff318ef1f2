// Drop-in include path of the reference (ufo/geometry/sphere.h): forwards to the H100-native facade, so a
// caller's #include <ufo/geometry/sphere.h> stays as it is when include/ of this repository is on the path.
#pragma once
#include <ufomap_b200/ufomap.hpp>
