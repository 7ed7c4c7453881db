// Boost stand-in: everything lives in boost/geometry.hpp.
#pragma once
#include <boost/geometry.hpp>
