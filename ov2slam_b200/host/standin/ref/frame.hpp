// Stand-in for the reference's include/frame.hpp: the Frame stand-in lives with the other map classes.
#pragma once
#include "map_manager.hpp"
