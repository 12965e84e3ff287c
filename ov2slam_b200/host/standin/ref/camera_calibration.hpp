// Stand-in for the reference's include/camera_calibration.hpp: the CameraCalibration stand-in lives with the other map classes.
#pragma once
#include "map_manager.hpp"
