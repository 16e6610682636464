// stub for Jittor's op.h: included by the Plenoxels data_spec.h, nothing of it is used
#pragma once
