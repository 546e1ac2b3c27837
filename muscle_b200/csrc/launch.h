// launch.h -- host-visible launch surface of the kernel translation units.
#pragma once
#include "common.cuh"

#define MB_MAX_C 16
// k_posterior_sm is compiled per shared-memory size class CM (columns per lane): 4, 8, 12, 14, 16.
// 14 is its own class: 4 warps x 6 words x 14 columns fit five CTAs in an SM's 228 KB (like 8 and
// 12), 16 columns only four.  Any C <= 16 runs in the smallest class that holds it.
static inline int mb_post_sm_class(int C)
	{
	return C <= 12 ? (C + 3)/4*4 : (C <= 14 ? 14 : 16);
	}
// The k_posterior_sm instantiation for size class cm, launched with one PostParams argument; nullptr if
// cm is not a size class.  dump: the instantiation that writes the dense debug arrays of PostParams
// (mb200_calc_post_dense).
const void *mb_post_sm_kernel(bool mega, bool dump, int cm);
