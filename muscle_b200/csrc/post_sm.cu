// post_sm.cu -- launch surface of k_posterior_sm (post_kernel_sm.cuh)
#include "post_kernel_sm.cuh"
#include "launch.h"

template <bool MEGA, bool DUMP>
static const void *kernel_cm(int cm)
	{
	switch (cm)
		{
		case 4:  return (const void *) k_posterior_sm<MEGA, 4, DUMP>;
		case 8:  return (const void *) k_posterior_sm<MEGA, 8, DUMP>;
		case 12: return (const void *) k_posterior_sm<MEGA, 12, DUMP>;
		case 14: return (const void *) k_posterior_sm<MEGA, 14, DUMP>;
		case 16: return (const void *) k_posterior_sm<MEGA, 16, DUMP>;
		default: return nullptr;
		}
	}

const void *mb_post_sm_kernel(bool mega, bool dump, int cm)
	{
	if (mega)
		return dump ? kernel_cm<true, true>(cm) : kernel_cm<true, false>(cm);
	return dump ? kernel_cm<false, true>(cm) : kernel_cm<false, false>(cm);
	}
