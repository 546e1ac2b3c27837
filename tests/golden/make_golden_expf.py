"""Writes tests/golden/expf_glibc.npz: the host libm's expf (glibc 2.39 when it was made) on every 4096th
float in [-4.7, -0.0] and on the 4096 floats nearest logf(0.01f) (bits 0xc0935d8e - 2048 ..
0xc0935d8e + 2047), as float32 bits.  test_logadd_expf_cpu.py::test_host_expf_is_glibc_2_39 checks the
host that runs the suite still computes these.

  python tests/golden/make_golden_expf.py
"""
import ctypes
import ctypes.util
import os
import platform
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
	libm = ctypes.CDLL(ctypes.util.find_library("m"))
	libm.expf.restype = ctypes.c_float
	libm.expf.argtypes = [ctypes.c_float]
	lo, hi = 0x80000000, int(np.float32(-4.7).view(np.uint32))
	near = 0xc0935d8e
	xb = np.unique(np.concatenate([np.arange(lo, hi + 1, 4096, dtype=np.uint64),
	  np.arange(near - 2048, near + 2048, dtype=np.uint64)])).astype(np.uint32)
	y = np.array([libm.expf(float(v)) for v in xb.view(np.float32)], np.float32)
	np.savez_compressed(os.path.join(HERE, "expf_glibc.npz"), x_bits=xb, expf_bits=y.view(np.uint32),
	  libc=np.array("%s %s" % platform.libc_ver()))
	print("%d values, %s" % (xb.size, platform.libc_ver()))


if __name__ == "__main__":
	main()
