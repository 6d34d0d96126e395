# Builds dlpack_check (CUDAArray<T>::to_dlpack / from_dlpack through include/enoki/cuda.h) with the compiler and link
# settings of this directory's Makefile; it allocates its foreign tensor with the CUDA runtime:
#   make -C tests/cpp -f dlpack_check.mk
include Makefile

dlpack_check: dlpack_check.cpp $(HDRS) $(ROOT)/include/enoki_b200_dlpack.h
	g++ $(CXXF) -I/usr/local/cuda/include $< -o $@ $(LIBS)

.DEFAULT_GOAL := dlpack_check
