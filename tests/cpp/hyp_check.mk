# Builds hyp_check (the native Float32 sinh / cosh / tanh / asinh / acosh / atanh / cbrt / sincosh against array_math.h's
# traced bodies, and DiffArray<CUDAArray<float>> gradients against the reference CPU tape) with the compiler and link
# settings of this directory's Makefile:  make -C tests/cpp -f hyp_check.mk
include Makefile

hyp_check: hyp_check.cpp $(HDRS) $(ROOT)/oracle/_ref/autodiff_off.o
	g++ $(CXXF) $< $(ROOT)/oracle/_ref/autodiff_off.o -o $@ $(LIBS)

.DEFAULT_GOAL := hyp_check
