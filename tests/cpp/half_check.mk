# Builds half_check (CUDAArray<half>: load half, compute in float, store half, against the reference's host half) with
# the compiler and link settings of this directory's Makefile:  make -C tests/cpp -f half_check.mk
include Makefile

half_check: half_check.cpp $(HDRS)
	g++ $(CXXF) $< -o $@ $(LIBS)

.DEFAULT_GOAL := half_check
