# Builds special_check (the native Float32 erf / erfc / erfinv / lgamma / tgamma against special.h's traced bodies) with
# the compiler and link settings of this directory's Makefile:  make -C tests/cpp -f special_check.mk
include Makefile

special_check: special_check.cpp $(HDRS) $(ROOT)/oracle/_ref/autodiff_off.o
	g++ $(CXXF) $< $(ROOT)/oracle/_ref/autodiff_off.o -o $@ $(LIBS)

.DEFAULT_GOAL := special_check
