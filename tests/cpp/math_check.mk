# Builds math_check (the native Float32 pow / fmod / ldexp / frexp / hypot / dawson / erfi against the traced bodies of
# array_math.h and special.h) with the compiler and link settings of this directory's Makefile:
#   make -C tests/cpp -f math_check.mk
include Makefile

math_check: math_check.cpp $(HDRS) $(ROOT)/oracle/_ref/autodiff_off.o
	g++ $(CXXF) $< $(ROOT)/oracle/_ref/autodiff_off.o -o $@ $(LIBS)

.DEFAULT_GOAL := math_check
