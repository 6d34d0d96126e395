# Builds trig_check (the native Float32 tan / cot / asin / acos / atan / atan2 against array_math.h's traced bodies, and
# DiffArray<CUDAArray<float>> gradients against the reference CPU tape) with the compiler and link settings of this
# directory's Makefile:  make -C tests/cpp -f trig_check.mk
include Makefile

trig_check: trig_check.cpp $(HDRS) $(ROOT)/oracle/_ref/autodiff_off.o
	g++ $(CXXF) $< $(ROOT)/oracle/_ref/autodiff_off.o -o $@ $(LIBS)

.DEFAULT_GOAL := trig_check
