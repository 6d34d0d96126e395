# Builds printf_check (cuda_printf through the reference's own template) with the compiler and link settings of
# this directory's Makefile:  make -C tests/cpp -f printf_check.mk
include Makefile

printf_check: printf_check.cpp $(HDRS)
	g++ $(CXXF) $< -o $@ $(LIBS)

.DEFAULT_GOAL := printf_check
