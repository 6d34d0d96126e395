# Builds ell_check (the native Float32 carlson_rf / carlson_rd / carlson_rc against the traced bodies of special.h) with
# the compiler and link settings of this directory's Makefile, plus -DNDEBUG (special.h's domain asserts would abort on
# the invalid inputs it compares as well):
#   make -C tests/cpp -f ell_check.mk
include Makefile

ell_check: ell_check.cpp $(HDRS) $(ROOT)/oracle/_ref/autodiff_off.o
	g++ $(CXXF) -DNDEBUG $< $(ROOT)/oracle/_ref/autodiff_off.o -o $@ $(LIBS)

.DEFAULT_GOAL := ell_check
