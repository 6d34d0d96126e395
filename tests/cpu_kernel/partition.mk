# Builds libemu_partition.so: the kernels of enoki_b200/csrc/ek_partition.cu compiled as HOST code (cuda_shim.h)
# together with emu_fast.cpp, whose emulator runtime they run on (see emu_partition.cpp).  Same flags as the Makefile.
#     make -C tests/cpu_kernel -f partition.mk
CXX ?= g++
libemu_partition.so: emu_partition.cpp emu_fast.cpp cuda_shim.h ../../enoki_b200/csrc/ek_partition.cu ../../enoki_b200/csrc/ek_sweep_fast.cu ../../enoki_b200/csrc/ek_sweep_common.cuh ../../enoki_b200/csrc/ek_math.cuh ../../enoki_b200/csrc/ek_isa.h
	$(CXX) -std=c++17 -O1 -g -fPIC -shared -x c++ -include cuda_shim.h -msse2 -mfma -mavx2 -ffp-contract=off -fno-strict-aliasing -w \
	    -o $@ emu_partition.cpp -lpthread
