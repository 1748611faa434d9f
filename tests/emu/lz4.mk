# Builds the SIMT-emulated copy of the LZ4 conversion kernels (test infrastructure only).  make -C tests/emu -f lz4.mk
CXX ?= g++
CXXFLAGS ?= -O1 -g -fPIC -std=c++17 -Wall -Wno-unused-function -Wno-unused-variable -Wno-unknown-pragmas -I.
all: libb2c_emu_lz4.so
libb2c_emu_lz4.so: simt_emu.cpp emu_lz4.cpp simt_emu.h $(wildcard ../../compress_b200/csrc/*.cuh)
	$(CXX) $(CXXFLAGS) -shared -o $@ simt_emu.cpp emu_lz4.cpp
clean:
	rm -f libb2c_emu_lz4.so
