# Builds the SIMT-emulated copy of the inflate kernels (test infrastructure only).  make -C tests/emu -f inflate.mk
CXX ?= g++
CXXFLAGS ?= -O1 -g -fPIC -std=c++17 -Wall -Wno-unused-function -Wno-unused-variable -Wno-unknown-pragmas -I.
all: libb2c_emu_inflate.so
libb2c_emu_inflate.so: simt_emu.cpp emu_inflate.cpp simt_emu.h $(wildcard ../../compress_b200/csrc/*.cuh)
	$(CXX) $(CXXFLAGS) -shared -o $@ simt_emu.cpp emu_inflate.cpp
clean:
	rm -f libb2c_emu_inflate.so
