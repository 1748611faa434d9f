# Builds the SIMT-emulated copy of the stateless deflate kernels (test infrastructure only).  make -C tests/emu -f deflate.mk
# -ffp-contract=off: the kernels' float32 / float64 estimates stay one rounded operation each, as on the device.
CXX ?= g++
CXXFLAGS ?= -O1 -g -fPIC -std=c++17 -Wall -Wno-unused-function -Wno-unused-variable -Wno-unknown-pragmas -I.
all: libb2c_emu_deflate.so
libb2c_emu_deflate.so: simt_emu.cpp emu_deflate.cpp simt_emu.h $(wildcard ../../compress_b200/csrc/*.cuh)
	$(CXX) $(CXXFLAGS) -ffp-contract=off -shared -o $@ simt_emu.cpp emu_deflate.cpp
clean:
	rm -f libb2c_emu_deflate.so
