# Builds the SIMT-emulated copy of the HuffmanOnly / NoCompression kernels (test infrastructure only).
# make -C tests/emu -f flate_nolz.mk
# -ffp-contract=off: the kernels' float64 test stays one rounded operation each, as on the device.
CXX ?= g++
CXXFLAGS ?= -O1 -g -fPIC -std=c++17 -Wall -Wno-unused-function -Wno-unused-variable -Wno-unknown-pragmas -I.
all: libb2c_emu_flate_nolz.so
libb2c_emu_flate_nolz.so: simt_emu.cpp emu_flate_nolz.cpp simt_emu.h $(wildcard ../../compress_b200/csrc/*.cuh)
	$(CXX) $(CXXFLAGS) -ffp-contract=off -shared -o $@ simt_emu.cpp emu_flate_nolz.cpp
clean:
	rm -f libb2c_emu_flate_nolz.so
