# TEST INFRASTRUCTURE ONLY.  The reference's notch input filters (notch_cc.cc, notch_lite_cc.cc) compiled WHERE THEY LIE, with
# the harness oracle/ref_notch.cc, into oracle/_ref/liboracle_ref_notch.so, which tests/notch_np.py loads.  Third-party
# headers come from oracle/shim, with oracle/shim_input_filter (Boost's chi-squared quantile) and oracle/shim_notch (the
# VOLK kernels only the notches call) ahead of it; gnss_sdr_fft.h's <gnuradio/fft/fft.h> is the shim's float32 FFT.
# Skipped, keeping a prebuilt library, where the reference tree is absent.
#
#   make -C oracle -f notch.mk

REF ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
VG := $(REF)/src/algorithms/libs/volk_gnsssdr_module/volk_gnsssdr
A := $(REF)/src/algorithms
C := $(REF)/src/core
# the system compilers, which link libstdc++.so dynamically (as oracle/Makefile explains)
CC  := $(firstword $(wildcard /usr/bin/gcc) gcc)
CXX := $(firstword $(wildcard /usr/bin/g++) g++)
DEFS := -DUSE_GLOG_AND_GFLAGS=1 -DGNURADIO_GREATER_THAN_38=1 -DGNURADIO_USES_STD_POINTERS=1 -DGNURADIO_FFT_USES_TEMPLATES=1 \
  -DLV_HAVE_GENERIC -DHAVE_POSIX_MEMALIGN=1
INC := -I$(HERE)shim_notch -I$(HERE)shim_input_filter -I$(HERE)shim -I$(VG)/include -I$(C)/interfaces -I$(A)/libs \
  -I$(A)/input_filter/gnuradio_blocks
# -ffp-contract=off: every float product and sum rounds on its own, as the generic VOLK kernels state
CXXFLAGS := -std=c++20 -O2 -fPIC -ffp-contract=off
OUT := $(HERE)_ref/liboracle_ref_notch.so
OBJ := $(HERE)_ref/notch
B := $(A)/input_filter/gnuradio_blocks
SRC := $(B)/notch_cc.cc $(B)/notch_lite_cc.cc

.PHONY: all
all:
	@if [ -f "$(B)/notch_cc.cc" ]; then $(MAKE) -f $(HERE)notch.mk $(OUT); \
	else echo "oracle: $(REF) absent - keeping prebuilt $(OUT) (if any)"; fi

$(OUT): $(HERE)ref_notch.cc $(SRC) $(HERE)shim_notch/volk/volk.h $(HERE)shim_input_filter/volk/volk.h $(HERE)shim/volk/volk.h \
  $(HERE)shim/gnuradio/fft/fft.h $(HERE)shim_input_filter/boost/math/distributions/chi_squared.hpp
	mkdir -p $(OBJ)
	$(CXX) $(CXXFLAGS) -w $(DEFS) $(INC) -c $(B)/notch_cc.cc -o $(OBJ)/notch_cc.o
	$(CXX) $(CXXFLAGS) -w $(DEFS) $(INC) -c $(B)/notch_lite_cc.cc -o $(OBJ)/notch_lite_cc.o
	$(CC) -std=gnu11 -O2 -fPIC $(DEFS) -I$(HERE)shim -I$(VG)/include -w -c $(VG)/lib/volk_gnsssdr_malloc.c -o $(OBJ)/volk_gnsssdr_malloc.o
	$(CXX) $(CXXFLAGS) -Wall $(DEFS) $(INC) -c $(HERE)ref_notch.cc -o $(OBJ)/ref_notch.o
	$(CXX) -shared -o $@ $(OBJ)/notch_cc.o $(OBJ)/notch_lite_cc.o $(OBJ)/volk_gnsssdr_malloc.o $(OBJ)/ref_notch.o -lm
