# TEST INFRASTRUCTURE ONLY.  The reference's pulse-blanking input filter (pulse_blanking_cc.cc) compiled WHERE IT LIES, with
# the harness oracle/ref_input_filter.cc, into oracle/_ref/liboracle_ref_filter.so, which tests/pulse_blanking_np.py loads.
# Third-party headers come from oracle/shim, with oracle/shim_input_filter ahead of it for what only the blanker uses: one more
# VOLK kernel and Boost's chi-squared quantile.
# Skipped, keeping a prebuilt library, where the reference tree is absent.
#
#   make -C oracle -f filter.mk

REF ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
VG := $(REF)/src/algorithms/libs/volk_gnsssdr_module/volk_gnsssdr
A := $(REF)/src/algorithms
C := $(REF)/src/core
# the system compilers, which link libstdc++.so dynamically (as oracle/Makefile explains)
CC  := $(firstword $(wildcard /usr/bin/gcc) gcc)
CXX := $(firstword $(wildcard /usr/bin/g++) g++)
DEFS := -DUSE_GLOG_AND_GFLAGS=1 -DGNURADIO_GREATER_THAN_38=1 -DGNURADIO_USES_STD_POINTERS=1 -DLV_HAVE_GENERIC -DHAVE_POSIX_MEMALIGN=1
INC := -I$(HERE)shim_input_filter -I$(HERE)shim -I$(VG)/include -I$(C)/interfaces -I$(A)/input_filter/gnuradio_blocks
# -ffp-contract=off: every float product and sum rounds on its own, as the generic VOLK kernels state
CXXFLAGS := -std=c++20 -O2 -fPIC -ffp-contract=off
OUT := $(HERE)_ref/liboracle_ref_filter.so
OBJ := $(HERE)_ref/filter
SRC := $(A)/input_filter/gnuradio_blocks/pulse_blanking_cc.cc

.PHONY: all
all:
	@if [ -f "$(SRC)" ]; then $(MAKE) -f $(HERE)filter.mk $(OUT); \
	else echo "oracle: $(REF) absent - keeping prebuilt $(OUT) (if any)"; fi

$(OUT): $(HERE)ref_input_filter.cc $(SRC) $(HERE)shim_input_filter/volk/volk.h $(HERE)shim/volk/volk.h \
  $(HERE)shim_input_filter/boost/math/distributions/chi_squared.hpp $(HERE)shim/boost/math/special_functions/gamma.hpp
	mkdir -p $(OBJ)
	$(CXX) $(CXXFLAGS) -w $(DEFS) $(INC) -c $(SRC) -o $(OBJ)/pulse_blanking_cc.o
	$(CC) -std=gnu11 -O2 -fPIC $(DEFS) -I$(HERE)shim -I$(VG)/include -w -c $(VG)/lib/volk_gnsssdr_malloc.c -o $(OBJ)/volk_gnsssdr_malloc.o
	$(CXX) $(CXXFLAGS) -Wall $(DEFS) $(INC) -c $(HERE)ref_input_filter.cc -o $(OBJ)/ref_input_filter.o
	$(CXX) -shared -o $@ $(OBJ)/pulse_blanking_cc.o $(OBJ)/volk_gnsssdr_malloc.o $(OBJ)/ref_input_filter.o -lm
