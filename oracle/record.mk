# oracle/record.mk — TEST INFRASTRUCTURE build recipe for the per-evaluation match record (make -C oracle -f record.mk).
#
#   _build/libhsoracle_record.so   the C port + hso_match_record (port_record.c); builds anywhere
#   _ref/libhsref_record.so        the reference driver + hsref_match_record with recording draw / debug hooks
#                                  (ref_record_driver.cpp), where $(REFERENCE) exists
#   _ref/dropin_hooks_check        the unmodified façade with recording hooks on MapRepMultiMap and on MapRepB200
#                                  (needs the CUDA library built: python -m hector_slam_b200.build)
# Flags as oracle/Makefile's.
REFERENCE ?= /root/reference
REF_INC   := $(REFERENCE)/hector_mapping/include/hector_slam_lib
CXX       := $(shell command -v /usr/bin/g++ || echo g++)
CC        := $(shell command -v /usr/bin/gcc || echo gcc)
CXXFLAGS  := -std=c++14 -O2 -fPIC -pthread
CFLAGS    := -std=c99 -O2 -fPIC -pthread -Wall

HSB_LIBDIR := ../hector_slam_b200/lib

.PHONY: all port ref
all: port $(if $(wildcard $(REF_INC)/slam_main/HectorSlamProcessor.h),ref,)

port: _build/libhsoracle_record.so
ref: _ref/libhsref_record.so $(if $(wildcard $(HSB_LIBDIR)/libhsb200.so),_ref/dropin_hooks_check,)

_build/libhsoracle_record.so: port_record.c hs_oracle.c
	@mkdir -p _build
	$(CC) $(CFLAGS) -shared port_record.c -o $@ -lm

_ref/libhsref_record.so: ref_record_driver.cpp ref_driver.cpp shim/Eigen/Core shim/Eigen/Geometry shim/Eigen/LU
	@mkdir -p _ref
	$(CXX) $(CXXFLAGS) -shared -I shim -I $(REF_INC) -I . ref_record_driver.cpp -o $@

_ref/dropin_hooks_check: dropin_hooks_check.cpp ../hector_slam_b200/host/MapRepB200.h ../include/hector_slam_b200.h $(HSB_LIBDIR)/libhsb200.so
	@mkdir -p _ref
	$(CXX) -std=c++14 -O2 -pthread -I shim -I $(REF_INC) -I ../include -I ../hector_slam_b200/host dropin_hooks_check.cpp \
	    -o $@ -L $(HSB_LIBDIR) -lhsb200 -Wl,-rpath,'$$ORIGIN/../../hector_slam_b200/lib'
