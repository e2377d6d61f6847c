# oracle/fleet_hooks.mk — TEST INFRASTRUCTURE build recipe for the fleet hook check (make -C oracle -f fleet_hooks.mk).
#
#   _ref/fleet_hooks_check   M unmodified HectorSlamProcessors with recording hooks next to hsb200::SlamProcessor's
#                            group steps with the step record on and the shared hook replay (fleet_hooks_check.cpp);
#                            built where $(REFERENCE) exists and the CUDA library is built
#                            (python -m hector_slam_b200.build)
# Flags as record.mk's.
REFERENCE ?= /root/reference
REF_INC   := $(REFERENCE)/hector_mapping/include/hector_slam_lib
CXX       := $(shell command -v /usr/bin/g++ || echo g++)

HSB_LIBDIR := ../hector_slam_b200/lib
HOST       := ../hector_slam_b200/host

.PHONY: all
all: $(if $(and $(wildcard $(REF_INC)/slam_main/HectorSlamProcessor.h),$(wildcard $(HSB_LIBDIR)/libhsb200.so)),_ref/fleet_hooks_check,)

_ref/fleet_hooks_check: fleet_hooks_check.cpp $(HOST)/MatchHooksB200.h $(HOST)/SlamProcessorB200.hpp ../include/hector_slam_b200.h \
                        $(HSB_LIBDIR)/libhsb200.so
	@mkdir -p _ref
	$(CXX) -std=c++14 -O2 -pthread -I shim -I $(REF_INC) -I ../include -I $(HOST) fleet_hooks_check.cpp \
	    -o $@ -L $(HSB_LIBDIR) -lhsb200 -Wl,-rpath,'$$ORIGIN/../../hector_slam_b200/lib'
