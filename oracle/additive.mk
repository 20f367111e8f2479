# oracle/additive.mk -- builds the additive oracle with the flags of oracle/Makefile. TEST INFRASTRUCTURE ONLY.
#   _ref/libaclref_additive.so   the unmodified reference's additive compression and apply_additive_to_base (ref_additive.cpp), only where
#                                the reference tree exists
ACL_REF ?= /root/reference
CXX     ?= g++
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF_FLAGS  := -std=c++14 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread \
              -static-libstdc++ -static-libgcc \
              -I$(ACL_REF)/includes -I$(ACL_REF)/external/rtm/includes

all: ref

ifneq ($(wildcard $(ACL_REF)/includes/acl/version.h),)
ref: $(HERE)_ref/libaclref_additive.so
$(HERE)_ref/libaclref_additive.so: $(HERE)ref_additive.cpp $(HERE)ref_tool.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(REF_FLAGS) -o $@ $(HERE)ref_additive.cpp
else
ref:
	@echo "reference tree $(ACL_REF) not present: keeping the prebuilt oracle/_ref/libaclref_additive.so (if any)"
endif

.PHONY: all ref
