# oracle/database.mk -- builds _ref/libaclref_db.so (oracle/ref_database.cpp: the reference's streaming database path) with the flags of
# oracle/Makefile, only where the reference tree exists. TEST INFRASTRUCTURE ONLY.
ACL_REF ?= /root/reference
CXX     ?= g++
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF_FLAGS := -std=c++14 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread \
             -static-libstdc++ -static-libgcc \
             -I$(ACL_REF)/includes -I$(ACL_REF)/external/rtm/includes

ifneq ($(wildcard $(ACL_REF)/includes/acl/version.h),)
all: $(HERE)_ref/libaclref_db.so
$(HERE)_ref/libaclref_db.so: $(HERE)ref_database.cpp $(HERE)ref_tool.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(REF_FLAGS) -o $@ $(HERE)ref_database.cpp
else
all:
	@echo "reference tree $(ACL_REF) not present: keeping the prebuilt oracle/_ref/libaclref_db.so (if any)"
endif

.PHONY: all
