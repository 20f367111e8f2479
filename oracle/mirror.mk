# oracle/mirror.mk -- builds the mirror oracles with the flags of oracle/inertialization.mk. TEST INFRASTRUCTURE ONLY.
#   liboracle_mirror.so         the mirrored row, the partner rule and the pose restated in C (mirror_oracle.c over acl_oracle.c)
#   _ref/libaclref_mirror.so    the same built from the unmodified reference's rtm::quat_mul and quat_mul_vector3 (ref_mirror.cpp), only
#                               where the reference tree exists
ACL_REF ?= /root/reference
CC      ?= gcc
CXX     ?= g++
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
PORT_FLAGS := -std=c11 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -Wall -Wextra
REF_FLAGS  := -std=c++14 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread \
              -static-libstdc++ -static-libgcc \
              -I$(ACL_REF)/includes -I$(ACL_REF)/external/rtm/includes

all: port ref

port: $(HERE)liboracle_mirror.so
$(HERE)liboracle_mirror.so: $(HERE)mirror_oracle.c $(HERE)acl_oracle.c $(HERE)acl_oracle.h
	$(CC) $(PORT_FLAGS) -o $@ $(HERE)mirror_oracle.c -lm

ifneq ($(wildcard $(ACL_REF)/includes/acl/version.h),)
ref: $(HERE)_ref/libaclref_mirror.so
$(HERE)_ref/libaclref_mirror.so: $(HERE)ref_mirror.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(REF_FLAGS) -o $@ $(HERE)ref_mirror.cpp
else
ref:
	@echo "reference tree $(ACL_REF) not present: keeping the prebuilt oracle/_ref/libaclref_mirror.so (if any)"
endif

.PHONY: all port ref
