# oracle/skinning.mk -- builds the skinning oracles with the flags of oracle/Makefile. TEST INFRASTRUCTURE ONLY.
#   liboracle_skinning.so            the port's matrix walk + matrix_mul(inverse_bind, object) (skinning_oracle.c over acl_oracle.c)
#   _ref/libaclref_skinning.so       the unmodified reference's (ref_skinning.cpp over ref_object_space.cpp), only where the reference tree exists
ACL_REF ?= /root/reference
CC      ?= gcc
CXX     ?= g++
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
PORT_FLAGS := -std=c11 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -Wall -Wextra
REF_FLAGS  := -std=c++14 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread \
              -static-libstdc++ -static-libgcc \
              -I$(ACL_REF)/includes -I$(ACL_REF)/external/rtm/includes

all: port ref

port: $(HERE)liboracle_skinning.so
$(HERE)liboracle_skinning.so: $(HERE)skinning_oracle.c $(HERE)acl_oracle.c $(HERE)acl_oracle.h
	$(CC) $(PORT_FLAGS) -o $@ $(HERE)skinning_oracle.c -lm

ifneq ($(wildcard $(ACL_REF)/includes/acl/version.h),)
ref: $(HERE)_ref/libaclref_skinning.so
$(HERE)_ref/libaclref_skinning.so: $(HERE)ref_skinning.cpp $(HERE)ref_object_space.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(REF_FLAGS) -o $@ $(HERE)ref_skinning.cpp
else
ref:
	@echo "reference tree $(ACL_REF) not present: keeping the prebuilt oracle/_ref/libaclref_skinning.so (if any)"
endif

.PHONY: all port ref
