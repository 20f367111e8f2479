# oracle/root_motion.mk -- builds the root motion oracles with the flags of oracle/Makefile. TEST INFRASTRUCTURE ONLY.
#   liboracle_root_motion.so           the port's qvv_inverse and root motion composition (root_motion_oracle.c over acl_oracle.c)
#   _ref/libaclref_root_motion.so      the unmodified reference's rtm::qvv_inverse / rtm::qvv_mul and its whole decode path
#                                      (ref_root_motion.cpp), only where the reference tree exists
ACL_REF ?= /root/reference
CC      ?= gcc
CXX     ?= g++
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
PORT_FLAGS := -std=c11 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -Wall -Wextra
REF_FLAGS  := -std=c++14 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread \
              -static-libstdc++ -static-libgcc \
              -I$(ACL_REF)/includes -I$(ACL_REF)/external/rtm/includes

all: port ref

port: $(HERE)liboracle_root_motion.so
$(HERE)liboracle_root_motion.so: $(HERE)root_motion_oracle.c $(HERE)acl_oracle.c $(HERE)acl_oracle.h
	$(CC) $(PORT_FLAGS) -o $@ $(HERE)root_motion_oracle.c -lm

ifneq ($(wildcard $(ACL_REF)/includes/acl/version.h),)
ref: $(HERE)_ref/libaclref_root_motion.so
$(HERE)_ref/libaclref_root_motion.so: $(HERE)ref_root_motion.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(REF_FLAGS) -o $@ $(HERE)ref_root_motion.cpp
else
ref:
	@echo "reference tree $(ACL_REF) not present: keeping the prebuilt oracle/_ref/libaclref_root_motion.so (if any)"
endif

.PHONY: all port ref
