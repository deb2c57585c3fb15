# tests/native/stamp.mk -- TEST INFRASTRUCTURE: the stamped ring frame model (B200_RING_STAMPED) and the
# b200_pair_ops tables over it.
# make -C tests/native -f stamp.mk
ROOT := ../..
all: libstamp_oracle.so
liboracle_pair_ops.so: oracle_pair_ops.c $(ROOT)/include/b200_endpoint.h $(ROOT)/oracle/liboracle.so
	$(MAKE) -f Makefile $@
libstamp_oracle.so: stamp_oracle.c liboracle_pair_ops.so $(ROOT)/include/b200_endpoint.h $(ROOT)/oracle/rb_oracle.h $(ROOT)/oracle/liboracle.so
	gcc -O2 -g -std=gnu11 -fPIC -shared -Wall -o $@ stamp_oracle.c -L. -loracle_pair_ops -L$(ROOT)/oracle -loracle -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/$(ROOT)/oracle'
.PHONY: all
