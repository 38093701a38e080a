# oracle/indel_reads.mk -- TEST INFRASTRUCTURE.  Builds the scalar restatement of the K6 -> K5b link (libindel_reads_oracle.so), with the
# flags of oracle/somatic_indel.mk.
CXX ?= g++
CXXFLAGS = -std=gnu++14 -O3 -fomit-frame-pointer -ffp-contract=off -fPIC -Wall -I../include

libindel_reads_oracle.so: indel_reads_oracle.cpp ../include/strelka_b200.h
	$(CXX) $(CXXFLAGS) -shared -o $@ indel_reads_oracle.cpp

.PHONY: clean
clean:
	rm -f libindel_reads_oracle.so
