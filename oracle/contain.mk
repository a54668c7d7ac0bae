# oracle/contain.mk -- builds _ref/libmash_ref_contain.so: the reference's OWN containSketches (CommandContain.cpp), compiled in
# place from $(REF) (nothing is copied) behind the grid entry point ref_contain.cpp.  Test infrastructure, like
# _ref/libmash_ref.so in oracle/Makefile; only built where $(REF) exists, the prebuilt library travels with the tree.
#
# CommandContain.cpp is the whole `within` command.  Only containSketches is wanted, and it needs nothing but HashList and
# hashLessThan, so:
#   - Sketch.h includes the generated capnp header "mash/capnp/MinHash.capnp.h", which containSketches does not use: an empty
#     stand-in is generated under _ref/stub;
#   - -ffunction-sections / --gc-sections with a version script that exports only ref_contain_grid drop the command driver and
#     with it every reference to Command / Sketch, which are not linked;
#   - `-include limits` as in oracle/Makefile (robin_hood.h under GCC 13).
REF ?= /root/reference/src/mash
CXX ?= g++
STUB := _ref/stub

all:
	@if [ -d $(REF) ]; then $(MAKE) -f contain.mk _ref/libmash_ref_contain.so; else echo "reference sources absent: keeping prebuilt oracle/_ref (if any)"; fi

$(STUB)/mash/capnp/MinHash.capnp.h:
	mkdir -p $(dir $@)
	: > $@

_ref/ref_contain.map:
	mkdir -p _ref
	echo '{ global: ref_contain_grid; local: *; };' > $@

_ref/libmash_ref_contain.so: ref_contain.cpp $(REF)/CommandContain.cpp $(REF)/HashList.cpp $(REF)/hash.cpp $(REF)/MurmurHash3.cpp \
                             $(STUB)/mash/capnp/MinHash.capnp.h _ref/ref_contain.map
	$(CXX) -O3 -std=c++14 -include limits -fPIC -shared -pthread -ffunction-sections -fdata-sections -Wl,--gc-sections \
	    -Wl,--version-script=_ref/ref_contain.map -Wl,--no-undefined -I$(REF) -I$(STUB) -o $@ \
	    ref_contain.cpp $(REF)/CommandContain.cpp $(REF)/HashList.cpp $(REF)/hash.cpp $(REF)/MurmurHash3.cpp -lz

.PHONY: all
