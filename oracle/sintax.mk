# oracle/sintax.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# oracle/_ref/libvsref_sintax.so: sintax_shim.cpp (the reference's SINTAX bootstraps behind a C ABI) linked against
# the untouched reference objects, next to the reference CLI the --tabbedout parity tests run.  Everything else
# (flags, objects, the reference itself) comes from Makefile:  make -f sintax.mk sintax
include Makefile

$(OUT)/libvsref_sintax.so: sintax_shim.cpp $(OUT)/libvsearch_ref.a
	$(CXX) $(CXXFL) -shared -o $@ sintax_shim.cpp $(OUT)/libvsearch_ref.a -lpthread -ldl

.PHONY: sintax
ifneq ($(wildcard $(SRC)/vsearch.cc),)
sintax: $(OUT)/vsearch $(OUT)/libvsref_sintax.so
else
sintax:
	@echo "reference sources not present at $(SRC): using prebuilt $(OUT)/ if any"
endif
