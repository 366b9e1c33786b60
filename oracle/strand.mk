# oracle/strand.mk — TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# The clustering-session driver with --strand both (seam2_cluster_strand_driver.cpp), linked like
# seam2_cluster_driver_ref / _gpu in Makefile: once against the untouched reference, once against the reference
# objects with cluster_session_* / cluster_assign_* replaced by shim/cluster_session_vsg.cpp.  Everything else
# (flags, objects, the reference itself) comes from Makefile:  make -f strand.mk strand
include Makefile

$(OUT)/seam2_cluster_strand_driver_ref: seam2_cluster_strand_driver.cpp seam2_cluster_driver.cpp $(OUT)/libvsearch_ref.a
	$(CXX) $(CXXFL) -I. -o $@ $< $(OUT)/libvsearch_ref.a -lpthread -ldl
$(OUT)/seam2_cluster_strand_driver_gpu: seam2_cluster_strand_driver.cpp seam2_cluster_driver.cpp $(SEAM2C_OBJS) $(VSG_DIR)/libvsg.so
	$(CXX) $(CXXFL) -I. -o $@ $< $(SEAM2C_OBJS) -L$(VSG_DIR) -lvsg -Wl,-rpath,'$$ORIGIN/../../vsearch_b200/csrc' -lpthread -ldl

.PHONY: strand
ifneq ($(wildcard $(SRC)/vsearch.cc),)
strand: ref $(OUT)/seam2_cluster_strand_driver_ref $(OUT)/seam2_cluster_strand_driver_gpu
else
strand:
	@echo "reference sources not present at $(SRC): using prebuilt $(OUT)/ if any"
endif
