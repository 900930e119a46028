# TEST INFRASTRUCTURE ONLY.  The reference sampling driver (oracle/ref_sample_driver.cpp), built with the variables
# and objects of oracle/Makefile:
#
#   make -C oracle -f Makefile -f sample.mk sample   -> oracle/_ref/nts_ref_sample_driver
.PHONY: sample
sample: $(OUT)/nts_ref_sample_driver $(OUT)/data/.stamp

$(OBJ)/ref_sample_driver.o: $(HERE)ref_sample_driver.cpp
	mkdir -p $(OBJ)
	g++ $(REF_CXX) $(REF_INC) -c $< -o $@

$(OUT)/nts_ref_sample_driver: $(OBJ)/ref_sample_driver.o $(OBJ)/GraphSegment.o $(OBJ)/network.o
	g++ $^ -o $@ $(REF_LD)
