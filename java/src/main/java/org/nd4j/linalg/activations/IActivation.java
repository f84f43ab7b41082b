package org.nd4j.linalg.activations;
/** An activation with its parameter, for Layer.Builder.activation(IActivation): the b2g_activation code and the value carried in act_alpha. */
public interface IActivation { int code(); float alpha(); }
