package org.nd4j.linalg.learning.config;
/** new NoOp(): u = g (the parameters move by the raw gradient after the division by the minibatch size); no learning rate. */
public class NoOp implements IUpdater {
    public int kind() { return 3; } public float lr() { return 0f; } public float beta1() { return 0f; } public float beta2() { return 0f; } public float eps() { return 0f; }
}
